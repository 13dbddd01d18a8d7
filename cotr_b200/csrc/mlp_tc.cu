// Fused transformer feed-forward block for sm_90a, one launch per layer:
//     out = LN(x + W2 relu(W1 x + b1) + b2)        (optionally followed by a second LayerNorm)
//
// At small sections (a few hundred to ~2000 rows) the two GEMMs and the LayerNorm of a feed-forward block are three
// latency-bound launches, and the 1024-wide hidden activation makes a round trip through L2.  Every step of the block
// is row-local, so one BM = 64-row tile is finished by one thread-block cluster of S CTAs that split the HIDDEN
// dimension: CTA s owns hidden columns [s 1024/S, (s+1) 1024/S) and streams only its own slice of W1 (rows) and of W2
// (K chunks) - both are contiguous in the tc_pack_weight images.  Numerics are those of gemm_tc.cu (split16 operands,
// three m64 wgmma per k16 step, separate correction accumulator, fp32 RN sums in the epilogue).
//
// CTA = 3 warpgroups.  Warpgroup 2 stages x by cp.async and issues the weight TMA (the first stages before the
// dependency wait: weights are constants); warpgroups 0-1 issue the wgmma, splitting the columns of each phase:
//   phase 1  h_s = relu(x W1[slice]^T * s1 + b1[slice]), 64 x HS over K = 256; h_s is split to fp16 hi / lo and written
//            straight into shared memory in the SWIZZLE_128B K-major layout, where it is the A operand of phase 2;
//   phase 2  P_s = h_s W2[:, slice]^T, a 64 x 256 fp32 partial over K = HS, parked as an fp32 tile in the idle stages;
//   phase 3  reduce-scatter over the cluster by rows (as gemm_tc.cu's split-K): CTA s owns rows [s 64/S, (s+1) 64/S) of
//            the tile; every CTA pushes the rows it does not own into the owner's shared memory (st.async, transaction
//            bytes on the owner's mbarrier).  The owner adds the peers' partials in rank order, undoes the weight
//            pre-scaling, adds b2 and the residual x and applies the LayerNorm(s), one warp per row.
// In-place use (out == x, the decoder) is safe: the only reads of x are the phase-1 loads of this tile's rows by the
// CTAs of this cluster, and the residual read of a row by the warp that later writes it.  Every CTA arrives on the
// cluster barrier only after all of its MMAs - and so all of its x loads - are complete, and no row is written before
// that barrier.  Row tiles of different clusters are disjoint.
#include "split16.cuh"
#include "tc_common.cuh"

namespace cotr {

namespace {

using namespace tc;

constexpr int BM = 64;
constexpr int BK = 64;
constexpr int kThreads = 384;               // 2 consumer warpgroups + 1 producer warpgroup
constexpr int kConsumerThreads = 256;
constexpr int kBarConsumers = 6;
constexpr int kK1Chunks = kDModel / BK;     // phase 1: K = 256

template <int S>
struct MlpCfg {
    static constexpr int HS = kFF / S;                                  // hidden columns of one CTA
    static constexpr int WN1 = HS / 2;                                  // phase-1 columns of one consumer warpgroup
    static constexpr int kMain1 = WN1 >= 128 ? 1 : 2;                   // main accumulators of phase 1 (as gemm_tc.cu)
    static constexpr int kK2Chunks = HS / BK;
    static constexpr int kIters = kK1Chunks + kK2Chunks;
    static constexpr uint32_t kAPlane = BM * 128u;                      // one fp16 plane of a 64 x 64 operand tile
    static constexpr uint32_t kW1Plane = HS * 128u;
    static constexpr uint32_t kW2Plane = kDModel * 128u;
    // a stage holds [x chunk hi | lo][W1 chunk hi | lo] in phase 1 and [W2 chunk hi | lo] in phase 2
    static constexpr uint32_t kStage1 = 2 * kAPlane + 2 * kW1Plane;
    static constexpr uint32_t kStage2 = 2 * kW2Plane;
    static constexpr uint32_t kStage = kStage1 > kStage2 ? kStage1 : kStage2;
    static constexpr uint32_t kHChunk = 2 * kAPlane;                    // 64 hidden columns of h, both planes
    static constexpr uint32_t kHBytes = kK2Chunks * kHChunk;
    static constexpr int kStages = (int)((227u * 1024u - 2048u - kHBytes) / kStage);
    static constexpr uint32_t kHOffset = kStages * kStage;
    static constexpr uint32_t kBarOffset = kHOffset + kHBytes;
    static constexpr uint32_t kSmemBytes = kBarOffset + 256 + 1024;     // + barriers + alignment slack
    // phase 3 re-uses the stages: the 64 x 256 fp32 partial tile (padded pitch), then the incoming peer rows
    static constexpr uint32_t kAccPitch = kDModel * 4u + 16u;
    static constexpr uint32_t kAccBytes = ((BM * kAccPitch + 1023u) / 1024u) * 1024u;
    static constexpr int kOwnRows = BM / S;
    static constexpr uint32_t kRowBytes = kDModel * 4u;
    static constexpr uint32_t kPartOffset = kAccBytes;
    static constexpr uint32_t kPartBytes = (S - 1) * kOwnRows * kRowBytes;
    static_assert(kStages >= 2, "pipeline needs at least two stages");
    static_assert(kSmemBytes <= 227u * 1024u, "shared memory");
    static_assert(kPartOffset + kPartBytes <= kStages * kStage, "partial tiles do not fit the idle stages");
    static_assert(kStage % 1024 == 0 && kW1Plane % 1024 == 0 && kHBytes % 1024 == 0, "SWIZZLE_128B needs 1024-byte alignment");
};

template <int S>
__global__ void __launch_bounds__(kThreads, 1) mlp_tc_kernel(const MlpParams p) {
    using C = MlpCfg<S>;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw_addr = smem_u32(smem_raw);
    uint8_t* base = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
    uint8_t* h_tile = base + C::kHOffset;
    uint64_t* full = reinterpret_cast<uint64_t*>(base + C::kBarOffset);
    uint64_t* empty = full + C::kStages;
    uint64_t* part_full = full + 2 * C::kStages;           // the peers' partial rows of this CTA's rows have landed

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int rank = blockIdx.z;                           // rank in the 1 x 1 x S cluster
    const int m0 = blockIdx.x * BM;
    const int h0 = rank * C::HS;

    if (threadIdx.x == 0) {
        for (int s = 0; s < C::kStages; ++s) {
            mbar_init(&full[s], 129);
            mbar_init(&empty[s], 8);          // one arrival per consumer warp
        }
        mbar_init(part_full, 1);
        mbar_fence_init();
        mbar_arrive_expect_tx(part_full, C::kPartBytes);
    }
    __syncthreads();

    if (warp >= 8) {
        // ================= producer warpgroup: x by cp.async, weight slices by bulk TMA =================================
        const int t = threadIdx.x - kConsumerThreads;
        const int kg = t & 7;          // 16-byte K group inside the 64-wide chunk
        const int rb = t >> 3;         // rows rb, rb+16, ...
        const uint8_t* w1 = reinterpret_cast<const uint8_t*>(p.w1);
        const uint8_t* w2 = reinterpret_cast<const uint8_t*>(p.w2);
        // images: [k chunk][plane][npad rows][128 bytes]; W1 (npad 1024): rows [h0, h0 + HS) of each (chunk, plane);
        // W2 (npad 256): K chunks h0 / 64 .., both planes of a chunk adjacent
        auto load_weights = [&](int it) {
            const int s = it % C::kStages;
            uint8_t* dst = base + (size_t)s * C::kStage;
            if (it < kK1Chunks) {
                mbar_arrive_expect_tx(&full[s], 2u * C::kW1Plane);
                const uint8_t* src = w1 + ((size_t)(it * 2) * kFF + h0) * 128;
                tma_bulk_g2s(dst + 2 * C::kAPlane, src, C::kW1Plane, &full[s]);
                tma_bulk_g2s(dst + 2 * C::kAPlane + C::kW1Plane, src + (size_t)kFF * 128, C::kW1Plane, &full[s]);
            } else {
                mbar_arrive_expect_tx(&full[s], C::kStage2);
                tma_bulk_g2s(dst, w2 + (size_t)(h0 / BK + it - kK1Chunks) * C::kStage2, C::kStage2, &full[s]);
            }
        };
        if (t == 0) {
            for (int it = 0; it < C::kStages; ++it) load_weights(it);
            pdl_launch_dependents();
        }
        pdl_wait();
        const uint32_t a_off = (uint32_t)rb * 128u + (uint32_t)((kg ^ (rb & 7)) << 4);   // swizzled chunk position
#pragma unroll 1
        for (int it = 0; it < C::kIters; ++it) {
            const int s = it % C::kStages;
            const uint32_t ph = (uint32_t)(it / C::kStages) & 1u;
            mbar_wait(&empty[s], ph ^ 1u);
            if (t == 0 && it >= C::kStages) load_weights(it);
            if (it < kK1Chunks) {
                const uint32_t dst = smem_u32(base + (size_t)s * C::kStage) + a_off;
                const int k = it * BK + kg * 8;
#pragma unroll
                for (int i = 0; i < BM / 16; ++i) {
                    const int row = m0 + rb + 16 * i;
                    const bool ok = row < p.M;
                    const size_t off = ok ? (size_t)row * kDModel + k : 0;     // src-size 0 -> 16 bytes of zeros
                    cp_async16(dst + i * 2048, p.x.hi + off, ok ? 16u : 0u);
                    cp_async16(dst + C::kAPlane + i * 2048, p.x.lo + off, ok ? 16u : 0u);
                }
                cp_async_mbar_arrive_noinc(&full[s]);
            } else {
                mbar_arrive(&full[s]);         // phase 2 stages carry weights only
            }
        }
    } else {
        // ================= consumer warpgroups ===========================================================================
        const int wg = warp >> 2;
        // accumulator fragment of m64nN: register 4 j + {0,1} = row (warp % 4) * 16 + lane / 4, columns
        // 8 j + 2 (lane % 4) + {0,1}; registers 4 j + {2,3} = the same columns 8 rows further down
        const int fr = (warp & 3) * 16 + (lane >> 2);
        const int fc = 2 * (lane & 3);
        {
            // ---- phase 1: warpgroup wg computes hidden columns [wg WN1, (wg+1) WN1) of this CTA's slice ----
            constexpr int WN = C::WN1, R = WN / 2;
            float acc_m[C::kMain1][R], acc_c[R];
#pragma unroll
            for (int a = 0; a < C::kMain1; ++a)
#pragma unroll
                for (int j = 0; j < R; ++j) acc_m[a][j] = 0.f;
#pragma unroll
            for (int j = 0; j < R; ++j) acc_c[j] = 0.f;
            auto mma = [&](float (&d)[R], uint64_t da, uint64_t db) {
                if constexpr (WN == 64) wgmma_ss_n64(d, da, db);
                else wgmma_ss_n128(d, da, db);
            };
            auto fence_all = [&]() {
#pragma unroll
                for (int a = 0; a < C::kMain1; ++a) fence_regs(acc_m[a]);
                fence_regs(acc_c);
            };
#pragma unroll 1
            for (int it = 0; it < kK1Chunks; ++it) {
                const int s = it % C::kStages;
                mbar_wait(&full[s], (uint32_t)(it / C::kStages) & 1u);
                fence_proxy_async_smem();                      // cp.async (generic proxy) data -> wgmma (async proxy)
                const uint32_t a_addr = smem_u32(base + (size_t)s * C::kStage);
                const uint32_t b_addr = a_addr + 2 * C::kAPlane + (uint32_t)wg * WN * 128u;
                fence_all();
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < BK / 16; ++ks) {
                    const uint64_t dah = make_desc_sw128(a_addr + 32 * ks);
                    const uint64_t dal = make_desc_sw128(a_addr + C::kAPlane + 32 * ks);
                    const uint64_t dbh = make_desc_sw128(b_addr + 32 * ks);
                    const uint64_t dbl = make_desc_sw128(b_addr + C::kW1Plane + 32 * ks);
                    mma(acc_c, dal, dbh);
                    mma(acc_m[ks % C::kMain1], dah, dbh);
                    mma(acc_c, dah, dbl);
                }
                wgmma_commit();
                wgmma_wait<1>();
                fence_all();
                if (it > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % C::kStages]);
            }
            wgmma_wait<0>();
            fence_all();
            if (lane == 0) mbar_arrive(&empty[(kK1Chunks - 1) % C::kStages]);
            // h = relu(acc * s1 + b1) -> split16 -> the h tile (chunk c / 64, row r: 16-byte piece (c % 64) / 8 at
            // position piece ^ (r % 8)); a warp's 32 four-byte stores hit 8 rows x 4 columns: all 32 banks
#pragma unroll
            for (int j = 0; j < R; j += 2) {
                const int row = fr + ((j >> 1) & 1) * 8;
                const int c = wg * WN + (j >> 2) * 8 + fc;                 // hidden column inside the slice
                float v[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float y = acc_m[0][j + e];
#pragma unroll
                    for (int a = 1; a < C::kMain1; ++a) y += acc_m[a][j + e];
                    v[e] = fmaxf((acc_c[j + e] + y) * p.w1_scale + __ldg(p.b1 + h0 + c + e), 0.f);
                }
                uint32_t hi, lo;
                split_f16x2(v[0], v[1], hi, lo);
                const int cc = c & 63;
                uint8_t* d = h_tile + (uint32_t)(c >> 6) * C::kHChunk + (uint32_t)row * 128u + (uint32_t)((((cc >> 3) ^ (row & 7)) << 4) + (cc & 7) * 2);
                *reinterpret_cast<uint32_t*>(d) = hi;
                *reinterpret_cast<uint32_t*>(d + C::kAPlane) = lo;
            }
            fence_proxy_async_smem();                          // h (generic-proxy stores) -> wgmma operand
            named_barrier_sync(kBarConsumers, kConsumerThreads);
        }
        {
            // ---- phase 2: warpgroup wg computes output columns [128 wg, 128 wg + 128) over K = HS ----
            float acc_m[64], acc_c[64];
#pragma unroll
            for (int j = 0; j < 64; ++j) { acc_m[j] = 0.f; acc_c[j] = 0.f; }
#pragma unroll 1
            for (int it = kK1Chunks; it < C::kIters; ++it) {
                const int s = it % C::kStages;
                mbar_wait(&full[s], (uint32_t)(it / C::kStages) & 1u);
                const uint32_t a_addr = smem_u32(h_tile) + (uint32_t)(it - kK1Chunks) * C::kHChunk;
                const uint32_t b_addr = smem_u32(base + (size_t)s * C::kStage) + (uint32_t)wg * 128u * 128u;
                fence_regs(acc_m);
                fence_regs(acc_c);
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < BK / 16; ++ks) {
                    const uint64_t dah = make_desc_sw128(a_addr + 32 * ks);
                    const uint64_t dal = make_desc_sw128(a_addr + C::kAPlane + 32 * ks);
                    const uint64_t dbh = make_desc_sw128(b_addr + 32 * ks);
                    const uint64_t dbl = make_desc_sw128(b_addr + C::kW2Plane + 32 * ks);
                    wgmma_ss_n128(acc_c, dal, dbh);
                    wgmma_ss_n128(acc_m, dah, dbh);
                    wgmma_ss_n128(acc_c, dah, dbl);
                }
                wgmma_commit();
                wgmma_wait<1>();
                fence_regs(acc_m);
                fence_regs(acc_c);
                if (it > kK1Chunks && lane == 0) mbar_arrive(&empty[(it - 1) % C::kStages]);
            }
            wgmma_wait<0>();
            fence_regs(acc_m);
            fence_regs(acc_c);
            // park the partial (correction + main, RN) as an fp32 tile once both warpgroups are done with the stages
            named_barrier_sync(kBarConsumers, kConsumerThreads);
#pragma unroll
            for (int j = 0; j < 64; j += 2) {
                const int row = fr + ((j >> 1) & 1) * 8;
                const int col = wg * 128 + (j >> 2) * 8 + fc;
                *reinterpret_cast<float2*>(base + (uint32_t)row * C::kAccPitch + col * 4) =
                    make_float2(acc_c[j] + acc_m[j], acc_c[j + 1] + acc_m[j + 1]);
            }
        }
    }

    // ================= phase 3: reduce-scatter of the partial tiles over the cluster, LayerNorm =========================
    // The cluster barrier: every CTA of the cluster has parked its partial tile, so its stages are free to receive the
    // peers' rows (and all of its x loads have completed, see the top comment).
    __syncthreads();
    cluster_arrive();
    cluster_wait();
    {
        const uint32_t part_local = smem_u32(base) + C::kPartOffset;
        constexpr int kPieces = (BM - C::kOwnRows) * (C::kRowBytes / 16);
#pragma unroll 1
        for (int i = threadIdx.x; i < kPieces; i += kThreads) {
            const int pr = i / (C::kRowBytes / 16), piece = i % (C::kRowBytes / 16);
            const int r = pr < rank * C::kOwnRows ? pr : pr + C::kOwnRows;      // a tile row this CTA does not own
            const int q = r / C::kOwnRows;                                      // its owner
            const uint32_t slot = (uint32_t)(rank < q ? rank : rank - 1);     // source slot in the owner's region
            const float4 v = *reinterpret_cast<const float4*>(base + (uint32_t)r * C::kAccPitch + piece * 16);
            const uint32_t dst = part_local + (slot * C::kOwnRows + (uint32_t)(r % C::kOwnRows)) * C::kRowBytes + piece * 16;
            st_async_f32x4(map_to_cta(dst, (uint32_t)q), v.x, v.y, v.z, v.w, map_to_cta(smem_u32(part_full), (uint32_t)q));
        }
    }
    // one warp per owned row; every warp with a row waits, valid row or not: this CTA must stay resident until the
    // peers' stores have landed
    if (warp < C::kOwnRows) mbar_wait(part_full, 0);
#pragma unroll 1
    for (int w = warp; w < C::kOwnRows; w += kThreads / 32) {
        const int rr = rank * C::kOwnRows + w;
        const int row = m0 + rr;
        if (row < p.M) {
            pdl_wait();                        // the residual comes from the previous kernels
            float v[8];
            const uint8_t* own = base + (uint32_t)rr * C::kAccPitch + lane * 32;
            const float4 a0 = *reinterpret_cast<const float4*>(own), a1 = *reinterpret_cast<const float4*>(own + 16);
            v[0] = a0.x; v[1] = a0.y; v[2] = a0.z; v[3] = a0.w; v[4] = a1.x; v[5] = a1.y; v[6] = a1.z; v[7] = a1.w;
#pragma unroll 1
            for (int slot = 0; slot < S - 1; ++slot) {
                const uint8_t* pp = base + C::kPartOffset + (uint32_t)(slot * C::kOwnRows + w) * C::kRowBytes + lane * 32;
                const float4 b0 = *reinterpret_cast<const float4*>(pp), b1 = *reinterpret_cast<const float4*>(pp + 16);
                v[0] += b0.x; v[1] += b0.y; v[2] += b0.z; v[3] += b0.w; v[4] += b1.x; v[5] += b1.y; v[6] += b1.z; v[7] += b1.w;
            }
            float bias[8], res[8];
            load_vec8(p.b2, lane, bias);
            const size_t off = (size_t)row * kDModel + lane * 8;
            load8_split(p.x, off, res);
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = v[j] * p.w2_scale + bias[j] + res[j];
            warp_layernorm256(v, p.g, p.be, lane);
            if (p.g2) warp_layernorm256(v, p.g2, p.be2, lane);
            store8_split(p.out, off, v);
        }
    }
}

template <int S>
int configure(size_t* smem) {
    static unsigned long long configured = 0;      // bit per device
    *smem = MlpCfg<S>::kSmemBytes;
    if (first_use_on_device(&configured))
        COTR_CHECK_CUDA(cudaFuncSetAttribute(mlp_tc_kernel<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MlpCfg<S>::kSmemBytes));
    return 0;
}

// Clusters of 8 of this kernel that fit the device at once (H100 SXM: GPCs of uneven size leave SMs that no cluster
// of 8 can use), cached per device.
int max_clusters_of_8(int* out) {
    static int cached[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    if (cached[dev & 63] > 0) { *out = cached[dev & 63]; return 0; }
    size_t smem = 0;
    if (configure<8>(&smem)) return 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(1, 1, 8);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 1;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 8;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int n = 0;
    COTR_CHECK_CUDA(cudaOccupancyMaxActiveClusters(&n, mlp_tc_kernel<8>, &cfg));
    cached[dev & 63] = n;
    *out = n;
    return 0;
}

template <int S>
int launch_split(const MlpParams& p, cudaStream_t s) {
    size_t smem = 0;
    if (configure<S>(&smem)) return 1;
    const dim3 grid((p.M + BM - 1) / BM, 1, S);
    COTR_CHECK_CUDA(launch_kernel_cluster(mlp_tc_kernel<S>, grid, dim3(kThreads), smem, s, S, p));
    return 0;
}

}  // namespace

int launch_mlp_tc(const MlpParams& p, cudaStream_t s) {
    COTR_CHECK(p.M > 0 && p.w1 && p.w2 && p.b1 && p.b2 && p.g && p.be && (p.g2 == nullptr) == (p.be2 == nullptr),
               "mlp_tc: bad parameters (M %d)", p.M);
    // Hidden split: 8 CTAs per row tile (each streams 1/8 of the weights) while all row tiles fit in one wave of
    // clusters of 8; beyond that, clusters of 4 (which fit where no cluster of 8 does) rather than a second wave.
    const int tiles = (p.M + BM - 1) / BM;
    int n8 = 0;
    if (max_clusters_of_8(&n8)) return 1;
    return launch_mlp_tc_split(p, tiles <= n8 ? 8 : 4, s);
}

int launch_mlp_tc_split(const MlpParams& p, int S, cudaStream_t s) {
    COTR_CHECK(S == 4 || S == 8, "mlp_tc: hidden split %d (4 or 8)", S);
    return S == 8 ? launch_split<8>(p, s) : launch_split<4>(p, s);
}

}  // namespace cotr
