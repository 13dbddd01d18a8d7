// wgmma attention over the 512-token context (encoder self-attention and decoder cross-attention), split16 I/O.
//
// One cluster of KS CTAs (KS = 1 or 2) per (128-query tile, head, image pair); CTA s of the cluster owns keys
// [s 512 / KS, (s + 1) 512 / KS), two warpgroups of 64 query rows each:
//   * all 256 threads stage Q and this CTA's slice of K and V^T of this head with asynchronous 16-byte copies (cp.async
//     -> LDGSTS, completion on an mbarrier): the operands already live in HBM as fp16 hi/lo planes and V is stored
//     transposed by the projection GEMM's epilogue, so staging is pure data movement into the wgmma K-major canonical
//     layout.  On the tensor-core schedule the K and V slices arrive instead from the operand images (common.cuh) by
//     bulk-TMA copies on two barriers, and the first Q K^T only waits for K;
//   * each warpgroup then walks its keys in chunks of 64 with an online softmax: S = Q K^T (64 x 64, fp32 registers,
//     hi/lo operand products lo*hi + hi*lo + hi*hi), the running row max and sum are kept per thread (a row is shared
//     by the 4 lanes of a quad), P = exp(S - max) is split to fp16 hi/lo straight from the accumulator fragment into
//     the register A operand of the next wgmma, and O += P_hi V_hi + P_lo V_hi + P_hi V_lo.  Because the tensor core's
//     fp32 accumulate truncates, even / odd chunks accumulate P_hi V_hi into different registers and the two small
//     products into a third set; they are summed with RN adds at the end of the CTA's chunks;
//   * KS > 1: every CTA but the cluster's leader (rank 0) pushes its unnormalised O and its row max / sum into its own
//     region of the leader's shared memory with st.async (completion bytes on a leader mbarrier, no cluster barrier
//     at the end); the leader rescales every partial to the common row max and adds them with RN fp32 arithmetic.
// Splitting the keys is for launches that would fill a fraction of the SMs (batch 1: 32 encoder / 64 decoder CTAs):
// it doubles the CTAs and halves each CTA's serial chunk chain and its K / V staging.
// q is expected pre-scaled by head_dim^-0.5 (folded into the projection weights).
#include "split16.cuh"
#include "tc_common.cuh"

namespace cotr {

namespace {

using namespace tc;

constexpr int kTile = kAttnTcTileRows;                    // 128
constexpr int kThreads = 256;                             // two warpgroups
constexpr int kChunk = 64;                                // keys per softmax chunk
constexpr int kChunks = kTokens / kChunk;                 // 8
constexpr uint32_t kQLbo = kTile * 16;                    // Q tile  [4 K-groups][128 rows][16 B]
constexpr uint32_t kQPlane = 4 * kQLbo;                   // 8 KB
constexpr uint32_t kKLbo = kTokens * 16;                  // K tile  [4 K-groups][512 keys][16 B]
constexpr uint32_t kKPlane = 4 * kKLbo;                   // 32 KB
constexpr uint32_t kVLbo = 2 * kHeadDim * 16 + 16;        // V^T tile [64 key-groups][hi: 32 d | lo: 32 d][16 B], padded against bank conflicts
constexpr uint32_t kVBytes = (kTokens / 8) * kVLbo;       // 65 KB
constexpr uint32_t kVLoOff = kHeadDim * 16;               // the lo rows of a key group follow its hi rows
constexpr uint32_t kSbo = 128;

constexpr uint32_t kOffQ = 0;
constexpr uint32_t kOffK = kOffQ + 2 * kQPlane;
constexpr uint32_t kOffV = kOffK + 2 * kKPlane;
constexpr uint32_t kOffBar = kOffV + kVBytes;
constexpr uint32_t kSmemBytes = kOffBar + 128;
// key split: the leader receives one region per peer CTA behind the barriers, [piece][thread][16 B] (conflict-free):
// pieces 0-3 the thread's 16 O values, piece 4 its rows' (max a, max b, sum a, sum b)
constexpr uint32_t kPartPiece = kThreads * 16;
constexpr uint32_t kPartSlot = 5 * kPartPiece;            // 20 KB per peer
constexpr uint32_t kOffPart = kSmemBytes;
constexpr int kMaxSplit = 2;
static_assert(kSmemBytes + (kMaxSplit - 1) * kPartSlot <= 227 * 1024, "attention tile does not fit shared memory");
// the operand images of common.cuh are byte-for-byte these shared-memory tiles
static_assert(2 * kKPlane == kAttnKImgBytes && kKPlane == kAttnKPlaneBytes && kVLbo == kAttnVGroupBytes && kVBytes == kAttnVImgBytes &&
              kOffV == kOffK + kAttnKImgBytes, "attention operand images and shared-memory tiles went out of step");

__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Capped at the 168 registers of the GEMM's budget: left free, the scheduler overlaps consecutive key chunks and takes
// more (no gain in occupancy: shared memory already limits the SM to one CTA).
template <int KS>
__global__ void __maxnreg__(168) attention_tc_kernel(const AttnParams p) {
    static_assert(KS >= 1 && KS <= kMaxSplit, "key split out of range");
    constexpr int kKeys = kTokens / KS;                   // keys of this CTA
    constexpr int kMyChunks = kChunks / KS;
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
    uint64_t* qk_full = bars + 0;
    uint64_t* v_full = bars + 1;
    uint64_t* k_img_full = bars + 2; // operand images: the bulk copies of the K slice (hi + lo planes) have landed
    uint64_t* part_full = bars + 3;  // key split, leader: every peer's partial O, max and sum have landed
    const bool img = p.kv_img != nullptr;       // keys / values arrive as operand images by bulk TMA (tensor-core schedule)

    const int t = threadIdx.x;
    const int warp = t >> 5, lane = t & 31;
    const int head = blockIdx.y;
    const int rank = blockIdx.z % KS;                     // rank in the cluster (1 x 1 x KS)
    const int key0 = rank * kKeys;
    const int chunk0 = rank * kMyChunks;
    // this CTA's query rows: q / out rows qrow0 .. qrow0 + nrows - 1 (at most kTile of them; the rest of the tile is masked)
    int pair_local, qrow0, nrows;
    if (p.tiles) {
        const int4 tl = p.tiles[blockIdx.x];
        pair_local = tl.x; qrow0 = tl.y; nrows = tl.z;
    } else {
        pair_local = blockIdx.z / KS;
        qrow0 = pair_local * p.nq + blockIdx.x * kTile;
        nrows = p.nq - blockIdx.x * kTile;
    }

    if (t == 0) {
        mbar_init(qk_full, kThreads);
        mbar_init(v_full, img ? 1 : kThreads);
        mbar_init(k_img_full, 1);
        mbar_init(part_full, 1);
        mbar_fence_init();
        if (KS > 1 && rank == 0) mbar_arrive_expect_tx(part_full, (uint32_t)(KS - 1) * kPartSlot);
    }
    __syncthreads();
    // key split: tell the cluster that this CTA runs and its barriers exist (waited for before the first remote access)
    if (KS > 1) cluster_arrive();
    const uint32_t sbase = smem_u32(smem);

    const size_t kv_row0 = (size_t)(p.pair0 + pair_local) * kTokens;
    if (t == 0) pdl_launch_dependents();             // the next kernel may start its prologue on idle SMs
    pdl_wait();                                      // prologue above overlaps the previous kernel

    if (img && t == 0) {
        // keys and values of this (pair, head, key slice): bulk-TMA copies (UBLKCP) of the operand images straight into
        // the tiles, issued by one thread before anything else; the 256 threads then only stage the 16 KB of Q.  A key
        // slice is one run per K plane and dim group, and one run of V key groups.
        const unsigned char* src = p.kv_img + (size_t)(p.pair0 + pair_local) * p.img_pair_stride + (size_t)head * kAttnHeadImgBytes;
        mbar_arrive_expect_tx(k_img_full, 2u * 4u * kKeys * 16u);
#pragma unroll
        for (int run = 0; run < (KS > 1 ? 8 : 1); ++run) {
            const uint32_t off = (uint32_t)run * kKLbo + (uint32_t)key0 * 16u;   // plane = run / 4, dim group = run % 4
            tma_bulk_g2s(smem + kOffK + off, src + off, KS > 1 ? kKeys * 16u : (uint32_t)kAttnKImgBytes, k_img_full);
        }
        const uint32_t voff = (uint32_t)(key0 / 8) * kVLbo;
        mbar_arrive_expect_tx(v_full, (uint32_t)(kKeys / 8) * kVLbo);
        tma_bulk_g2s(smem + kOffV + voff, src + kAttnKImgBytes + voff, (uint32_t)(kKeys / 8) * kVLbo, v_full);
    }
    // ---- stage Q (row t % 128, two of the four 16-byte K groups per thread) and K (kKeys / 128 keys per thread) -----
    {
        const int r = t & 127, kg0 = (t >> 7) * 2;
        const bool ok = r < nrows;
        const size_t qoff = ((size_t)qrow0 + (ok ? r : 0)) * p.ldq + head * kHeadDim;
        const uint32_t bytes = ok ? 16u : 0u;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int kg = kg0 + j;
            const uint32_t dst = sbase + kOffQ + kg * kQLbo + r * 16;
            cp_async16(dst, p.q.hi + qoff + kg * 8, bytes);
            cp_async16(dst + kQPlane, p.q.lo + qoff + kg * 8, bytes);
        }
        if (!img) {
#pragma unroll
            for (int i = 0; i < kKeys / 128; ++i) {
                const int key = key0 + r + 128 * i;
                const size_t koff = (kv_row0 + key) * p.ldk + head * kHeadDim;
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int kg = kg0 + j;
                    const uint32_t dst = sbase + kOffK + kg * kKLbo + key * 16;
                    cp_async16(dst, p.k.hi + koff + kg * 8, 16u);
                    cp_async16(dst + kKPlane, p.k.lo + koff + kg * 8, 16u);
                }
            }
        }
    }
    cp_async_mbar_arrive_noinc(qk_full);

    // ---- stage V^T (already transposed in HBM): piece (key-group kg8, d) = 8 consecutive keys of row d ----
    if (!img) {
        constexpr int kGroups = kKeys / 8;
        const size_t vbase = (size_t)(p.pair0 + pair_local) * p.vt_pair_stride + (size_t)head * kHeadDim * kTokens;
#pragma unroll
        for (int i = 0; i < kGroups * kHeadDim / kThreads; ++i) {
            const int u = t + kThreads * i;
            const int kg8 = key0 / 8 + u % kGroups, d = u / kGroups;
            const uint32_t dst = sbase + kOffV + kg8 * kVLbo + d * 16;
            const size_t voff = vbase + (size_t)d * kTokens + kg8 * 8;
            cp_async16(dst, p.vt.hi + voff, 16u);
            cp_async16(dst + kVLoOff, p.vt.lo + voff, 16u);
        }
        cp_async_mbar_arrive_noinc(v_full);
    }

    // ---- online softmax over 64-key chunks ------------------------------------------------------------------------
    // Fragment of an m64nN accumulator: register 4 j + {0,1} = row (warp % 4) * 16 + lane / 4 ("row a"), columns
    // 8 j + 2 (lane % 4) + {0,1}; registers 4 j + {2,3} = the same columns of row a + 8 ("row b").
    const int wg = warp >> 2;
    const uint32_t q_sub = (uint32_t)wg * 64u * 16u;                 // this warpgroup's 64 rows of the Q tile
    mbar_wait(qk_full, 0);
    if (img) mbar_wait(k_img_full, 0);                   // V is waited for before the first P V
    fence_proxy_async_smem();                            // cp.async (generic proxy) data -> wgmma (async proxy)
    const float kLog2e = 1.4426950408889634f;
    float mx_a = -INFINITY, mx_b = -INFINITY, sum_a = 0.f, sum_b = 0.f;
    float om[2][16], oc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) { om[0][j] = 0.f; om[1][j] = 0.f; oc[j] = 0.f; }
#pragma unroll 1
    for (int c2 = chunk0; c2 < chunk0 + kMyChunks; c2 += 2) {
#pragma unroll
    for (int par = 0; par < 2; ++par) {                  // static parity: om[par] stays in registers
        const int c = c2 + par;
        float sc[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) sc[j] = 0.f;
        fence_regs(sc);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            const uint32_t qa = sbase + kOffQ + q_sub + ks * 2 * kQLbo;
            const uint32_t ka = sbase + kOffK + c * kChunk * 16 + ks * 2 * kKLbo;
            const uint64_t qh = make_smem_desc(qa, kQLbo, kSbo), ql = make_smem_desc(qa + kQPlane, kQLbo, kSbo);
            const uint64_t kh = make_smem_desc(ka, kKLbo, kSbo), kl = make_smem_desc(ka + kKPlane, kKLbo, kSbo);
            wgmma_ss_n64(sc, ql, kh);
            wgmma_ss_n64(sc, qh, kl);
            wgmma_ss_n64(sc, qh, kh);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(sc);
        float cm_a = -INFINITY, cm_b = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            cm_a = fmaxf(cm_a, fmaxf(sc[4 * j], sc[4 * j + 1]));
            cm_b = fmaxf(cm_b, fmaxf(sc[4 * j + 2], sc[4 * j + 3]));
        }
#pragma unroll
        for (int step = 1; step < 4; step <<= 1) {
            cm_a = fmaxf(cm_a, __shfl_xor_sync(0xffffffffu, cm_a, step));
            cm_b = fmaxf(cm_b, __shfl_xor_sync(0xffffffffu, cm_b, step));
        }
        const float nm_a = fmaxf(mx_a, cm_a), nm_b = fmaxf(mx_b, cm_b);
        const float f_a = fast_exp2((mx_a - nm_a) * kLog2e), f_b = fast_exp2((mx_b - nm_b) * kLog2e);   // 0 on the first chunk
        mx_a = nm_a; mx_b = nm_b;
        sum_a *= f_a; sum_b *= f_b;
#pragma unroll
        for (int j = 0; j < 16; j += 4) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                om[0][j + e] *= f_a; om[1][j + e] *= f_a; oc[j + e] *= f_a;
                om[0][j + 2 + e] *= f_b; om[1][j + 2 + e] *= f_b; oc[j + 2 + e] *= f_b;
            }
        }
        const float ms_a = mx_a * kLog2e, ms_b = mx_b * kLog2e;
        uint32_t ph[4][4], pl[4][4];        // A fragments of the 4 k16 steps: P hi / lo planes
#pragma unroll
        for (int kb = 0; kb < 4; ++kb) {
            float v[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = fast_exp2(fmaf(sc[8 * kb + e], kLog2e, (e & 2) ? -ms_b : -ms_a));
            sum_a += (v[0] + v[1]) + (v[4] + v[5]);
            sum_b += (v[2] + v[3]) + (v[6] + v[7]);
#pragma unroll
            for (int r = 0; r < 4; ++r) split_f16x2(v[2 * r], v[2 * r + 1], ph[kb][r], pl[kb][r]);
        }
        if (par == 0 && c2 == chunk0) {
            mbar_wait(v_full, 0);
            fence_proxy_async_smem();
        }
        fence_regs(om[0]); fence_regs(om[1]); fence_regs(oc);
        wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < 4; ++kb) {
            const uint32_t va = sbase + kOffV + (c * (kChunk / 8) + kb * 2) * kVLbo;
            const uint64_t vh = make_smem_desc(va, kVLbo, kSbo), vl = make_smem_desc(va + kVLoOff, kVLbo, kSbo);
            wgmma_rs_n32(oc, pl[kb], vh);
            wgmma_rs_n32(om[par], ph[kb], vh);
            wgmma_rs_n32(oc, ph[kb], vl);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(om[0]); fence_regs(om[1]); fence_regs(oc);
    }
    }
#pragma unroll
    for (int step = 1; step < 4; step <<= 1) {
        sum_a += __shfl_xor_sync(0xffffffffu, sum_a, step);
        sum_b += __shfl_xor_sync(0xffffffffu, sum_b, step);
    }
    float o[16];                                       // this CTA's unnormalised O (the accumulators summed, RN)
#pragma unroll
    for (int j = 0; j < 16; ++j) o[j] = oc[j] + (om[0][j] + om[1][j]);

    // ---- key split: peers push (O, max, sum) to the leader, which rescales to the common row max and adds ----------
    if constexpr (KS > 1) {
        cluster_wait();                                // every CTA of the cluster has initialised its barriers
        if (rank != 0) {
            const uint32_t remote = map_to_cta(sbase + kOffPart + (uint32_t)(rank - 1) * kPartSlot + (uint32_t)t * 16u, 0);
            const uint32_t remote_bar = map_to_cta(smem_u32(part_full), 0);
#pragma unroll
            for (int j = 0; j < 4; ++j)
                st_async_f32x4(remote + j * kPartPiece, o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3], remote_bar);
            st_async_f32x4(remote + 4 * kPartPiece, mx_a, mx_b, sum_a, sum_b, remote_bar);
            return;
        }
        mbar_wait(part_full, 0);                       // (KS - 1) x 20 KB have landed
        const uint8_t* part = smem + kOffPart + t * 16;
        float4 st[KS - 1];
        float m_a = mx_a, m_b = mx_b;
#pragma unroll
        for (int peer = 0; peer < KS - 1; ++peer) {
            st[peer] = *reinterpret_cast<const float4*>(part + peer * kPartSlot + 4 * kPartPiece);
            m_a = fmaxf(m_a, st[peer].x);
            m_b = fmaxf(m_b, st[peer].y);
        }
        {
            const float f_a = fast_exp2((mx_a - m_a) * kLog2e), f_b = fast_exp2((mx_b - m_b) * kLog2e);
            sum_a *= f_a; sum_b *= f_b;
#pragma unroll
            for (int j = 0; j < 16; ++j) o[j] *= (j & 2) ? f_b : f_a;       // registers 4 j + {2,3} belong to row b
        }
#pragma unroll
        for (int peer = 0; peer < KS - 1; ++peer) {
            const float f_a = fast_exp2((st[peer].x - m_a) * kLog2e), f_b = fast_exp2((st[peer].y - m_b) * kLog2e);
            sum_a = fmaf(st[peer].z, f_a, sum_a);
            sum_b = fmaf(st[peer].w, f_b, sum_b);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float4 v = *reinterpret_cast<const float4*>(part + peer * kPartSlot + j * kPartPiece);
                o[4 * j] = fmaf(v.x, f_a, o[4 * j]);
                o[4 * j + 1] = fmaf(v.y, f_a, o[4 * j + 1]);
                o[4 * j + 2] = fmaf(v.z, f_b, o[4 * j + 2]);
                o[4 * j + 3] = fmaf(v.w, f_b, o[4 * j + 3]);
            }
        }
    }

    // ---- O / sum -> global (split16) ----------------------------------------------------------------------------
    {
        const int ra = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const float inv_a = 1.f / sum_a, inv_b = 1.f / sum_b;
#pragma unroll
        for (int h = 0; h < 2; ++h) {                  // row a, row b
            const int qi = ra + 8 * h;
            if (qi >= nrows) continue;
            const float inv = h ? inv_b : inv_a;
            const size_t ooff = ((size_t)qrow0 + qi) * p.ldo + head * kHeadDim + 2 * (lane & 3);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i0 = 4 * j + 2 * h;
                const float x = o[i0] * inv;
                const float y = o[i0 + 1] * inv;
                uint32_t hi, lo;
                split_f16x2(x, y, hi, lo);
                *reinterpret_cast<uint32_t*>(p.out.hi + ooff + 8 * j) = hi;
                *reinterpret_cast<uint32_t*>(p.out.lo + ooff + 8 * j) = lo;
            }
        }
    }
}

template <int KS>
int launch_split(const AttnParams& p, dim3 grid, cudaStream_t s) {
    constexpr size_t smem = kSmemBytes + (size_t)(KS - 1) * kPartSlot;
    static unsigned long long configured = 0;      // bit per device
    if (first_use_on_device(&configured)) {
        COTR_CHECK_CUDA(cudaFuncSetAttribute(attention_tc_kernel<KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    grid.z *= KS;                                  // the KS CTAs of one (tile, head, pair) are neighbours in z: one cluster
    COTR_CHECK_CUDA(launch_kernel_cluster(attention_tc_kernel<KS>, grid, dim3(kThreads), smem, s, KS, p));
    return 0;
}

}  // namespace

// CTAs of one key slice: (tiles, heads, pairs); an empty launch has none
static dim3 tc_grid(const AttnParams& p) {
    if (p.tiles) return dim3(p.n_tiles > 0 ? p.n_tiles : 0, kHeads, 1);
    if (p.nq <= 0 || p.npairs <= 0) return dim3(0, kHeads, 1);
    return dim3((p.nq + kTile - 1) / kTile, kHeads, p.npairs);
}

int launch_attention_tc(const AttnParams& p, cudaStream_t s) {
    // ragged decode (p.tiles): the caller has already sent the pairs with < kAttnTcMinRows rows to the SIMT kernel
    if (!p.tiles && p.nq > 0 && p.npairs > 0 && p.nq < kAttnTcMinRows)
        return launch_attention_simt(p, s);           // a 128-row MMA tile would be > 75% padding
    // Key split over a cluster pair for launches that leave SMs idle (one CTA per SM: shared memory), as long as the
    // doubled grid still fits one wave.  No split by 4: at this shared-memory size an H100 SXM holds only 30 clusters
    // of 4 CTAs at once (cudaOccupancyMaxActiveClusters), so the batch-1 encoder's 32 would take two waves.
    const dim3 grid = tc_grid(p);
    const long long ctas = (long long)grid.x * grid.y * grid.z;
    return launch_attention_tc_split(p, ctas * 2 <= kNumSms ? 2 : 1, s);
}

int launch_attention_tc_split(const AttnParams& p, int ks, cudaStream_t s) {
    const dim3 grid = tc_grid(p);
    if (grid.x == 0) return 0;
    COTR_CHECK(ks == 1 || ks == 2, "attention_tc: key split %d (1 or 2)", ks);
    COTR_CHECK(p.tiles || p.npairs <= 65535, "attention: too many pairs in one launch (%d)", p.npairs);
    COTR_CHECK((p.ldq & 7) == 0 && (p.ldk & 7) == 0 && (p.ldo & 7) == 0 && (p.vt_pair_stride & 7) == 0,
               "attention_tc: leading dimensions must be multiples of 8 elements");
    return ks == 2 ? launch_split<2>(p, grid, s) : launch_split<1>(p, grid, s);
}

}  // namespace cotr
