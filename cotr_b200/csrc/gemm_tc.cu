// wgmma GEMM for sm_90a:  D[M,N] = epilogue( A[M,K] * W[N,K]^T ) on split16 activations (common.cuh).
//
// Precision: the 1e-3 parity bar on predicted (x,y) rules out single-pass bf16 / tf32 / fp16 operands
// (SURVEY.md appendix E.3).  Every operand is a pair of fp16 values (x ~= hi + lo, ~22 mantissa bits) and a product
// is formed as  hi*hi + hi*lo + lo*hi  with fp32 accumulation in registers - three m64 wgmma per k16 step.  Weights
// are pre-multiplied by a per-tensor power of two so that their lo terms stay in fp16's normal range; the epilogue
// multiplies the accumulator by the inverse (exact).  The tensor core adds into its fp32 accumulator with truncation
// (a systematic bias that grows with the number of chained MMAs), so where registers allow the k16 steps are dealt
// round-robin onto several main accumulators, and the small hi*lo / lo*hi products always go to separate correction
// accumulators; the epilogue adds them up with fp32 round-to-nearest.
//
// CTA = 3 warpgroups, one BM x BN output tile, K walked in chunks of 64.  Both operands sit in shared memory in the
// SWIZZLE_128B K-major layout (128-byte rows, 16-byte chunks XOR-swizzled by row % 8):
//   * warpgroups 0-1 (warps 0-7) issue the wgmma: BN <= 128 tiles are 128 x BN, warpgroup g owns rows 64 g ..;
//     the LayerNorm tile (BN = 256) is 64 x 256, warpgroup g owns columns 128 g .. (a 64 x 256 fp32 accumulator pair
//     per warpgroup would not fit the register file);
//   * warpgroup 2 (warps 8-11) stages the A tile with asynchronous 16-byte copies (cp.async -> LDGSTS, zero-filled
//     for im2col padding / row tails; 8 lanes cover one 128-byte row on both sides: coalesced reads, conflict-free
//     writes) whose completion arrives on the stage's mbarrier (cp.async.mbarrier.arrive.noinc).  Activations are
//     already split16 in HBM (the producer's epilogue split them).  The 7x7 stem reads a zero-bordered split16 NHWC4
//     copy of the canvas (common.cuh) with the same copies.  Its thread 0 also issues the weight TMA: weights are
//     pre-split, pre-swizzled in HBM at model creation (tc_pack_weight) as [k chunk][plane][row][128 B], so a stage is
//     two contiguous bulk-TMA copies (cp.async.bulk -> UBLKCP) completing on the SAME mbarrier (128 loader arrivals +
//     1 expect_tx); the first kStages of them are issued before the dependency wait (weights are constants);
//   * long reductions on under-filled grids are split over a thread-block cluster (1 x 1 x {2,4}) and reduce-scattered
//     over 32-row groups through distributed shared memory (st.async + mbarrier, no cluster barrier);
//   * the consumer warpgroups then park their summed accumulators as an fp32 tile in shared memory (the pipeline
//     stages are idle) and all 8 warps run the epilogue from it: warp w owns rows 32 (w % 4).. and the column half
//     w / 4 of the tile (software pipelined: the global operands of chunk c+1 are in flight while chunk c is
//     combined): bias / constant add-matrix / residual / ReLU, or - on warps 0-1 only - the fused residual + LayerNorm
//     over the full 256-wide row (each thread owns one row, so no cross-thread reduction), and write split16
//     (optionally with the value-projection blocks transposed for the attention kernels).
// The kernel is templated on the A-operand addressing mode so that each instantiation carries exactly one loader
// (an all-modes-in-one kernel is large enough to be instruction-cache bound).
#include <cmath>
#include <cstring>
#include <vector>

#include "a_loader.cuh"
#include "tc_common.cuh"

namespace cotr {

int g_tc_variant = 0;                   // bring-up switch (reserved)
int g_use_pdl = 1;                      // programmatic dependent launch (common.cuh); cotr_debug_set_variant bit 8 clears it

namespace {

using namespace tc;

constexpr int BK = 64;
constexpr int kThreads = 384;           // 2 consumer warpgroups + 1 producer warpgroup
constexpr int kConsumerThreads = 256;
constexpr int kBarConsumers = 6;        // named barrier of the 8 consumer warps (1..4: the epilogue's row quarters)
// CTAs of about one wave on the 132 SMs of an H100 SXM (one CTA per SM: the pipeline takes most of shared memory)
constexpr long long kWaveCtas = 144;

enum LoaderMode : int { LD_GATHER = 0, LD_CONV = 1, LD_STEM4 = 2, LD_HALO = 3 };

__host__ __device__ inline int tc_npad(int N) { return N >= 64 ? ((N + 63) / 64) * 64 : ((N + 15) / 16) * 16; }

// Halo loader (LD_HALO) of the 3x3 stride-1 convolutions.  The implicit im2col stages a 128 x 64 A tile per (tap,
// 64-channel) chunk, i.e. every input pixel nine times.  Instead, the output rows of an image are numbered over the
// zero-padded (H+2) x (W+2) grid, m = oh (W+2) + ow with ow in [0, W+2) (rows with ow >= W, and those past the last
// output row, are computed and dropped by the epilogue; tiles never cross images), so that tap (kh, kw) of output row m
// is padded input position m + kh (W+2) + kw.  A tile of 128 rows starting at q0 then needs the padded positions
// [q0, q0 + 128 + 2 (W+2) + 2) of each 64-channel chunk: the producer stages them ONCE (zero-filled outside the image,
// SWIZZLE_128B keyed by the absolute halo row) and they stay resident; tap (kh, kw) is the view of that tile at row
// offset kh (W+2) + kw: a plain make_desc_sw128 of the view's address, base-offset field 0 (the unit applies the
// 128-byte swizzle to the absolute shared-memory address bits, so a view that starts at any row keeps the tile's
// phase; checked on H100 for row offsets 0..23, whereas base offset (addr >> 7) & 7 is wrong).  Only the weights
// stream through the pipeline stages.  The K order is the implicit im2col's (tap-major, channel-minor); split-K
// hands each CTA of the cluster whole channel chunks.
constexpr uint32_t kHaloMaxBytes = 100u * 1024u;        // resident halo tiles of one CTA (both planes, all its chunks)
constexpr int kHaloMaxChunks = 4;
constexpr long long kHaloMinCtas = 86;                  // two thirds of the 132 SMs (see halo_fits)
__host__ __device__ inline int halo_pitch(const GemmParams& p) { return p.W + 2; }
__host__ __device__ inline int halo_tiles_per_img(const GemmParams& p) { return (p.OH * halo_pitch(p) + 127) / 128; }
__host__ __device__ inline int halo_rows(const GemmParams& p) { return 128 + 2 * halo_pitch(p) + 2; }
__host__ __device__ inline uint32_t halo_plane_bytes(const GemmParams& p) { return (uint32_t)((halo_rows(p) + 7) / 8 * 8) * 128u; }
// dense NHWC output row of padded-grid row m, or -1 for the rows the halo grid adds
__device__ __forceinline__ int halo_out_row(const GemmParams& p, int m) {
    const int tpi = halo_tiles_per_img(p), pitch = halo_pitch(p);
    const int tile = m >> 7, n = tile / tpi;
    const int local = (tile - n * tpi) * 128 + (m & 127);
    const int oh = local / pitch, ow = local - oh * pitch;
    return (oh < p.OH && ow < p.OW) ? (n * p.OH + oh) * p.OW + ow : -1;
}

template <int BN, int MODE = LD_GATHER>
struct Cfg {
    static constexpr int BM = BN >= 256 ? 64 : 128;
    static constexpr int WN = BN >= 256 ? 128 : BN;                     // columns of one consumer warpgroup's wgmma
    static constexpr uint32_t kAPlane = BM * 128u;                      // one fp16 plane (hi or lo) of the BM x 64 A tile
    static constexpr uint32_t kBPlane = BN * 128u;                      // BN rows x 128 bytes
    // LD_HALO: the A halo tiles sit in their own region in front of the stages, which then carry the weights only
    static constexpr uint32_t kHaloBytes = MODE == LD_HALO ? kHaloMaxBytes : 0u;
    static constexpr uint32_t kAStage = MODE == LD_HALO ? 0u : 2 * kAPlane;
    static constexpr uint32_t kStage = kAStage + 2 * kBPlane;
    static constexpr int kStagesRaw = (int)((227u * 1024u - 3072u - kHaloBytes) / kStage);
    static constexpr int kStages = kStagesRaw > 4 ? 4 : kStagesRaw;
    // register accumulators of one warpgroup (WN / 2 floats per thread each): kMain slots take the hi*hi products
    // round-robin over the k16 steps, kCorr slots the lo*hi / hi*lo products
    static constexpr int kMain = WN >= 128 ? 1 : (WN == 64 ? 2 : 4);
    static constexpr int kCorr = WN >= 64 ? 1 : 2;
    static constexpr int kAccRegs = WN / 2;
    // fp32 accumulator tile in shared memory for the epilogue (re-uses the pipeline stages): BM rows, padded pitch
    static constexpr uint32_t kAccPitch = BN * 4u + 16u;
    static constexpr uint32_t kAccTileBytes = ((BM * kAccPitch + 1023u) / 1024u) * 1024u;
    // epilogue output staging (behind the accumulator tile): per row quarter 2 planes x 32 rows, pitch padded by 16 B
    static constexpr uint32_t kOutPitch = BN * 2u + 16u;
    static constexpr uint32_t kWarpStaging = 2u * 32u * kOutPitch;
    static constexpr int kChunksN = BN / 16;
    // Epilogue warps: the row quarters x kEpiHalves column halves (warp w: rows 32 (w % 4) ..., columns
    // [w / 4 * BN / 2, ...)).  The LayerNorm tile (BN = 256) keeps one thread per full row.
    static constexpr int kEpiHalves = (BN >= 32 && BN < 256) ? 2 : 1;
    static constexpr int kChunksW = kChunksN / kEpiHalves;             // 16-column chunks per epilogue warp
    // epilogue operand prefetch depth (2 x 48 registers: a 384-thread CTA leaves 168 registers per thread)
    static constexpr int kRing = kChunksW < 2 ? kChunksW : 2;
    // behind the stages: 256 bytes of barriers, then the per-column vectors of the deferred LayerNorm (column sums of
    // W' or gamma | beta of this tile's BN columns, staged by two producer warps while the main loop runs), then split-K partials
    static constexpr uint32_t kVecOffset = kStages * kStage + 256;       // (offsets behind the halo region)
    static constexpr uint32_t kVecBytes = 2u * BN * 4u + 2u * BM * 8u;   // + (mean, rstd) of the BM A rows and of the BM residual rows
    static constexpr uint32_t kSmemBytes = kHaloBytes + kStages * kStage + 2048 + kVecBytes;     // + alignment slack + barriers + vectors
    // split-K (reduce-scatter over the rows): every CTA of the cluster finishes 128 / ksplit rows of the tile and
    // receives the other CTAs' fp32 partial rows behind the barriers (a dedicated region, so peers may push while this
    // CTA's pipeline is still running); rows of BN * 4 bytes, 16-byte pieces XOR-swizzled by row % 8 (thread-per-row
    // accesses would otherwise all land in the same banks)
    static constexpr uint32_t kPartOffset = kVecOffset + kVecBytes;
    static constexpr uint32_t kPartPitch = BN * 4u;
    static constexpr int kMaxSplit = BN <= 64 ? 4 : 1;
    static constexpr uint32_t kPartMaxBytes = kMaxSplit > 1 ? 96u * kPartPitch : 0u;   // ksplit 4: 3 x 32 rows; 2: 1 x 64 rows
    static_assert(kSmemBytes + kPartMaxBytes <= 227u * 1024u, "split-K partial tiles do not fit");
    static_assert(kStages >= 2, "pipeline needs at least two stages");
    static_assert(kAccTileBytes + (BM / 32) * kWarpStaging <= kHaloBytes + kStages * kStage, "epilogue tiles do not fit the idle stages");
    static_assert(kStage % 1024 == 0 && kAPlane % 1024 == 0 && kHaloBytes % 1024 == 0, "stages must stay 1024-byte aligned for SWIZZLE_128B");
    static_assert(kMaxSplit == 1 || BM == 128, "split-K hands over 32-row groups of a 128-row tile");
};

// global operands of one 16-column epilogue chunk, fetched one chunk ahead of their use
struct EpiOperands {
    float4 bias[4];
    float4 add[4];
    uint4 res_hi[2], res_lo[2];
};

// DLN: the instantiation carries the deferred-LayerNorm operands (GemmParams::a_ln_cs / res_ln_part / ln_part_out).
// The default schedule uses DLN = false kernels, which contain none of it.
template <int BN, bool LN, int MODE, bool DLN>
__global__ void __launch_bounds__(kThreads, 1) gemm_tc_kernel(const GemmParams p, const int npad) {
    using C = Cfg<BN, MODE>;
    constexpr int BM = C::BM;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw_addr = smem_u32(smem_raw);
    uint8_t* tile_mem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);        // SWIZZLE_128B needs 1024-byte alignment
    uint8_t* stage_base = tile_mem + C::kHaloBytes;                                     // LD_HALO: behind the resident halo tiles
    uint64_t* bars = reinterpret_cast<uint64_t*>(stage_base + C::kStages * C::kStage);
    uint64_t* full_a = bars;
    uint64_t* empty = bars + C::kStages;
    uint64_t* part_full = bars + 2 * C::kStages;           // split-K leader: all peers' partial tiles have landed
    uint64_t* vec_full = bars + 2 * C::kStages + 1;        // deferred LayerNorm: the per-column vectors are staged
    uint64_t* halo_full = bars + 2 * C::kStages + 2;       // LD_HALO: halo tile c of this CTA has landed
    float* vec_a = reinterpret_cast<float*>(stage_base + C::kVecOffset);      // a_ln: column sums of W'; res_ln: gamma
    float* vec_b = vec_a + BN;                                                  //                         res_ln: beta
    float2* st_a = reinterpret_cast<float2*>(vec_b + BN);                       // (mean, rstd) of the A rows of this tile
    float2* st_r = st_a + BM;                                                   // (mean, rstd) of the residual rows
    float* acc_tile = reinterpret_cast<float*>(tile_mem);                       // epilogue: summed accumulators [BM][kAccPitch]
    // deferred LayerNorm (GemmParams::a_ln_cs / res_ln_part / ln_part_out): only the row-major loader instantiations carry it
    static_assert(!DLN || (MODE == LD_GATHER && !LN), "deferred LayerNorm: row-major operand tiles only");
    constexpr bool kCanLnA = DLN;
    const bool has_aln = kCanLnA && p.a_ln_cs != nullptr;
    const bool stage_vec = kCanLnA && !LN && (has_aln || p.res_ln_part != nullptr);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    // split-K: gridDim.z CTAs of one cluster (cluster dims 1 x 1 x gridDim.z) share the output tile; CTA z walks the
    // K chunks [it0, it0 + KC) and then finishes the 32-row groups it owns: the other CTAs hand it their partial sums of
    // those rows through distributed shared memory - asynchronous remote stores (st.async) that complete transaction
    // bytes on an mbarrier of the owner, so the hand-over needs no cluster-wide barrier and each CTA receives only
    // (ksplit-1)/ksplit of a tile.
    const int ksplit = gridDim.z;
    const int kz = blockIdx.z;
    const int KC = ((p.K + BK - 1) / BK) / ksplit;
    const int it0 = kz * KC;
    // LD_HALO: this CTA's channel chunks [kz ccp, (kz+1) ccp) of cc; iteration it = tap * ccp + chunk
    const int cc = p.C / BK, ccp = cc / ksplit;
    const uint32_t halo_plane = MODE == LD_HALO ? halo_plane_bytes(p) : 0u;
    // weight image chunk of iteration it (k = tap * C + channel)
    auto w_chunk = [&](int it) {
        if constexpr (MODE == LD_HALO) {
            const int tap = it / ccp;
            return tap * cc + kz * ccp + (it - tap * ccp);
        }
        return it0 + it;
    };

    if (threadIdx.x == 0) {
        for (int s = 0; s < C::kStages; ++s) {
            mbar_init(&full_a[s], MODE == LD_HALO ? 1 : 129);      // (128 loader arrivals) + 1 expect_tx
            mbar_init(&empty[s], 8);          // one arrival per consumer warp
        }
        if (MODE == LD_HALO)
            for (int c = 0; c < ccp; ++c) mbar_init(&halo_full[c], 128);
        mbar_init(part_full, 1);
        if (DLN) mbar_init(vec_full, 64);
        mbar_fence_init();
        if (ksplit > 1) mbar_arrive_expect_tx(part_full, (uint32_t)(ksplit - 1) * (uint32_t)(BM / ksplit) * C::kPartPitch);
    }
    __syncthreads();
    // split-K: tell the cluster that this CTA runs and its barriers exist (waited for just before the first remote access)
    if (ksplit > 1) cluster_arrive();

    if (warp >= 8) {
        // ================= producer warpgroup: A tile by cp.async, weights by bulk TMA ============================
        const int t = threadIdx.x - kConsumerThreads;
        const int kg = t & 7;          // 16-byte K group (8 halves) inside the 64-wide chunk
        const int rb = t >> 3;         // rows rb, rb+16, ...  (row % 8 == rb % 8 for all of them)
        constexpr int kRowIters = BM / 16;
        const uint8_t* wimg = reinterpret_cast<const uint8_t*>(p.Wtc);
        // image: [k chunk][plane][npad rows][128 bytes]; the BN rows of this tile are contiguous per plane
        auto load_weights = [&](int it) {
            const int s = it % C::kStages;
            mbar_arrive_expect_tx(&full_a[s], 2u * C::kBPlane);
            uint8_t* b_dst = stage_base + (size_t)s * C::kStage + C::kAStage;
            const uint8_t* src = wimg + (((size_t)w_chunk(it) * 2) * npad + n0) * 128;
            tma_bulk_g2s(b_dst, src, C::kBPlane, &full_a[s]);
            tma_bulk_g2s(b_dst + C::kBPlane, src + (size_t)npad * 128, C::kBPlane, &full_a[s]);
        };
        // the constant per-column vectors of the deferred LayerNorm (model constants: loaded before the dependency wait)
        const int u = (warp - 10) * 32 + lane;
        const float* src_a = has_aln ? p.a_ln_cs : p.res_ln_gamma;
        float va[(BN + 63) / 64], vb[(BN + 63) / 64];
        if (stage_vec && warp >= 10) {
#pragma unroll
            for (int k = 0; k < (BN + 63) / 64; ++k) {
                const int i = u + 64 * k;
                const bool ok = i < BN && n0 + i < p.N;
                va[k] = ok ? __ldg(src_a + n0 + i) : 0.f;
                vb[k] = (ok && !has_aln) ? __ldg(p.res_ln_beta + n0 + i) : 0.f;
            }
        }
        ARow rows[kRowIters];
        if constexpr (MODE != LD_HALO) {
#pragma unroll
            for (int i = 0; i < kRowIters; ++i) rows[i] = decode_a_row(p, m0 + rb + 16 * i);
        }
        const uint32_t a_off = (uint32_t)rb * 128u + (uint32_t)((kg ^ (rb & 7)) << 4);   // swizzled chunk position
        const uint32_t dst0 = smem_u32(stage_base) + a_off;
        // Weights are constants: the first stages' copies overlap the previous kernel.  Then let the next kernel of the
        // stream / graph start its prologue on idle SMs; it still waits (griddepcontrol.wait) for this grid to complete
        // before touching activations.
        if (t == 0) {
            for (int it = 0; it < KC && it < C::kStages; ++it) load_weights(it);
            pdl_launch_dependents();
        }
        pdl_wait();

        if constexpr (MODE == LD_HALO) {
            // the halo tiles of this CTA's channel chunks, once: halo row j = padded input position q0 + j of image n
            const int pitch = halo_pitch(p), tpi = halo_tiles_per_img(p), hrows = halo_rows(p);
            const int n = blockIdx.x / tpi, q0 = (blockIdx.x - n * tpi) * 128;
            const size_t img = (size_t)n * p.H * p.W * p.C;
            for (int c = 0; c < ccp; ++c) {
                const int ch = (kz * ccp + c) * BK + kg * 8;
                const uint32_t dst = smem_u32(tile_mem) + (uint32_t)c * 2u * halo_plane;
#pragma unroll 4
                for (int j = rb; j < hrows; j += 16) {
                    const int q = q0 + j;
                    const int ih = q / pitch - 1, iw = q - (ih + 1) * pitch - 1;
                    const bool ok = ih >= 0 && ih < p.H && iw >= 0 && iw < p.W;
                    const size_t off = ok ? img + ((size_t)ih * p.W + iw) * p.C + ch : 0;
                    const uint32_t d = dst + (uint32_t)j * 128u + (uint32_t)((kg ^ (j & 7)) << 4);
                    cp_async16(d, p.a.hi + off, ok ? 16u : 0u);
                    cp_async16(d + halo_plane, p.a.lo + off, ok ? 16u : 0u);
                }
                cp_async_mbar_arrive_noinc(&halo_full[c]);
            }
        }

#pragma unroll 1
        for (int it = 0; it < KC; ++it) {
            // (every producer thread walks the loop, so that the warps reach the final __syncthreads converged)
            const int s = it % C::kStages;
            const uint32_t ph = (uint32_t)(it / C::kStages) & 1u;
            mbar_wait(&empty[s], ph ^ 1u);
            if (t == 0 && it >= C::kStages) load_weights(it);
            if constexpr (MODE == LD_HALO) continue;             // the stages carry weights only
            const int k0 = (it0 + it) * BK;
            {
                const uint32_t dst = dst0 + (uint32_t)s * C::kStage;
                int kh = 0, kw = 0, koff = k0 + kg * 8;          // LD_GATHER: koff = column inside the row
                if constexpr (MODE == LD_CONV) {                 // C % 64 == 0: the chunk lies inside one filter tap
                    const int tap = k0 / p.C;
                    koff = k0 - tap * p.C + kg * 8;
                    kh = tap / p.KW;
                    kw = tap - kh * p.KW;
                }
                if constexpr (MODE == LD_STEM4) {               // filter row kh = 64 contiguous bytes of the bordered canvas
                    const int kk = k0 + kg * 8;
                    koff = (kk >> 5) * (kStemCanvasPitch * 4) + (kk & 31);
                }
                const bool k_ok = (k0 + kg * 8) < p.K;
#pragma unroll
                for (int i = 0; i < kRowIters; ++i) {
                    bool ok = rows[i].valid && k_ok;
                    size_t off = rows[i].off + koff;
                    if constexpr (MODE == LD_CONV) {
                        const int ih = rows[i].ih0 + kh, iw = rows[i].iw0 + kw;
                        ok = ok && ih >= 0 && ih < p.H && iw >= 0 && iw < p.W;
                        off = rows[i].off + ((size_t)ih * p.W + iw) * p.C + koff;
                    }
                    if (!ok) off = 0;                            // src-size 0 -> 16 bytes of zeros, address unused
                    const uint32_t bytes = ok ? 16u : 0u;
                    cp_async16(dst + i * 2048, p.a.hi + off, bytes);                  // 16 rows x 128 bytes further down
                    cp_async16(dst + C::kAPlane + i * 2048, p.a.lo + off, bytes);
                }
                cp_async_mbar_arrive_noinc(&full_a[s]);
            }
        }

        if (stage_vec && warp >= 10) {
            // ================= warps 10-11: operands of the deferred LayerNorm ====================================
            // (mean, rstd) of the 128 rows of this tile from the 16 partial statistics per row their producer's epilogue
            // left behind ((mean, M2) per 16-column chunk, GemmParams::ln_part_out).  8 lanes read one row's 128-byte line
            // (coalesced: 4 rows per instruction, all 16 loads of a lane in flight before the first use) and add up
            //     S1 = sum mean_i,  S2 = sum mean_i^2,  S3 = sum M2_i     (3 butterfly steps)
            // -> mean = S1 / 16,  M2 = S3 + 16 (S2 - S1^2 / 16)  (the chunk means are of the row's own magnitude, so the
            // difference is benign).  ld.global.cg, never .nc: the producer may still have been running when this CTA
            // became resident (see load8_split).
            auto stage_stats = [&](const float2* part, float2* dst) {
                const int sub = lane & 7;                      // which 16 bytes (2 partials) of the row's line
                float4 ld[16];
#pragma unroll
                for (int it = 0; it < 16; ++it) {
                    const int grow = m0 + (warp - 10) * 64 + it * 4 + (lane >> 3);
                    ld[it] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (grow < p.M) ld[it] = __ldcg(reinterpret_cast<const float4*>(part + (size_t)grow * 16) + sub);
                }
#pragma unroll
                for (int it = 0; it < 16; ++it) {
                    const float4 t4 = ld[it];
                    // chunk means relative to the row's first chunk mean: the sums below then do not cancel
                    const float ref = __shfl_sync(0xffffffffu, t4.x, lane & ~7);
                    const float d0 = t4.x - ref, d1 = t4.z - ref;
                    float s1 = d0 + d1;
                    float s2 = fmaf(d0, d0, d1 * d1);
                    float s3 = t4.y + t4.w;
#pragma unroll
                    for (int step = 1; step < 8; step <<= 1) {
                        s1 += __shfl_xor_sync(0xffffffffu, s1, step);
                        s2 += __shfl_xor_sync(0xffffffffu, s2, step);
                        s3 += __shfl_xor_sync(0xffffffffu, s3, step);
                    }
                    const float mean = fmaf(s1, 1.f / 16.f, ref);
                    const float m2 = s3 + fmaxf(fmaf(16.f, s2, -s1 * s1), 0.f);          // sum M2_i + 16 sum (mean_i - mean)^2
                    if (sub == 0) dst[(warp - 10) * 64 + it * 4 + (lane >> 3)] = make_float2(mean, rsqrtf(m2 * (1.f / 256.f) + 1e-5f));
                }
            };
            for (int k = 0; k < (BN + 63) / 64; ++k) {
                const int i = u + 64 * k;
                if (i < BN) { vec_a[i] = va[k]; vec_b[i] = vb[k]; }
            }
            if (has_aln) stage_stats(p.a_ln_part, st_a);
            if (p.res_ln_part != nullptr) stage_stats(p.res_ln_part, st_r);
            mbar_arrive(vec_full);
        }
    } else {
        // ================= consumer warpgroups: wgmma main loop ===================================================
        const int wg = warp >> 2;
        const uint32_t a_sub = BN >= 256 ? 0u : (uint32_t)wg * 64u * 128u;              // this warpgroup's 64 rows
        const uint32_t b_sub = BN >= 256 ? (uint32_t)wg * 128u * 128u : 0u;             // ... or its 128 columns
        float acc_m[C::kMain][C::kAccRegs], acc_c[C::kCorr][C::kAccRegs];
#pragma unroll
        for (int a = 0; a < C::kMain; ++a)
#pragma unroll
            for (int j = 0; j < C::kAccRegs; ++j) acc_m[a][j] = 0.f;
#pragma unroll
        for (int a = 0; a < C::kCorr; ++a)
#pragma unroll
            for (int j = 0; j < C::kAccRegs; ++j) acc_c[a][j] = 0.f;
        auto mma = [&](float (&d)[C::kAccRegs], uint64_t da, uint64_t db) {
            if constexpr (C::WN == 16) wgmma_ss_n16(d, da, db);
            else if constexpr (C::WN == 32) wgmma_ss_n32(d, da, db);
            else if constexpr (C::WN == 64) wgmma_ss_n64(d, da, db);
            else wgmma_ss_n128(d, da, db);
        };
        auto fence_all = [&]() {
#pragma unroll
            for (int a = 0; a < C::kMain; ++a) fence_regs(acc_m[a]);
#pragma unroll
            for (int a = 0; a < C::kCorr; ++a) fence_regs(acc_c[a]);
        };
#pragma unroll 1
        for (int it = 0; it < KC; ++it) {
            const int s = it % C::kStages;
            const uint32_t ph = (uint32_t)(it / C::kStages) & 1u;
            uint32_t a_addr = smem_u32(stage_base + (size_t)s * C::kStage);
            uint32_t a_plane = C::kAPlane;
            if constexpr (MODE == LD_HALO) {                   // tap (kh, kw) = the halo tile seen kh (W+2) + kw rows further down
                const int tap = it / ccp, c = it - tap * ccp, kh = tap / 3;
                mbar_wait(&halo_full[c], 0);
                a_plane = halo_plane;
                a_addr = smem_u32(tile_mem) + (uint32_t)c * 2u * halo_plane + (uint32_t)(kh * halo_pitch(p) + tap - 3 * kh) * 128u;
            }
            mbar_wait(&full_a[s], ph);
            fence_proxy_async_smem();                          // cp.async (generic proxy) data -> wgmma (async proxy)
            const uint32_t b_addr = smem_u32(stage_base + (size_t)s * C::kStage) + C::kAStage;
            fence_all();
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < BK / 16; ++ks) {
                // a k16 step = 32 bytes inside the 128-byte swizzle atom
                const uint64_t dah = make_desc_sw128(a_addr + a_sub + 32 * ks);
                const uint64_t dal = make_desc_sw128(a_addr + a_plane + a_sub + 32 * ks);
                const uint64_t dbh = make_desc_sw128(b_addr + b_sub + 32 * ks);
                const uint64_t dbl = make_desc_sw128(b_addr + C::kBPlane + b_sub + 32 * ks);
                mma(acc_c[0], dal, dbh);
                mma(acc_m[ks % C::kMain], dah, dbh);           // (it * 4) % kMain == 0: the slot is static
                mma(acc_c[C::kCorr - 1], dah, dbl);
            }
            wgmma_commit();
            wgmma_wait<1>();                                   // the previous chunk's MMAs have read their stage
            fence_all();
            if (it > 0 && lane == 0) mbar_arrive(&empty[(it - 1) % C::kStages]);
        }
        wgmma_wait<0>();
        fence_all();
        // park the sums (corrections first, then the main slots, RN adds) as an fp32 tile once both warpgroups are done
        // with the stages.  Fragment of m64nWN: register 4 j + {0,1} = row (warp % 4) * 16 + lane / 4, columns
        // 8 j + 2 (lane % 4) + {0,1}; registers 4 j + {2,3} = the same columns 8 rows further down.
        named_barrier_sync(kBarConsumers, kConsumerThreads);
        const int r0 = (BN >= 256 ? 0 : wg * 64) + (warp & 3) * 16 + (lane >> 2);
        const int c0 = (BN >= 256 ? wg * 128 : 0) + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < C::kAccRegs; j += 2) {
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                float x = acc_c[0][j + e];
#pragma unroll
                for (int a = 1; a < C::kCorr; ++a) x += acc_c[a][j + e];
                float y = acc_m[0][j + e];
#pragma unroll
                for (int a = 1; a < C::kMain; ++a) y += acc_m[a][j + e];
                v[e] = x + y;
            }
            const int row = r0 + ((j >> 1) & 1) * 8;
            const int col = c0 + (j >> 2) * 8;
            *reinterpret_cast<float2*>(reinterpret_cast<uint8_t*>(acc_tile) + (uint32_t)row * C::kAccPitch + col * 4) = make_float2(v[0], v[1]);
        }
        named_barrier_sync(kBarConsumers, kConsumerThreads);
    }

    // ================= epilogue: accumulator tile -> registers -> global ==========================================
    const int ew = warp & 3;                 // 32-row group of the tile this warp handles
    const int half = warp >> 2;              // column half of the tile it handles
    if (ksplit > 1) cluster_wait();          // every CTA of the cluster has started (long ago by now)
    if (warp < 8 && half < C::kEpiHalves && ew * 32 < BM) {
        pdl_wait();                          // residual / add operands come from the previous kernels
        const int cbeg = half * C::kChunksW * 16;
        const int row = m0 + ew * 32 + lane;
        // split-K: row group q is finished by CTA q * ksplit / 4; the other CTAs only contribute partial sums
        const int owner = (ew * ksplit) >> 2;
        const bool mine = owner == kz;
        const bool row_ok = mine && row < p.M;
        uint8_t* arow = reinterpret_cast<uint8_t*>(acc_tile) + (uint32_t)(ew * 32 + lane) * C::kAccPitch;
        const float* add_row = (row_ok && p.addmat) ? p.addmat + (size_t)(row % p.add_period) * p.ld_add : nullptr;
        const bool has_res = row_ok && p.res.hi != nullptr;
        const size_t res_off = (size_t)(row_ok ? row : 0) * p.ldr;
        const float acc_scale = p.acc_scale;
        // Deferred LayerNorm: (mean, rstd) of this thread's A row / residual row, staged by warps 10-11
        const bool res_ln = kCanLnA && has_res && p.res_ln_part != nullptr;
        float2 res_st = make_float2(0.f, 1.f);
        float res_shift = 0.f;                          // -mean * rstd of the residual row
        float2 a_st = make_float2(0.f, 1.f);
        const bool emit_part = kCanLnA && row_ok && p.ln_part_out != nullptr;
        const bool tail = p.out_f32 != nullptr && (p.N & 15) != 0;      // only the N = 2 prediction head
        const bool has_bias = p.bias != nullptr && !tail;

        // issue the global loads of the chunk starting at column nb (bias / add-matrix / residual); N % 16 == 0 here
        auto prefetch = [&](int nb, EpiOperands& o) {
            if (nb >= p.N || tail) return;
            if (has_bias) {
#pragma unroll
                for (int j = 0; j < 4; ++j) o.bias[j] = __ldg(reinterpret_cast<const float4*>(p.bias + nb) + j);
            }
            if (add_row) {
#pragma unroll
                for (int j = 0; j < 4; ++j) o.add[j] = __ldg(reinterpret_cast<const float4*>(add_row + nb) + j);
            }
            if (has_res) {
                // 16 halves of one plane = one 32-byte sector (activations bypass L1, see load8_split)
                ld_cg_32b(p.res.hi + res_off + nb, o.res_hi[0], o.res_hi[1]);
                ld_cg_32b(p.res.lo + res_off + nb, o.res_lo[0], o.res_lo[1]);
            }
        };
        auto apply = [&](const EpiOperands& o, float (&v)[16], int nb) {
            const int cl = nb - n0;                   // column inside the tile (the staged vectors are tile-local)
            if (kCanLnA && has_aln) {                 // y = rstd * (x W'^T - mean * colsum(W'))
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float4 cs4 = *reinterpret_cast<const float4*>(vec_a + cl + 4 * j);
                    v[4 * j] = a_st.y * fmaf(-a_st.x, cs4.x, v[4 * j]);
                    v[4 * j + 1] = a_st.y * fmaf(-a_st.x, cs4.y, v[4 * j + 1]);
                    v[4 * j + 2] = a_st.y * fmaf(-a_st.x, cs4.z, v[4 * j + 2]);
                    v[4 * j + 3] = a_st.y * fmaf(-a_st.x, cs4.w, v[4 * j + 3]);
                }
            }
            if (has_bias) {
#pragma unroll
                for (int j = 0; j < 4; ++j) { v[4 * j] += o.bias[j].x; v[4 * j + 1] += o.bias[j].y; v[4 * j + 2] += o.bias[j].z; v[4 * j + 3] += o.bias[j].w; }
            }
            if (add_row) {
#pragma unroll
                for (int j = 0; j < 4; ++j) { v[4 * j] += o.add[j].x; v[4 * j + 1] += o.add[j].y; v[4 * j + 2] += o.add[j].z; v[4 * j + 3] += o.add[j].w; }
            }
            if (has_res) {
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const uint32_t h[4] = {o.res_hi[j].x, o.res_hi[j].y, o.res_hi[j].z, o.res_hi[j].w};
                    const uint32_t l[4] = {o.res_lo[j].x, o.res_lo[j].y, o.res_lo[j].z, o.res_lo[j].w};
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        float2 f = join_f16x2(h[q], l[q]);
                        if (kCanLnA && res_ln) {      // the residual is a deferred LayerNorm of the stored rows
                            const float2 g2 = *reinterpret_cast<const float2*>(vec_a + cl + 8 * j + 2 * q);
                            const float2 b2 = *reinterpret_cast<const float2*>(vec_b + cl + 8 * j + 2 * q);
                            f.x = fmaf(fmaf(f.x, res_st.y, res_shift), g2.x, b2.x);
                            f.y = fmaf(fmaf(f.y, res_st.y, res_shift), g2.y, b2.y);
                        }
                        v[8 * j + 2 * q] += f.x;
                        v[8 * j + 2 * q + 1] += f.y;
                    }
                }
            }
        };
        constexpr uint32_t kPartPitch = C::kPartPitch, kPartOffset = C::kPartOffset;
        const uint32_t part_slot = (uint32_t)(BM / ksplit) * kPartPitch;       // one source CTA's rows in the owner's region
        const uint32_t part_row = (uint32_t)((ew - owner * (4 / ksplit)) * 32 + lane) * kPartPitch;   // row inside a slot
        const uint32_t part_swz = (uint32_t)(lane & 7);                        // == row % 8
        // v = this CTA's (unscaled) sums of columns [c, c+16) of its row
        auto sum_acc = [&](int c, float (&v)[16]) {
#pragma unroll
            for (int j = 0; j < 16; j += 4) {
                const float4 t4 = *reinterpret_cast<const float4*>(arow + (c + j) * 4);
                v[j] = t4.x; v[j + 1] = t4.y; v[j + 2] = t4.z; v[j + 3] = t4.w;
            }
        };
        // own sums -> final accumulator: add the peers' partial rows (split-K owner), undo the weight pre-scaling
        auto finish_acc = [&](int c, float (&v)[16]) {
            if (ksplit > 1) {                             // owner: add the partial sums the peers pushed over DSMEM
                const uint8_t* part = stage_base + kPartOffset + part_row;
                for (int peer = 0; peer < ksplit - 1; ++peer) {
#pragma unroll
                    for (int j = 0; j < 16; j += 4) {
                        const uint32_t piece = ((uint32_t)((c + j) >> 2) ^ part_swz) << 4;
                        const float4 t4 = *reinterpret_cast<const float4*>(part + (uint32_t)peer * part_slot + piece);
                        v[j] += t4.x; v[j + 1] += t4.y; v[j + 2] += t4.z; v[j + 3] += t4.w;
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] *= acc_scale;
        };
        auto load_acc = [&](int c, float (&v)[16]) {
            sum_acc(c, v);
            finish_acc(c, v);
        };

        // Output path.  split16 row-major tiles are staged in shared memory (the pipeline stages are idle once the
        // accumulator is complete) and written out as full coalesced rows; a thread-per-row direct store would touch
        // 32 different cache lines per instruction.  The two warps of a lane quarter stage their column halves into the
        // same 32-row region, meet on a named barrier and drain one fp16 plane each.  Transposed value blocks and the
        // fp32 prediction head keep the direct path.
        size_t tile_base = 0;
        const bool direct = p.out_f32 != nullptr || out_location(p, m0, n0, tile_base);
        uint8_t* const stg_base = tile_mem + C::kAccTileBytes;            // behind the accumulator tile
        uint8_t* stg = stg_base + (uint32_t)ew * C::kWarpStaging + (uint32_t)lane * C::kOutPitch;
        auto emit16 = [&](int c, const float (&v)[16]) {          // c = column inside the tile
            if (direct) {
                if (row_ok && n0 + c < p.N) store16(p, row, n0 + c, v);
                return;
            }
            uint4 h0, l0, h1, l1;
            split_f16x2(v[0], v[1], h0.x, l0.x);   split_f16x2(v[2], v[3], h0.y, l0.y);
            split_f16x2(v[4], v[5], h0.z, l0.z);   split_f16x2(v[6], v[7], h0.w, l0.w);
            split_f16x2(v[8], v[9], h1.x, l1.x);   split_f16x2(v[10], v[11], h1.y, l1.y);
            split_f16x2(v[12], v[13], h1.z, l1.z); split_f16x2(v[14], v[15], h1.w, l1.w);
            uint8_t* d = stg + c * 2;
            *reinterpret_cast<uint4*>(d) = h0;
            *reinterpret_cast<uint4*>(d + 16) = h1;
            *reinterpret_cast<uint4*>(d + 32 * C::kOutPitch) = l0;
            *reinterpret_cast<uint4*>(d + 32 * C::kOutPitch + 16) = l1;
        };
        auto drain_plane = [&](int plane) {
            constexpr int kLanesPerRow = BN * 2 / 16;                     // 16-byte pieces per row of one plane
            constexpr int kRowsPerPass = kLanesPerRow >= 32 ? 1 : 32 / kLanesPerRow;
            constexpr int kPiecesPerLane = kLanesPerRow > 32 ? kLanesPerRow / 32 : 1;
            const uint8_t* wbase = stg_base + (uint32_t)ew * C::kWarpStaging;
            const int r_in = kLanesPerRow >= 32 ? 0 : lane / kLanesPerRow;
            const int piece0 = kLanesPerRow >= 32 ? lane : lane % kLanesPerRow;
            __half* gout = plane == 0 ? p.out.hi : p.out.lo;
#pragma unroll 4
            for (int r0 = 0; r0 < 32; r0 += kRowsPerPass) {
                const int rr = r0 + r_in;
                const int grow_ = m0 + ew * 32 + rr;
                bool ok = grow_ < p.M;
                size_t roff = tile_base + (size_t)(ew * 32 + rr) * p.ldc;          // element (row, n0 mapped)
                if constexpr (MODE == LD_HALO) {               // padded-grid row -> dense NHWC row; the grid's extra rows are dropped
                    const int orow = halo_out_row(p, grow_);
                    ok = orow >= 0;
                    roff = (size_t)orow * p.ldc + n0;
                }
#pragma unroll
                for (int q = 0; q < kPiecesPerLane; ++q) {
                    const int piece = piece0 + q * 32;
                    const uint4 val = *reinterpret_cast<const uint4*>(wbase + (uint32_t)(plane * 32 + rr) * C::kOutPitch + piece * 16);
                    if (ok && n0 + piece * 8 < p.N) *reinterpret_cast<uint4*>(gout + roff + piece * 8) = val;     // the last column tile may pass N
                }
            }
        };
        auto drain = [&]() {
            if (direct) return;
            if constexpr (C::kEpiHalves == 2) {
                named_barrier_sync(1 + ew, 64);                           // both column halves of these 32 rows are staged
                drain_plane(half);
            } else {
                __syncwarp();
                drain_plane(0);
                drain_plane(1);
            }
        };

        // get the epilogue's global operands in flight (kRing chunks deep), then keep the ring full
        EpiOperands ops[C::kRing];
        const int nbase = (LN ? 0 : n0) + cbeg;
#pragma unroll
        for (int i = 0; i < C::kRing; ++i) prefetch(nbase + 16 * i, ops[i]);
        if (kCanLnA && (has_aln || p.res_ln_part != nullptr)) {
            mbar_wait(vec_full, 0);
            if (has_aln) a_st = st_a[ew * 32 + lane];
            if (res_ln) { res_st = st_r[ew * 32 + lane]; res_shift = -res_st.x * res_st.y; }
        }
        // Narrow tiles read their own accumulators into registers right away: senders push them, owners overlap the
        // shared-memory reads with the wait for the peers' partial rows.
        constexpr bool kPreload = !LN && C::kChunksW <= 2;
        float pre[kPreload ? C::kChunksW : 1][16];
        if constexpr (kPreload) {
#pragma unroll
            for (int ci = 0; ci < C::kChunksW; ++ci) sum_acc(cbeg + ci * 16, pre[ci]);
        }
        if (C::kMaxSplit > 1 && ksplit > 1) {
            if (!mine) {
                // the partial rows have their own region in the owner's shared memory: push as soon as this CTA's
                // MMAs have retired, whatever the owner is doing (source slot: this CTA's rank among the non-owners)
                const uint32_t local = smem_u32(stage_base) + kPartOffset + (uint32_t)(kz < owner ? kz : kz - 1) * part_slot + part_row;
                const uint32_t remote = map_to_cta(local, (uint32_t)owner);
                const uint32_t remote_bar = map_to_cta(smem_u32(part_full), (uint32_t)owner);
                // unscaled partial sums travel; the leader applies acc_scale once in load_acc
#pragma unroll
                for (int ci = 0; ci < C::kChunksW; ++ci) {
                    const int c = cbeg + ci * 16;
                    const float (&v)[16] = pre[kPreload ? ci : 0];      // (split-K only exists on preloading tiles)
#pragma unroll
                    for (int j = 0; j < 16; j += 4)
                        st_async_f32x4(remote + (((uint32_t)((c + j) >> 2) ^ part_swz) << 4), v[j], v[j + 1], v[j + 2], v[j + 3], remote_bar);
                }
            } else {
                mbar_wait(part_full, 0);             // (ksplit - 1) x (128 / ksplit) rows x BN floats have landed
            }
        }
        if (mine) {

        if constexpr (!LN) {
#pragma unroll
            for (int ci = 0; ci < C::kChunksW; ++ci) {
                const int c = cbeg + ci * 16;
                const int nb = n0 + c;
                float v[16];
                if constexpr (kPreload) {
#pragma unroll
                    for (int j = 0; j < 16; ++j) v[j] = pre[ci][j];
                    finish_acc(c, v);
                } else {
                    load_acc(c, v);
                }
                if (BN > 16 || !tail) {                          // (a ragged N only exists in the 16-wide instantiation)
                    apply(ops[ci % C::kRing], v, nb);
                } else {
#pragma unroll
                    for (int j = 0; j < 16; ++j)                 // static indexing keeps v[] in registers
                        if (p.bias && nb + j < p.N) v[j] += __ldg(p.bias + nb + j);
                }
                if (p.relu) {
#pragma unroll
                    for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], 0.f);
                }
                if (kCanLnA && emit_part) {
                    // (mean, M2) of these 16 final values for the consumers' deferred LayerNorm
                    float sm = 0.f;
#pragma unroll
                    for (int j = 0; j < 16; ++j) sm += v[j];
                    sm *= (1.f / 16.f);
                    float m2 = 0.f;
#pragma unroll
                    for (int j = 0; j < 16; ++j) { const float d = v[j] - sm; m2 = fmaf(d, d, m2); }
                    p.ln_part_out[(size_t)row * 16 + (nb >> 4)] = make_float2(sm, m2);
                }
                emit16(c, v);
                if (ci + C::kRing < C::kChunksW) prefetch(nb + 16 * C::kRing, ops[ci % C::kRing]);
            }
            drain();
        } else {
            // fused residual + LayerNorm (eps 1e-5, biased variance) over the 256 columns this thread owns.  One pass
            // over the accumulators: sum and shifted sum of squares (shift = the row's first value, so the
            // E[(x-s)^2] - (mean-s)^2 form does not cancel), values parked back in the accumulator tile for the normalisation pass.
            float sum = 0.f, sq = 0.f, shift = 0.f;
#pragma unroll
            for (int ci = 0; ci < C::kChunksN; ++ci) {
                const int c = ci * 16;
                float v[16];
                load_acc(c, v);
                apply(ops[ci % C::kRing], v, c);
                if (ci + C::kRing < C::kChunksN) prefetch(c + 16 * C::kRing, ops[ci % C::kRing]);
                if (ci == 0) shift = v[0];
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    sum += v[j];
                    const float d = v[j] - shift;
                    sq = fmaf(d, d, sq);
                }
#pragma unroll
                for (int j = 0; j < 16; j += 4)
                    *reinterpret_cast<float4*>(arow + (c + j) * 4) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
            }
            const float mean = sum * (1.f / 256.f);
            const float dm = mean - shift;
            const float var = fmaxf(sq * (1.f / 256.f) - dm * dm, 0.f);
            const float rstd = 1.f / sqrtf(var + 1e-5f);
#pragma unroll 1
            for (int c = 0; c < BN; c += 32) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float r[16];
                    sum_acc(c + h * 16, r);
                    float v[16];
#pragma unroll
                    for (int j = 0; j < 16; j += 4) {
                        const float4 g4 = __ldg(reinterpret_cast<const float4*>(p.ln_gamma + c + h * 16 + j));
                        const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.ln_beta + c + h * 16 + j));
                        v[j] = (r[j] - mean) * rstd * g4.x + b4.x;
                        v[j + 1] = (r[j + 1] - mean) * rstd * g4.y + b4.y;
                        v[j + 2] = (r[j + 2] - mean) * rstd * g4.z + b4.z;
                        v[j + 3] = (r[j + 3] - mean) * rstd * g4.w + b4.w;
                    }
                    emit16(c + h * 16, v);
                }
            }
            drain();
        }
        }   // leader / unsplit epilogue
    }

    // the producer warps leave with the rest of the CTA, after the consumers have seen all of their copies land
    __syncthreads();
}

// ---- host side: a plan (tile width, A loader, deferred-LayerNorm instantiation, split-K, grid), then its launch ----

int bm_of(int bn) { return bn >= 256 ? 64 : 128; }
// Cfg::kMaxSplit, except that the 16-wide tile does not split: the partial rows are XOR-swizzled over 8 16-byte pieces
// per row, and its rows have 4, so a swizzled piece would land in the next row
int max_split(int bn) { return bn == 32 || bn == 64 ? 4 : 1; }

// 3x3 stride-1 "same" convolutions over whole images take the halo loader; cotr_debug_set_variant bit 20 keeps them on
// the implicit im2col (an in-process A/B and the reference of tests/test_conv_halo_gpu.py)
inline bool halo_conv(const GemmParams& p) {
    return p.a_mode == A_CONV_NHWC && p.KH == 3 && p.KW == 3 && p.stride == 1 && p.pad == 1 && p.OH == p.H && p.OW == p.W &&
           (p.C & 63) == 0 && !(g_tc_variant & (1 << 20));
}

// The loader (kernel instantiation) of a tile width; 1 with the error set when none is instantiated.
int plan_loader(const GemmParams& p, GemmPlan& plan) {
    const bool gather = (p.a_mode == A_ROWMAJOR || p.a_mode == A_TOKENS);
    plan.dln = 0;
    if (gather && (p.K & 7) == 0 && (p.lda & 7) == 0) {
        plan.loader = LD_GATHER;
        plan.dln = plan.bn < 256 && (p.a_ln_cs != nullptr || p.res_ln_part != nullptr || p.ln_part_out != nullptr);
        return 0;
    }
    if (plan.bn >= 32 && plan.bn < 256 && p.a_mode == A_CONV_NHWC && (p.C & 63) == 0) {
        plan.loader = halo_conv(p) ? LD_HALO : LD_CONV;
        return 0;
    }
    if (plan.bn == 64 && p.a_mode == A_STEM_NHWC4 && p.K == kStemK) {
        plan.loader = LD_STEM4;
        return 0;
    }
    set_error("gemm_tc: no kernel instantiation for a_mode %d, K %d, lda %d, C %d with tile N %d", p.a_mode, p.K, p.lda, p.C, plan.bn);
    return 1;
}

void plan_grid(const GemmParams& p, GemmPlan& plan) {
    plan.grid_x = plan.loader == LD_HALO ? p.M / (p.OH * p.OW) * halo_tiles_per_img(p) : (p.M + bm_of(plan.bn) - 1) / bm_of(plan.bn);
    plan.grid_y = (p.N + plan.bn - 1) / plan.bn;
}

// Split-K over a thread-block cluster for long reductions on under-filled grids (the K loop is the serial part of
// these latency-bound launches): 4 or 2 CTAs per output tile, each >= 4 chunks, at most ~one wave of CTAs.
// LD_HALO splits by whole channel chunks, into at most one wave of the 132 SMs (layer2 at one pair: 72 tiles split
// by 2 measured 23.4 us against 17.3 us for the im2col launch, its 12 CTAs past the wave running on their own; H100 at 400 W).
int rule_split(const GemmParams& p, const GemmPlan& plan) {
    if (plan.bn >= 256 || plan.loader == LD_STEM4) return 1;
    const int kc = (p.K + BK - 1) / BK;
    const int cc = plan.loader == LD_HALO ? p.C / BK : kc;
    const long long ctas = (long long)plan.grid_x * plan.grid_y;
    const long long wave = plan.loader == LD_HALO ? kNumSms : kWaveCtas;
    if (!(g_tc_variant & 512) && kc >= (16 >> ((g_tc_variant >> 14) & 3))) {     // bring-up knob: bits 14-15
        if (max_split(plan.bn) >= 4 && kc % 4 == 0 && cc % 4 == 0 && ctas * 4 <= wave) return 4;
        if (max_split(plan.bn) >= 2 && kc % 2 == 0 && cc % 2 == 0 && ctas * 2 <= wave) return 2;
    }
    return 1;
}

// The implicit im2col runs the launch when the halo tiles of a CTA's channel chunks do not fit their region, or when the
// halo grid would leave a third of the SMs idle (layer2 at one pair: 72 CTAs of 18 chunks measured 19.0 us against
// 17.3 us for the 128 im2col CTAs of 9 chunks; layer3's 96 halo CTAs beat its im2col grid).
bool halo_fits(const GemmParams& p, const GemmPlan& plan) {
    const int ccp = p.C / BK / plan.ksplit;
    return ccp <= kHaloMaxChunks && (uint32_t)ccp * 2u * halo_plane_bytes(p) <= kHaloMaxBytes &&
           (long long)plan.grid_x * plan.grid_y * plan.ksplit >= kHaloMinCtas;
}

// Split and loader of a plan whose tile width is set: the split rule (or a forced split, 0 = the rule), then the halo
// fit with its fallback to the im2col loader (which takes the split rule again when it was not forced).
int plan_split(const GemmParams& p, GemmPlan& plan, int forced_split) {
    if (plan_loader(p, plan)) return 1;
    plan_grid(p, plan);
    const int kc = (p.K + BK - 1) / BK;
    if (forced_split) {
        const int ks = forced_split;
        const int cc = plan.loader == LD_HALO ? p.C / BK : kc;
        COTR_CHECK(ks == 1 || ks == 2 || ks == 4, "gemm_tc: split-K %d (1, 2 or 4)", ks);
        COTR_CHECK(ks <= max_split(plan.bn) && (ks == 1 || plan.loader != LD_STEM4),
                   "gemm_tc: split-K %d on the %d-wide tile with loader %d", ks, plan.bn, plan.loader);
        COTR_CHECK(kc % ks == 0 && cc % ks == 0, "gemm_tc: split-K %d does not divide %d K chunks (%d channel chunks)", ks, kc, cc);
    }
    plan.ksplit = forced_split ? forced_split : rule_split(p, plan);
    if (plan.loader == LD_HALO && !halo_fits(p, plan)) {
        plan.loader = LD_CONV;
        plan_grid(p, plan);
        if (!forced_split) plan.ksplit = rule_split(p, plan);
    }
    return 0;
}

int check_params(const GemmParams& p) {
    COTR_CHECK(p.M > 0 && p.N > 0 && p.K > 0, "gemm_tc: empty problem %d x %d x %d", p.M, p.N, p.K);
    COTR_CHECK(p.Wtc != nullptr, "gemm_tc: weight has no tensor-core image");
    COTR_CHECK(p.out_f32 != nullptr || (p.N & 15) == 0, "gemm_tc: split16 outputs need N %% 16 == 0 (N=%d)", p.N);
    COTR_CHECK(p.res.hi == nullptr || ((p.ldr & 15) == 0 && (p.N & 15) == 0 && ((uintptr_t)p.res.hi & 31) == 0 && ((uintptr_t)p.res.lo & 31) == 0),
               "gemm_tc: residual needs ldr %% 16 == 0 and 32-byte aligned planes");
    COTR_CHECK(p.addmat == nullptr || ((p.ld_add & 3) == 0 && (p.N & 15) == 0), "gemm_tc: add-matrix needs ld %% 4 == 0");
    COTR_CHECK(p.out_f32 != nullptr || (p.ldc & 7) == 0, "gemm_tc: split16 output needs ldc %% 8 == 0");
    if (p.ln_gamma) COTR_CHECK(p.N == 256 && p.relu == 0 && p.out_f32 == nullptr && !p.remap, "gemm_tc: LayerNorm epilogue needs N = 256");
    return 0;
}

template <int BN, bool LN, int MODE, bool DLN = false>
int launch_one(const GemmParams& p, const GemmPlan& plan, cudaStream_t s) {
    using C = Cfg<BN, MODE>;
    static unsigned long long configured = 0;      // bit per device
    if (first_use_on_device(&configured)) {
        COTR_CHECK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, LN, MODE, DLN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)(C::kSmemBytes + C::kPartMaxBytes)));
    }
    const int ksplit = plan.ksplit;
    const size_t smem = C::kSmemBytes + (size_t)(ksplit - 1) * (C::BM / ksplit) * C::kPartPitch;     // incoming partial rows
    COTR_CHECK_CUDA(launch_kernel_cluster(gemm_tc_kernel<BN, LN, MODE, DLN>, dim3(plan.grid_x, plan.grid_y, ksplit), dim3(kThreads),
                                          smem, s, ksplit, p, tc_npad(p.N)));
    return 0;
}

int launch_plan(const GemmParams& p, const GemmPlan& plan, cudaStream_t s) {
    if (plan.loader == LD_HALO)
        COTR_CHECK(p.M == p.M / (p.OH * p.OW) * p.OH * p.OW && p.res.hi == nullptr && p.addmat == nullptr && !p.remap && p.out_f32 == nullptr,
                   "gemm_tc: the halo loader needs whole images and a plain split16 output");
    COTR_CHECK(p.a_ln_cs == nullptr || (plan.dln && p.K == 256 && p.a_mode == A_ROWMAJOR && p.a_ln_part != nullptr),
               "gemm_tc: the deferred LayerNorm on A needs a row-major operand with K = 256 and its partial statistics");
    COTR_CHECK((p.res_ln_part == nullptr && p.ln_part_out == nullptr) || plan.dln,
               "gemm_tc: deferred-LayerNorm residual / statistics on an unsupported tile");
    COTR_CHECK(p.ln_part_out == nullptr || (p.N == 256 && !p.remap && p.out_f32 == nullptr), "gemm_tc: row statistics need a plain N = 256 output");
    switch (plan.bn) {
        case 256:
            return launch_one<256, true, LD_GATHER>(p, plan, s);
        case 16:
            return plan.dln ? launch_one<16, false, LD_GATHER, true>(p, plan, s) : launch_one<16, false, LD_GATHER>(p, plan, s);
        case 32:
            switch (plan.loader) {
                case LD_GATHER: return plan.dln ? launch_one<32, false, LD_GATHER, true>(p, plan, s) : launch_one<32, false, LD_GATHER>(p, plan, s);
                case LD_CONV: return launch_one<32, false, LD_CONV>(p, plan, s);
                case LD_HALO: return launch_one<32, false, LD_HALO>(p, plan, s);
            }
            break;
        case 64:
            switch (plan.loader) {
                case LD_GATHER: return plan.dln ? launch_one<64, false, LD_GATHER, true>(p, plan, s) : launch_one<64, false, LD_GATHER>(p, plan, s);
                case LD_CONV: return launch_one<64, false, LD_CONV>(p, plan, s);
                case LD_HALO: return launch_one<64, false, LD_HALO>(p, plan, s);
                case LD_STEM4: return launch_one<64, false, LD_STEM4>(p, plan, s);
            }
            break;
    }
    set_error("gemm_tc: no kernel instantiation for tile N %d with loader %d", plan.bn, plan.loader);
    return 1;
}

inline uint16_t f32_to_f16_rn(float f) {     // round-to-nearest-even, saturating, subnormals supported
    uint32_t x;
    memcpy(&x, &f, 4);
    const uint16_t sign = (uint16_t)((x >> 16) & 0x8000u);
    x &= 0x7FFFFFFFu;
    if (x >= 0x47800000u) return sign | 0x7BFFu;                     // >= 65536 (or NaN): clamp to max finite
    if (x < 0x38800000u) {                                           // < 2^-14: fp16 subnormal, spacing 2^-24
        float af;
        memcpy(&af, &x, 4);
        const uint32_t m = (uint32_t)nearbyintf(af * 16777216.0f);   // <= 0x400 (== smallest normal when it rounds up)
        return sign | (uint16_t)m;
    }
    const uint32_t mant = x & 0x7FFFFFu;
    uint32_t h = (((x >> 23) - 112u) << 10) | (mant >> 13);
    const uint32_t rem = mant & 0x1FFFu;
    if (rem > 0x1000u || (rem == 0x1000u && (h & 1u))) ++h;
    if (h >= 0x7C00u) h = 0x7BFFu;
    return sign | (uint16_t)h;
}
inline float f16_to_f32(uint16_t h) {
    const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
    const uint32_t e = (h >> 10) & 0x1Fu, m = h & 0x3FFu;
    float mag;
    if (e == 0) mag = (float)m * (1.0f / 16777216.0f);
    else {
        const uint32_t u = ((e + 112u) << 23) | (m << 13);
        memcpy(&mag, &u, 4);
    }
    uint32_t u;
    memcpy(&u, &mag, 4);
    u |= sign;
    float out;
    memcpy(&out, &u, 4);
    return out;
}

}  // namespace

size_t tc_weight_bytes(int N, int K) {
    const size_t kc = (K + BK - 1) / BK;
    return kc * 2 * (size_t)tc_npad(N) * 128;
}

// Image layout: [k chunk (64)][plane: hi, lo][row (npad)][128 bytes = 8 chunks of 8 halves], chunk c of row r stored
// at chunk position c ^ (r % 8) (SWIZZLE_128B); zero padded in N and K.  The matrix is multiplied by 2^e, e chosen so
// that max|w| * 2^e lies in [2^12, 2^13); returns 2^-e for the epilogue.
float tc_pack_weight(const float* w, int N, int K, void* dst_host) {
    const int npad = tc_npad(N);
    const int kc_n = (K + BK - 1) / BK;
    float amax = 0.f;
    for (size_t i = 0; i < (size_t)N * K; ++i) amax = fmaxf(amax, fabsf(w[i]));
    int e = 0;
    if (amax > 0.f && std::isfinite(amax)) {
        e = 12 - (int)floorf(log2f(amax));
        if (e > 24) e = 24;
        if (e < -24) e = -24;
    }
    const float scale = ldexpf(1.f, e);
    uint16_t* out = reinterpret_cast<uint16_t*>(dst_host);
    for (int kc = 0; kc < kc_n; ++kc)
        for (int r = 0; r < npad; ++r)
            for (int c = 0; c < 8; ++c)
                for (int el = 0; el < 8; ++el) {
                    const int k = kc * BK + c * 8 + el;
                    const float x = (r < N && k < K) ? w[(size_t)r * K + k] * scale : 0.f;
                    const uint16_t hi = f32_to_f16_rn(x);
                    const uint16_t lo = f32_to_f16_rn(x - f16_to_f32(hi));
                    const size_t pos = (size_t)r * 64 + (size_t)((c ^ (r & 7)) * 8) + el;      // in halves
                    out[((size_t)kc * 2 + 0) * npad * 64 + pos] = hi;
                    out[((size_t)kc * 2 + 1) * npad * 64 + pos] = lo;
                }
    return ldexpf(1.f, -e);
}

namespace {

// The tile-width rule.
int rule_tile(const GemmParams& p, int& bn) {
    if (p.ln_gamma) { bn = 256; return 0; }
    if (p.N < 64) {
        COTR_CHECK(p.N <= 16, "gemm_tc: N between 17 and 63 is not instantiated");
        bn = 16;
        return 0;
    }
    // Tile width: at small batch most GEMMs of this network have a handful of 128-row tiles, so the 64-wide tile wins
    // once it yields ~86 CTAs (two thirds of the 132 SMs); the 32-wide tile trades tensor efficiency for parallelism
    // and a shorter per-CTA epilogue (the critical path of these latency-bound launches).  There is no wider tile: a
    // 128 x 128 register accumulator leaves room for a single main slot, and the longer truncating chain of the
    // K = 1152 / 2304 convolutions then moved the 16-pair fixture's predictions 3.7e-4 from the fp64 reference (H100)
    // where the 64-wide tile's two main slots keep it within the 3e-4 the tests hold it to.
    const long long mt = halo_conv(p) ? (long long)(p.M / (p.OH * p.OW)) * halo_tiles_per_img(p) : (p.M + 127) / 128;
    // bring-up knob (cotr_debug_set_variant): bits 10-11 move the CTA-count threshold of the 64-wide tile
    static const long long kThr[4] = {86, 43, 57, 132};
    const long long thr64 = kThr[(g_tc_variant >> 10) & 3];
    bn = (mt * ((p.N + 63) / 64) >= thr64 || p.a_mode == A_STEM_NHWC4 || (p.N % 32) != 0) ? 64 : 32;
    return 0;
}

}  // namespace

int launch_gemm_tc(const GemmParams& p, cudaStream_t s) {
    GemmPlan plan{};
    if (check_params(p) || rule_tile(p, plan.bn) || plan_split(p, plan, 0)) return 1;
    return launch_plan(p, plan, s);
}

int launch_gemm_tc_forced(const GemmParams& p, int bn, int ksplit, GemmPlan* used, cudaStream_t s) {
    GemmPlan plan{};
    if (check_params(p)) return 1;
    if (bn == 0) {
        if (rule_tile(p, plan.bn)) return 1;
    } else {
        const bool ok = p.ln_gamma ? bn == 256 : (p.N <= 16 ? bn == 16 : (p.N >= 64 && (bn == 64 || (bn == 32 && p.N % 32 == 0))));
        COTR_CHECK(ok, "gemm_tc: no %d-wide tile for N = %d%s", bn, p.N, p.ln_gamma ? " with the LayerNorm epilogue" : "");
        plan.bn = bn;
    }
    if (plan_split(p, plan, ksplit)) return 1;
    if (used) *used = plan;
    return launch_plan(p, plan, s);
}

}  // namespace cotr
