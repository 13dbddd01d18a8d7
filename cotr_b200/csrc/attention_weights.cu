// Head-averaged attention weights over the 512-token context: out[i][key] = (1/8) sum_{h=0..7} softmax_key(q_h[i] . k_h[key]),
// the second output of the reference's nn.MultiheadAttention (need_weights=True, average_attn_weights=True).  The
// forward never needs them (attention_tc.cu keeps P in registers); these kernels materialise them for the layers a
// caller asks for (cotr_encode_context_attention / cotr_decode_attention), reading the operands the layer's attention
// launch read and writing fp32.
//
// Tensor-core kernel: one CTA (one warpgroup) per (64-query tile, image pair) owns all 8 heads of its rows, so the
// head sum is a fixed-order sum in shared memory (no atomics: bitwise reproducible).  Per head:
//   * the head's K operand image (64 KB, common.cuh) arrives by one bulk-TMA copy, its 64 x 32 Q slice by cp.async;
//   * stats pass: S = Q K^T per 64-key chunk with the split16 products of attention_tc.cu (Q_hi K_hi into the main
//     accumulator, Q_lo K_hi + Q_hi K_lo into a separate correction accumulator: the tensor core's fp32 accumulate
//     truncates), online row max and sum over all 512 keys;
//   * weights pass: the same chunks are recomputed (bit-identical S), P = exp(S - max) / sum is exact against the full
//     row, and the 64 x 512 fp32 head-sum tile in shared memory accumulates P in head order 0..7.
// Then the tile, times 1/8, is streamed to HBM row by row.  Rows past nq are zero-filled on staging and never stored.
//
// fp32 SIMT kernel: the same map in plain fp32 arithmetic from the row-major K the SIMT path keeps (cross-check path).
#include "split16.cuh"
#include "tc_common.cuh"

namespace cotr {

namespace {

using namespace tc;

constexpr int kRows = 64;                                  // query rows per CTA
constexpr int kThreads = 128;                              // one warpgroup
constexpr int kChunk = 64;                                 // keys per MMA chunk
constexpr int kChunks = kTokens / kChunk;                  // 8
constexpr uint32_t kQLbo = kRows * 16;                     // Q tile [4 K-groups][64 rows][16 B]
constexpr uint32_t kQPlane = 4 * kQLbo;                    // 4 KB
constexpr uint32_t kKLbo = kTokens * 16;                   // K image [4 K-groups][512 keys][16 B]
constexpr uint32_t kKPlane = 4 * kKLbo;                    // 32 KB
constexpr uint32_t kSbo = 128;
constexpr int kAccPitch = kTokens + 8;                     // floats per head-sum row: padded, conflict-free float2 updates

constexpr uint32_t kOffK = 0;
constexpr uint32_t kOffQ = kOffK + 2 * kKPlane;
constexpr uint32_t kOffAcc = kOffQ + 2 * kQPlane;
constexpr uint32_t kOffBar = kOffAcc + (uint32_t)(kRows * kAccPitch * sizeof(float));
constexpr uint32_t kSmemBytes = kOffBar + 64;              // 202 KB + barriers
static_assert(kSmemBytes <= 227 * 1024, "attention-weights tile does not fit shared memory");
static_assert(2 * kKPlane == kAttnKImgBytes && kKPlane == kAttnKPlaneBytes, "K operand image and shared-memory tile went out of step");

constexpr float kLog2e = 1.4426950408889634f;

__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// S (64 rows x keys [64 c, 64 c + 64)) of the staged head, accumulator fragment layout: register 4 j + {0,1} = row
// (warp % 4) * 16 + lane / 4 ("row a"), columns 8 j + 2 (lane % 4) + {0,1}; registers 4 j + {2,3} = row a + 8 ("row b").
__device__ __forceinline__ void chunk_scores(uint32_t sbase, int c, float (&s)[32]) {
    float sm[32], sc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) { sm[j] = 0.f; sc[j] = 0.f; }
    fence_regs(sm); fence_regs(sc);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
        const uint32_t qa = sbase + kOffQ + ks * 2 * kQLbo;
        const uint32_t ka = sbase + kOffK + c * kChunk * 16 + ks * 2 * kKLbo;
        const uint64_t qh = make_smem_desc(qa, kQLbo, kSbo), ql = make_smem_desc(qa + kQPlane, kQLbo, kSbo);
        const uint64_t kh = make_smem_desc(ka, kKLbo, kSbo), kl = make_smem_desc(ka + kKPlane, kKLbo, kSbo);
        wgmma_ss_n64(sc, ql, kh);
        wgmma_ss_n64(sc, qh, kl);
        wgmma_ss_n64(sm, qh, kh);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(sm); fence_regs(sc);
#pragma unroll
    for (int j = 0; j < 32; ++j) s[j] = sm[j] + sc[j];
}

__global__ void __launch_bounds__(kThreads) attention_weights_tc_kernel(const AttnWeightsParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t* k_full = reinterpret_cast<uint64_t*>(smem + kOffBar);      // the head's K image has landed (bulk TMA)
    uint64_t* q_full = k_full + 1;                                       // every thread's Q copies have landed
    float* acc = reinterpret_cast<float*>(smem + kOffAcc);

    const int t = threadIdx.x;
    const int warp = t >> 5, lane = t & 31;
    const int pair_local = blockIdx.y;
    const int row0 = blockIdx.x * kRows;
    if (t == 0) {
        mbar_init(k_full, 1);
        mbar_init(q_full, kThreads);
        mbar_fence_init();
    }
    __syncthreads();
    const uint32_t sbase = smem_u32(smem);
    if (t == 0) pdl_launch_dependents();
    pdl_wait();                                          // q and the K images are written by the previous launches

    const unsigned char* img = p.kv_img + (size_t)(p.pair0 + pair_local) * p.img_pair_stride;
    // Q staging: row t % 64, two of the four 16-byte K groups per thread; rows past nq are zero-filled
    const int qr = t & (kRows - 1), kg0 = (t >> 6) * 2;
    const bool q_ok = row0 + qr < p.nq;
    const size_t qrow = ((size_t)pair_local * p.nq + (q_ok ? row0 + qr : 0)) * p.ldq;
    const int ra = warp * 16 + (lane >> 2);              // fragment rows ra (registers 4 j + {0,1}) and ra + 8
    float* acc_a = acc + ra * kAccPitch + 2 * (lane & 3);
    float* acc_b = acc_a + 8 * kAccPitch;

#pragma unroll 1
    for (int h = 0; h < kHeads; ++h) {
        if (t == 0) {
            mbar_arrive_expect_tx(k_full, (uint32_t)kAttnKImgBytes);
            tma_bulk_g2s(smem + kOffK, img + (size_t)h * kAttnHeadImgBytes, (uint32_t)kAttnKImgBytes, k_full);
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int kg = kg0 + j;
            const uint32_t dst = sbase + kOffQ + kg * kQLbo + qr * 16;
            cp_async16(dst, p.q.hi + qrow + h * kHeadDim + kg * 8, q_ok ? 16u : 0u);
            cp_async16(dst + kQPlane, p.q.lo + qrow + h * kHeadDim + kg * 8, q_ok ? 16u : 0u);
        }
        cp_async_mbar_arrive_noinc(q_full);
        mbar_wait(q_full, h & 1);
        mbar_wait(k_full, h & 1);
        fence_proxy_async_smem();                        // cp.async (generic proxy) data -> wgmma (async proxy)

        // ---- stats pass: row max and sum over all 512 keys (online over the chunks; a row is shared by a quad) ----
        float mx_a = -INFINITY, mx_b = -INFINITY, sum_a = 0.f, sum_b = 0.f;
#pragma unroll 1
        for (int c = 0; c < kChunks; ++c) {
            float s[32];
            chunk_scores(sbase, c, s);
            float cm_a = -INFINITY, cm_b = -INFINITY;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                cm_a = fmaxf(cm_a, fmaxf(s[4 * j], s[4 * j + 1]));
                cm_b = fmaxf(cm_b, fmaxf(s[4 * j + 2], s[4 * j + 3]));
            }
#pragma unroll
            for (int step = 1; step < 4; step <<= 1) {
                cm_a = fmaxf(cm_a, __shfl_xor_sync(0xffffffffu, cm_a, step));
                cm_b = fmaxf(cm_b, __shfl_xor_sync(0xffffffffu, cm_b, step));
            }
            const float nm_a = fmaxf(mx_a, cm_a), nm_b = fmaxf(mx_b, cm_b);
            sum_a *= fast_exp2((mx_a - nm_a) * kLog2e);  // 0 on the first chunk
            sum_b *= fast_exp2((mx_b - nm_b) * kLog2e);
            mx_a = nm_a; mx_b = nm_b;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                sum_a += fast_exp2((s[4 * j] - mx_a) * kLog2e) + fast_exp2((s[4 * j + 1] - mx_a) * kLog2e);
                sum_b += fast_exp2((s[4 * j + 2] - mx_b) * kLog2e) + fast_exp2((s[4 * j + 3] - mx_b) * kLog2e);
            }
        }
#pragma unroll
        for (int step = 1; step < 4; step <<= 1) {
            sum_a += __shfl_xor_sync(0xffffffffu, sum_a, step);
            sum_b += __shfl_xor_sync(0xffffffffu, sum_b, step);
        }
        const float inv_a = 1.f / sum_a, inv_b = 1.f / sum_b;

        // ---- weights pass: recompute S, P = exp(S - max) / sum, add into the head-sum tile (each thread owns its
        // fragment's elements, so the order over heads is fixed and no synchronisation is needed between heads) ----
#pragma unroll 1
        for (int c = 0; c < kChunks; ++c) {
            float s[32];
            chunk_scores(sbase, c, s);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int col = c * kChunk + 8 * j;
                float2 pa = make_float2(fast_exp2((s[4 * j] - mx_a) * kLog2e) * inv_a, fast_exp2((s[4 * j + 1] - mx_a) * kLog2e) * inv_a);
                float2 pb = make_float2(fast_exp2((s[4 * j + 2] - mx_b) * kLog2e) * inv_b, fast_exp2((s[4 * j + 3] - mx_b) * kLog2e) * inv_b);
                float2* da = reinterpret_cast<float2*>(acc_a + col);
                float2* db = reinterpret_cast<float2*>(acc_b + col);
                if (h > 0) {
                    const float2 oa = *da, ob = *db;
                    pa.x += oa.x; pa.y += oa.y;
                    pb.x += ob.x; pb.y += ob.y;
                }
                *da = pa;
                *db = pb;
            }
        }
        __syncthreads();                                 // every warp is done with this head's Q and K tiles
    }

    // ---- the head-sum tile / 8 -> HBM: one 2 KB row per step, 16 bytes per thread, streaming stores ----
    float* out = p.out + (size_t)pair_local * p.out_pair_stride + (size_t)row0 * kTokens;
    const int rows = min(kRows, p.nq - row0);
#pragma unroll 4
    for (int i = 0; i < rows; ++i) {
        float4 v = *reinterpret_cast<const float4*>(acc + i * kAccPitch + 4 * t);
        v.x *= 0.125f; v.y *= 0.125f; v.z *= 0.125f; v.w *= 0.125f;
        __stcs(reinterpret_cast<float4*>(out + (size_t)i * kTokens + 4 * t), v);
    }
}

// ---- fp32 SIMT twin: 8 warps x 4 rows per CTA, the head sum in registers ---------------------------------------
constexpr int kSimtWarps = 8;
constexpr int kSimtRowsPerWarp = 4;
constexpr int kSimtRows = kSimtWarps * kSimtRowsPerWarp;
constexpr int kKStride = kHeadDim + 1;                     // padded: lane j reads key (j + 32 i) without bank conflicts
constexpr size_t kSimtSmemBytes = (size_t)(kTokens * kKStride + kSimtRows * kHeadDim) * sizeof(float);

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__global__ void __launch_bounds__(kSimtWarps * 32) attention_weights_simt_kernel(const AttnWeightsParams p) {
    extern __shared__ __align__(16) float smem_f[];
    float* Ks = smem_f;                                  // [512][33]
    float* Qs = Ks + kTokens * kKStride;                 // [32 rows][32]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int pair_local = blockIdx.y;
    const int row_begin = blockIdx.x * kSimtRows + warp * kSimtRowsPerWarp;
    const size_t kv_row0 = (size_t)(p.pair0 + pair_local) * kTokens;
    if (tid == 0) pdl_launch_dependents();
    pdl_wait();

    float acc[kSimtRowsPerWarp][kTokens / 32];
#pragma unroll
    for (int r = 0; r < kSimtRowsPerWarp; ++r)
#pragma unroll
        for (int u = 0; u < kTokens / 32; ++u) acc[r][u] = 0.f;
    float* qs = Qs + warp * kSimtRowsPerWarp * kHeadDim;
#pragma unroll 1
    for (int h = 0; h < kHeads; ++h) {
        __syncthreads();                                 // the previous head's keys are no longer read
        for (int idx = tid; idx < kTokens * (kHeadDim / 8); idx += blockDim.x) {
            const int key = idx >> 2, d8 = (idx & 3) * 8;
            float v[8];
            load8_split(p.k, (kv_row0 + key) * p.ldk + h * kHeadDim + d8, v);
#pragma unroll
            for (int j = 0; j < 8; ++j) Ks[key * kKStride + d8 + j] = v[j];
        }
#pragma unroll
        for (int r = 0; r < kSimtRowsPerWarp; ++r) {
            const int i = row_begin + r;
            const size_t q = ((size_t)pair_local * p.nq + i) * p.ldq + h * kHeadDim + lane;
            qs[r * kHeadDim + lane] = i < p.nq ? join_f16(p.q.hi[q], p.q.lo[q]) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < kSimtRowsPerWarp; ++r) {
            if (row_begin + r >= p.nq) break;
            float s[kTokens / 32];
#pragma unroll
            for (int u = 0; u < kTokens / 32; ++u) s[u] = 0.f;
#pragma unroll 8
            for (int d = 0; d < kHeadDim; ++d) {
                const float qd = qs[r * kHeadDim + d];
#pragma unroll
                for (int u = 0; u < kTokens / 32; ++u) s[u] = fmaf(qd, Ks[(lane + 32 * u) * kKStride + d], s[u]);
            }
            float mx = s[0];
#pragma unroll
            for (int u = 1; u < kTokens / 32; ++u) mx = fmaxf(mx, s[u]);
            mx = warp_max(mx);
            float sum = 0.f;
#pragma unroll
            for (int u = 0; u < kTokens / 32; ++u) { s[u] = expf(s[u] - mx); sum += s[u]; }
            sum = warp_sum(sum);
#pragma unroll
            for (int u = 0; u < kTokens / 32; ++u) acc[r][u] += s[u] / sum;
        }
    }
#pragma unroll
    for (int r = 0; r < kSimtRowsPerWarp; ++r) {
        const int i = row_begin + r;
        if (i >= p.nq) break;
        float* o = p.out + (size_t)pair_local * p.out_pair_stride + (size_t)i * kTokens;
#pragma unroll
        for (int u = 0; u < kTokens / 32; ++u) o[lane + 32 * u] = acc[r][u] * 0.125f;
    }
}

}  // namespace

int launch_attention_weights_tc(const AttnWeightsParams& p, cudaStream_t s) {
    if (p.nq <= 0 || p.npairs <= 0) return 0;
    COTR_CHECK(p.kv_img != nullptr, "attention_weights_tc: the keys must be attention operand images");
    COTR_CHECK(p.npairs <= 65535, "attention_weights: too many pairs in one launch (%d)", p.npairs);
    COTR_CHECK((p.ldq & 7) == 0, "attention_weights_tc: the leading dimension of q must be a multiple of 8 elements");
    static unsigned long long configured = 0;      // bit per device
    if (first_use_on_device(&configured)) {
        COTR_CHECK_CUDA(cudaFuncSetAttribute(attention_weights_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
    }
    const dim3 grid((p.nq + kRows - 1) / kRows, p.npairs);
    COTR_CHECK_CUDA(launch_kernel(attention_weights_tc_kernel, grid, dim3(kThreads), kSmemBytes, s, p));
    return 0;
}

int launch_attention_weights_simt(const AttnWeightsParams& p, cudaStream_t s) {
    if (p.nq <= 0 || p.npairs <= 0) return 0;
    COTR_CHECK(p.k.hi != nullptr, "attention_weights_simt: the keys must be row-major split16");
    COTR_CHECK(p.npairs <= 65535, "attention_weights: too many pairs in one launch (%d)", p.npairs);
    static unsigned long long configured = 0;      // bit per device
    if (first_use_on_device(&configured)) {
        COTR_CHECK_CUDA(cudaFuncSetAttribute(attention_weights_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSimtSmemBytes));
    }
    const dim3 grid((p.nq + kSimtRows - 1) / kSimtRows, p.npairs);
    COTR_CHECK_CUDA(launch_kernel(attention_weights_simt_kernel, grid, dim3(kSimtWarps * 32), kSimtSmemBytes, s, p));
    return 0;
}

}  // namespace cotr
