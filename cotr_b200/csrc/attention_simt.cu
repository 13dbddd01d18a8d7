// fp32 SIMT attention over the 512-token context on split16 operands: exact softmax(q k^T) v per head in plain fp32
// arithmetic.  Numerical cross-check path for attention_tc.cu; also used for launches with very few query rows per
// pair (the default engine's one-query-per-context step), where a 128-row MMA tile would be almost all padding.
#include "split16.cuh"

namespace cotr {

namespace {

constexpr int kRowsPerCta = kAttnSimtTileRows;   // 64
constexpr int kWarps = 8;
constexpr int kKStride = kHeadDim + 1;   // padded: lane j reads key (j + 32 i) without bank conflicts

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__global__ void __launch_bounds__(kWarps * 32) attention_simt_kernel(const AttnParams p) {
    extern __shared__ __align__(16) float smem_f[];
    float* Ks = smem_f;                                // [512][33]
    float* Vs = Ks + kTokens * kKStride;               // [512][32]
    float* Qs = Vs + kTokens * kHeadDim;               // [kWarps][32]

    const int head = blockIdx.y;
    // this CTA's query rows: q / out rows qrow0 .. qrow0 + nrows - 1 (at most kRowsPerCta)
    int pair_local, qrow0, nrows;
    if (p.tiles) {
        const int4 tl = p.tiles[blockIdx.x];
        pair_local = tl.x; qrow0 = tl.y; nrows = tl.z;
    } else {
        pair_local = blockIdx.z;
        qrow0 = pair_local * p.nq + blockIdx.x * kRowsPerCta;
        nrows = min(kRowsPerCta, p.nq - blockIdx.x * kRowsPerCta);
    }
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    const size_t kv_row0 = (size_t)(p.pair0 + pair_local) * kTokens;
    if (tid == 0) pdl_launch_dependents();
    pdl_wait();
    // keys / values either row-major / transposed (fp32 SIMT schedule) or as the attention operand images the
    // tensor-core schedule writes (common.cuh kAttnHeadImgBytes) - this kernel also serves its launches with < 32 query rows
    const unsigned char* img = p.kv_img ? p.kv_img + (size_t)(p.pair0 + pair_local) * p.img_pair_stride + (size_t)head * kAttnHeadImgBytes : nullptr;
    for (int idx = tid; idx < kTokens * (kHeadDim / 8); idx += blockDim.x) {        // K rows: 8 elements per step
        const int key = idx >> 2, d8 = (idx & 3) * 8;
        float v[8];
        if (img) {
            const CSplit16 kimg{reinterpret_cast<const __half*>(img), reinterpret_cast<const __half*>(img + kAttnKPlaneBytes)};
            load8_split(kimg, ((size_t)(d8 >> 3) * kTokens + key) * 8, v);
        } else
        load8_split(p.k, (kv_row0 + key) * p.ldk + head * kHeadDim + d8, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) Ks[key * kKStride + d8 + j] = v[j];
    }
    const size_t vbase = (size_t)(p.pair0 + pair_local) * p.vt_pair_stride + (size_t)head * kHeadDim * kTokens;
    for (int idx = tid; idx < kHeadDim * (kTokens / 8); idx += blockDim.x) {        // V^T rows: 8 keys per step
        const int d = idx >> 6, k8 = (idx & 63) * 8;
        float v[8];
        if (img) {
            const unsigned char* g = img + kAttnKImgBytes + (size_t)(k8 >> 3) * kAttnVGroupBytes + (size_t)d * 16;
            const CSplit16 vimg{reinterpret_cast<const __half*>(g), reinterpret_cast<const __half*>(g + kHeadDim * 16)};
            load8_split(vimg, 0, v);
        } else
        load8_split(p.vt, vbase + (size_t)d * kTokens + k8, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) Vs[(k8 + j) * kHeadDim + d] = v[j];
    }
    __syncthreads();

    float* qs = Qs + warp * kHeadDim;
    for (int i = warp; i < nrows; i += kWarps) {
        const size_t r = (size_t)qrow0 + i;
        qs[lane] = join_f16(p.q.hi[r * p.ldq + head * kHeadDim + lane], p.q.lo[r * p.ldq + head * kHeadDim + lane]);
        __syncwarp();
        float s[kTokens / 32];
#pragma unroll
        for (int t = 0; t < kTokens / 32; ++t) s[t] = 0.f;
#pragma unroll 8
        for (int d = 0; d < kHeadDim; ++d) {
            const float qd = qs[d];
#pragma unroll
            for (int t = 0; t < kTokens / 32; ++t) s[t] = fmaf(qd, Ks[(lane + 32 * t) * kKStride + d], s[t]);
        }
        float mx = s[0];
#pragma unroll
        for (int t = 1; t < kTokens / 32; ++t) mx = fmaxf(mx, s[t]);
        mx = warp_max(mx);
        float sum = 0.f;
#pragma unroll
        for (int t = 0; t < kTokens / 32; ++t) { s[t] = expf(s[t] - mx); sum += s[t]; }
        sum = warp_sum(sum);
        float acc = 0.f;
#pragma unroll
        for (int t = 0; t < kTokens / 32; ++t) {
#pragma unroll
            for (int l = 0; l < 32; ++l) {
                const float pj = __shfl_sync(0xffffffffu, s[t], l);
                acc = fmaf(pj, Vs[(l + 32 * t) * kHeadDim + lane], acc);
            }
        }
        __half h, lo;
        split_f16(acc / sum, h, lo);
        p.out.hi[r * p.ldo + head * kHeadDim + lane] = h;
        p.out.lo[r * p.ldo + head * kHeadDim + lane] = lo;
        __syncwarp();
    }
}

constexpr size_t kSmemBytes = (size_t)(kTokens * kKStride + kTokens * kHeadDim + kWarps * kHeadDim) * sizeof(float);

}  // namespace

int launch_attention_simt(const AttnParams& p, cudaStream_t s) {
    if (p.tiles ? p.n_tiles <= 0 : (p.nq <= 0 || p.npairs <= 0)) return 0;
    static unsigned long long configured = 0;      // bit per device
    if (first_use_on_device(&configured)) {
        COTR_CHECK_CUDA(cudaFuncSetAttribute(attention_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes));
    }
    COTR_CHECK(p.tiles || p.npairs <= 65535, "attention: too many pairs in one launch (%d)", p.npairs);
    const dim3 grid = p.tiles ? dim3(p.n_tiles, kHeads, 1) : dim3((p.nq + kRowsPerCta - 1) / kRowsPerCta, kHeads, p.npairs);
    COTR_CHECK_CUDA(launch_kernel(attention_simt_kernel, grid, dim3(kWarps * 32), kSmemBytes, s, p));
    return 0;
}

}  // namespace cotr
