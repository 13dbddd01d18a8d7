// fp32 SIMT GEMM on split16 activations with the same implicit-im2col A addressing and the same epilogue contract as
// the wgmma GEMM.  Numerical cross-check path (cotr_set_gemm_path(m, 1): plain fp32 FMA arithmetic on the
// reconstructed hi + lo values) and the producer of the constant position-bias matrices at model creation.
#include "a_loader.cuh"

namespace cotr {

namespace {

constexpr int BM = 64, BN = 64, BK = 16, PADM = 4;

// A[m, k..k+3] as fp32 (k % 4 == 0)
__device__ __forceinline__ float4 load_a4_f32(const GemmParams& p, const ARow& r, int k) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    size_t off;
    if (!a_offset8(p, r, k & ~7, off)) return v;     // all split16 operands have K % 8 == 0
    off += (k & 4);
    const uint2 h = __ldcg(reinterpret_cast<const uint2*>(p.a.hi + off));
    const uint2 l = __ldcg(reinterpret_cast<const uint2*>(p.a.lo + off));
    const float2 a = join_f16x2(h.x, l.x), b = join_f16x2(h.y, l.y);
    return make_float4(a.x, a.y, b.x, b.y);
}

__global__ void __launch_bounds__(256) gemm_simt_kernel(const GemmParams p, float* __restrict__ raw_out) {
    __shared__ __align__(16) float As[BK][BM + PADM];
    __shared__ __align__(16) float Bs[BK][BN + PADM];

    const int tid = threadIdx.x;
    const int m0 = blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    if (tid == 0) pdl_launch_dependents();
    pdl_wait();

    const int lrow = tid >> 2;          // 0..63
    const int lk = (tid & 3) * 4;       // 0,4,8,12
    const ARow arow = decode_a_row(p, m0 + lrow);
    const int wn = n0 + lrow;
    const float* wrow = p.Wt + (size_t)wn * p.K;
    const bool w_vec = (p.K & 3) == 0;

    const int ty = tid >> 4, tx = tid & 15;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < p.K; k0 += BK) {
        const int k = k0 + lk;
        const float4 a = load_a4_f32(p, arow, k);
        float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
        if (wn < p.N && k < p.K) {
            if (w_vec) {
                b = __ldg(reinterpret_cast<const float4*>(wrow + k));
            } else {
                b.x = __ldg(wrow + k);
                if (k + 1 < p.K) b.y = __ldg(wrow + k + 1);
                if (k + 2 < p.K) b.z = __ldg(wrow + k + 2);
                if (k + 3 < p.K) b.w = __ldg(wrow + k + 3);
            }
        }
        __syncthreads();
        As[lk + 0][lrow] = a.x; As[lk + 1][lrow] = a.y; As[lk + 2][lrow] = a.z; As[lk + 3][lrow] = a.w;
        Bs[lk + 0][lrow] = b.x; Bs[lk + 1][lrow] = b.y; Bs[lk + 2][lrow] = b.z; Bs[lk + 3][lrow] = b.w;
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            const float4 av = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 bv = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            const float ar[4] = {av.x, av.y, av.z, av.w};
            const float br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
        }
    }

#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= p.M) continue;
        const float* add_row = p.addmat ? p.addmat + (size_t)(m % p.add_period) * p.ld_add : nullptr;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= p.N) continue;
            float v = acc[i][j];
            if (p.bias) v += __ldg(p.bias + n);
            if (add_row) v += __ldg(add_row + n);
            if (p.res.hi) v += join_f16(p.res.hi[(size_t)m * p.ldr + n], p.res.lo[(size_t)m * p.ldr + n]);
            if (p.relu) v = fmaxf(v, 0.f);
            if (raw_out) {                       // fp32 scratch (pre-LayerNorm rows, or a constant add-matrix)
                raw_out[(size_t)m * p.N + n] = v;
            } else if (p.out_f32) {
                p.out_f32[(size_t)m * p.ldc + n] = v;
            } else {
                size_t base;
                const bool transposed = out_location(p, m, n & ~15, base);
                const size_t idx = transposed ? base + (size_t)(n & 15) * kTokens : base + (n & 15);
                __half h, l;
                split_f16(v, h, l);
                if (transposed) { p.vt.hi[idx] = h; p.vt.lo[idx] = l; }
                else { p.out.hi[idx] = h; p.out.lo[idx] = l; }
            }
        }
    }
}

}  // namespace

// raw_out != nullptr: write the epilogue result as plain fp32 [M, N] there instead of p.out (used for the constant
// add-matrices and as the LayerNorm staging buffer of the SIMT path).
int launch_gemm_simt_raw(const GemmParams& p, float* raw_out, cudaStream_t s) {
    COTR_CHECK(p.M > 0 && p.N > 0 && p.K > 0, "gemm_simt: empty problem %d x %d x %d", p.M, p.N, p.K);
    COTR_CHECK((p.K & 7) == 0, "gemm_simt: split16 operands need K %% 8 == 0 (K=%d)", p.K);
    COTR_CHECK(p.a_mode != A_CONV_NHWC || (p.C & 7) == 0, "gemm_simt: NHWC conv needs C %% 8 == 0 (C=%d)", p.C);
    COTR_CHECK(p.ln_gamma == nullptr, "gemm_simt: fused LayerNorm is a tensor-core-path feature");
    dim3 grid((p.M + BM - 1) / BM, (p.N + BN - 1) / BN);
    COTR_CHECK_CUDA(launch_kernel(gemm_simt_kernel, grid, dim3(256), 0, s, p, raw_out));
    return 0;
}

int launch_gemm_simt(const GemmParams& p, cudaStream_t s) { return launch_gemm_simt_raw(p, nullptr, s); }

}  // namespace cotr
