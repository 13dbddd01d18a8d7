// Small HBM-bound kernels of the hot path on split16 activations: stem max-pool, LayerNorm, lin_sine query encoding,
// and the fp32 <-> split16 converters used at the boundary (test hooks, debug reads, constant tables).
#include "split16.cuh"

namespace cotr {

namespace {

// torchvision resnet stem: MaxPool2d(kernel 3, stride 2, padding 1) on NHWC, 8 channels per thread.
__global__ void maxpool_3x3s2_nhwc_kernel(const CSplit16 in, const Split16 out, int N, int H, int W, int C8) {
    const int OH = H / 2, OW = W / 2;
    const size_t total = (size_t)N * OH * OW * C8;
    if (threadIdx.x == 0) pdl_launch_dependents();
    pdl_wait();
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total;
         idx += (size_t)gridDim.x * blockDim.x) {
        const int c8 = idx % C8;
        size_t t = idx / C8;
        const int ow = t % OW; t /= OW;
        const int oh = t % OH;
        const int n = t / OH;
        float m[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) m[j] = -INFINITY;
#pragma unroll
        for (int dh = 0; dh < 3; ++dh) {
            const int ih = oh * 2 - 1 + dh;
            if (ih < 0 || ih >= H) continue;
#pragma unroll
            for (int dw = 0; dw < 3; ++dw) {
                const int iw = ow * 2 - 1 + dw;
                if (iw < 0 || iw >= W) continue;
                float v[8];
                load8_split(in, ((((size_t)n * H + ih) * W + iw) * C8 + c8) * 8, v);
#pragma unroll
                for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], v[j]);
            }
        }
        store8_split(out, idx * 8, m);      // hi + lo is exact in fp32, so the re-split is lossless
    }
}

// The stem's operand (common.cuh "The stem's input"): fp32 NCHW 256x256 images -> per image n the split16 NHWC4 copy with
// a zero border.  Image n starts at img + (n >> 1) * pair_stride + (n & 1) * half_offset and has row pitch `pitch` (channel
// stride 256 * pitch), which covers both sources: the halves of a (B,3,256,512) canvas (3*256*512, 256, 512) and a
// (N,3,256,256) batch (2*3*256*256, 3*256*256, 256).  One thread per pixel: three coalesced channel reads, one 8-byte
// store per plane.
__global__ void __launch_bounds__(256) stem_canvas_kernel(const float* __restrict__ img, size_t pair_stride, size_t half_offset,
                                                          int pitch, const Split16 canvas, int n_img) {
    if (threadIdx.x == 0) pdl_launch_dependents();
    pdl_wait();
    const size_t total = (size_t)n_img * 256 * 256;
    const size_t plane = (size_t)256 * pitch;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(idx & 255), y = (int)((idx >> 8) & 255), n = (int)(idx >> 16);
        const float* src = img + (size_t)(n >> 1) * pair_stride + (n & 1) * half_offset + (size_t)y * pitch + x;
        const float r = __ldcg(src), g = __ldcg(src + plane), b = __ldcg(src + 2 * plane);
        uint2 h, l;
        split_f16x2(r, g, h.x, l.x);
        split_f16x2(b, 0.f, h.y, l.y);
        const size_t off = (size_t)n * kStemCanvasElems + ((size_t)(y + 3) * kStemCanvasPitch + (x + 3)) * 4;
        *reinterpret_cast<uint2*>(canvas.hi + off) = h;
        *reinterpret_cast<uint2*>(canvas.lo + off) = l;
    }
}

// (mean, M2) of every 16-channel chunk of a row: two neighbouring lanes (8 channels each) share a chunk
__global__ void __launch_bounds__(256) ln_partials_kernel(const CSplit16 x, float2* __restrict__ part, int rows) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= rows) return;
    float v[8];
    load8_split(x, (size_t)warp * kDModel + lane * 8, v);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += v[j];
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    const float mean = s * (1.f / 16.f);
    float m2 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float d = v[j] - mean; m2 = fmaf(d, d, m2); }
    m2 += __shfl_xor_sync(0xffffffffu, m2, 1);
    if ((lane & 1) == 0) part[(size_t)warp * 16 + (lane >> 1)] = make_float2(mean, m2);
}

// out = LN_b(LN_a(x)), one warp per row (the decoder's last norm3 followed by decoder.norm)
__global__ void __launch_bounds__(256) layernorm256_twice_kernel(const CSplit16 x, const float* __restrict__ g1, const float* __restrict__ b1,
                                                                 const float* __restrict__ g2, const float* __restrict__ b2,
                                                                 const Split16 out, int rows) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) pdl_launch_dependents();
    pdl_wait();
    if (warp < rows) {
        const size_t off = (size_t)warp * kDModel + lane * 8;
        float v[8];
        load8_split(x, off, v);
        warp_layernorm256(v, g1, b1, lane);
        warp_layernorm256(v, g2, b2, lane);
        store8_split(out, off, v);
    }
}

template <bool F32_IN>
__global__ void __launch_bounds__(256) layernorm256_kernel(const CSplit16 x, const float* __restrict__ x_f32,
                                                           const float* __restrict__ gamma, const float* __restrict__ beta,
                                                           const Split16 out, int rows) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) pdl_launch_dependents();
    pdl_wait();
    if (warp >= rows) return;
    const size_t off = (size_t)warp * kDModel + lane * 8;
    float v[8];
    if constexpr (F32_IN) {
        const float4 a = __ldcg(reinterpret_cast<const float4*>(x_f32 + off));
        const float4 b = __ldcg(reinterpret_cast<const float4*>(x_f32 + off + 4));
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
        load8_split(x, off, v);
    }
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += v[j];
    const float mean = warp_sum(s) * (1.f / kDModel);
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) { v[j] -= mean; sq = fmaf(v[j], v[j], sq); }
    const float rstd = 1.f / sqrtf(warp_sum(sq) * (1.f / kDModel) + 1e-5f);
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + lane * 8)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + lane * 8 + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + lane * 8)), b1 = __ldg(reinterpret_cast<const float4*>(beta + lane * 8 + 4));
    const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = v[j] * rstd * g[j] + b[j];
    store8_split(out, off, v);
}

// position_encoding.py:41-45 with bases 1..64 on (x, y):
// channel 2(k-1)+a = sin(fp32(k*pi) * p_a), channel 128 + 2(k-1)+a = cos(...).  Accurate sincosf: |angle| <= 64*pi.
__global__ void __launch_bounds__(128) query_encode_kernel(const float* __restrict__ queries, const Split16 qpos, int rows) {
    const int row = blockIdx.x;
    if (threadIdx.x == 0) pdl_launch_dependents();
    pdl_wait();
    if (row >= rows) return;
    const int t = threadIdx.x;          // 0..127 = 2*(k-1) + axis
    const int k = (t >> 1) + 1;
    const float p = __ldg(queries + (size_t)row * 2 + (t & 1));
    const float kpi = (float)((double)k * 3.14159265358979323846);
    const float angle = __fmul_rn(kpi, p);
    float s, c;
    sincosf(angle, &s, &c);
    __half h, l;
    split_f16(s, h, l);
    qpos.hi[(size_t)row * kDModel + t] = h;
    qpos.lo[(size_t)row * kDModel + t] = l;
    split_f16(c, h, l);
    qpos.hi[(size_t)row * kDModel + 128 + t] = h;
    qpos.lo[(size_t)row * kDModel + 128 + t] = l;
}

__global__ void f32_to_split16_kernel(const float* __restrict__ in, const Split16 out, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        __half h, l;
        split_f16(in[i], h, l);
        out.hi[i] = h;
        out.lo[i] = l;
    }
}
__global__ void split16_to_f32_kernel(const CSplit16 in, float* __restrict__ out, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        out[i] = join_f16(in.hi[i], in.lo[i]);
}

int grid_for(size_t total, int block) {
    const size_t blocks = (total + block - 1) / block;
    return (int)(blocks < kNumSms * 16 ? (blocks ? blocks : 1) : kNumSms * 16);
}

}  // namespace

int launch_maxpool_3x3s2_nhwc(CSplit16 in, Split16 out, int N, int H, int W, int C, cudaStream_t s) {
    COTR_CHECK((C & 7) == 0 && (H & 1) == 0 && (W & 1) == 0, "maxpool: unsupported shape");
    const size_t total = (size_t)N * (H / 2) * (W / 2) * (C / 8);
    COTR_CHECK_CUDA(launch_kernel(maxpool_3x3s2_nhwc_kernel, dim3(grid_for(total, 256)), dim3(256), 0, s, in, out, N, H, W, C / 8));
    return 0;
}

int launch_layernorm(CSplit16 x, const float* gamma, const float* beta, Split16 out, int rows, cudaStream_t s) {
    if (rows <= 0) return 0;
    COTR_CHECK_CUDA(launch_kernel(layernorm256_kernel<false>, dim3((rows + 7) / 8), dim3(256), 0, s, x, (const float*)nullptr, gamma, beta, out, rows));
    return 0;
}

int launch_ln_partials(CSplit16 x, float2* part, int rows, cudaStream_t s) {
    if (rows <= 0) return 0;
    ln_partials_kernel<<<(rows + 7) / 8, 256, 0, s>>>(x, part, rows);
    COTR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_layernorm_twice(CSplit16 x, const float* g1, const float* b1, const float* g2, const float* b2, Split16 out, int rows, cudaStream_t s) {
    if (rows <= 0) return 0;
    COTR_CHECK_CUDA(launch_kernel(layernorm256_twice_kernel, dim3((rows + 7) / 8), dim3(256), 0, s, x, g1, b1, g2, b2, out, rows));
    return 0;
}

int launch_layernorm_f32(const float* x, const float* gamma, const float* beta, Split16 out, int rows, cudaStream_t s) {
    if (rows <= 0) return 0;
    COTR_CHECK_CUDA(launch_kernel(layernorm256_kernel<true>, dim3((rows + 7) / 8), dim3(256), 0, s, CSplit16{nullptr, nullptr}, x, gamma, beta, out, rows));
    return 0;
}

int launch_query_encode(const float* queries, Split16 qpos, int rows, cudaStream_t s) {
    if (rows <= 0) return 0;
    COTR_CHECK_CUDA(launch_kernel(query_encode_kernel, dim3(rows), dim3(128), 0, s, queries, qpos, rows));
    return 0;
}

int launch_stem_canvas(const float* img, bool halves, Split16 canvas, int n_img, cudaStream_t s) {
    if (n_img <= 0) return 0;
    const size_t img_elems = (size_t)3 * 256 * 256;
    const size_t pair_stride = 2 * img_elems, half_offset = halves ? 256 : img_elems;
    const int pitch = halves ? 512 : 256;
    COTR_CHECK_CUDA(launch_kernel(stem_canvas_kernel, dim3(grid_for((size_t)n_img * 256 * 256, 256)), dim3(256), 0, s, img, pair_stride,
                                  half_offset, pitch, canvas, n_img));
    return 0;
}

int launch_f32_to_split16(const float* in, Split16 out, size_t n, cudaStream_t s) {
    if (n == 0) return 0;
    f32_to_split16_kernel<<<grid_for(n, 256), 256, 0, s>>>(in, out, n);
    COTR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_split16_to_f32(CSplit16 in, float* out, size_t n, cudaStream_t s) {
    if (n == 0) return 0;
    split16_to_f32_kernel<<<grid_for(n, 256), 256, 0, s>>>(in, out, n);
    COTR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace cotr
