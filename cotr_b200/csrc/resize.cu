// Whole-image resizes with Pillow's bilinear filter, bit for bit (cotr_resize_image / cotr_resize_maps,
// include/cotr_b200.h).  They move the stretch of SparseEngine's 'stretching' mode to the device:
//   * uint8 HWC RGB images, as PIL.Image.fromarray(img).resize((W', H'), BILINEAR) (stretch_to_square_np): the 22-bit
//     fixed-point tables of preprocess.cu at any output size, horizontal pass first, uint8 rounding and clipping in
//     between, then the vertical pass (libImaging/Resample.c ImagingResampleHorizontal_8bpc / Vertical_8bpc).
//   * fp32 HWC maps of 1 .. 3 channels, as utils.float_image_resize (Pillow mode 'F', channel by channel): double
//     coefficients, double accumulation with separate multiply and add, float32 store after each pass (the restatement of
//     engine_ops.cu's flow merge, here without the affine and the merge).
// Like Pillow (need_horizontal / need_vertical in ImagingResampleInner) an axis whose size does not change is not
// resampled: its identity pass would not be harmless, since the 0.0 weight of the neighbour turns a NaN or an infinity
// there into NaN.  With neither axis changing the output is a copy.
#include <map>
#include <utility>
#include <vector>

#include "common.cuh"

namespace cotr {

namespace {

constexpr int kPrecisionBits = 32 - 8 - 2;
constexpr int kThreads = 256;

struct Table {
    int ksize = 0;
    int* bounds = nullptr;
    void* weights = nullptr;
};

__device__ __forceinline__ unsigned char clip8(int v) {
    v >>= kPrecisionBits;
    return (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// One output pixel per thread.  Horizontal: source row r, output column j (taps along the row, stride c); vertical:
// output row r, column j (taps down the column, stride row_len * c).  `row_len` is the source row length in pixels.
template <bool kVertical>
__global__ void __launch_bounds__(kThreads) image_pass_kernel(const unsigned char* __restrict__ src, int row_len, int rows, int cols,
                                                              const int* __restrict__ bounds, const int* __restrict__ weights, int ksize,
                                                              unsigned char* __restrict__ dst) {
    const int64_t n = (int64_t)rows * cols;
    for (int64_t idx = blockIdx.x * (int64_t)kThreads + threadIdx.x; idx < n; idx += (int64_t)gridDim.x * kThreads) {
        const int r = (int)(idx / cols), j = (int)(idx - (int64_t)r * cols);
        const int o = kVertical ? r : j;
        const int first = bounds[2 * o], taps = bounds[2 * o + 1];
        const int* k = weights + (size_t)o * ksize;
        const int64_t step = kVertical ? (int64_t)row_len * 3 : 3;
        const unsigned char* p = kVertical ? src + ((int64_t)first * row_len + j) * 3 : src + ((int64_t)r * row_len + first) * 3;
        int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
        for (int t = 0; t < taps; ++t, p += step) {
            const int w = k[t];
            a0 += p[0] * w;
            a1 += p[1] * w;
            a2 += p[2] * w;
        }
        unsigned char* q = dst + idx * 3;
        q[0] = clip8(a0); q[1] = clip8(a1); q[2] = clip8(a2);
    }
}

template <bool kVertical>
__global__ void __launch_bounds__(kThreads) map_pass_kernel(const float* __restrict__ src, int row_len, int rows, int cols, int c,
                                                            const int* __restrict__ bounds, const double* __restrict__ weights, int ksize,
                                                            float* __restrict__ dst) {
    const int64_t n = (int64_t)rows * cols;
    for (int64_t idx = blockIdx.x * (int64_t)kThreads + threadIdx.x; idx < n; idx += (int64_t)gridDim.x * kThreads) {
        const int r = (int)(idx / cols), j = (int)(idx - (int64_t)r * cols);
        const int o = kVertical ? r : j;
        const int first = bounds[2 * o], taps = bounds[2 * o + 1];
        const double* k = weights + (size_t)o * ksize;
        const int64_t step = kVertical ? (int64_t)row_len * c : c;
        const float* p = kVertical ? src + ((int64_t)first * row_len + j) * c : src + ((int64_t)r * row_len + first) * c;
        double s0 = 0.0, s1 = 0.0, s2 = 0.0;
        for (int t = 0; t < taps; ++t, p += step) {
            const double w = k[t];
            s0 = __dadd_rn(s0, __dmul_rn((double)p[0], w));
            if (c > 1) s1 = __dadd_rn(s1, __dmul_rn((double)p[1], w));
            if (c > 2) s2 = __dadd_rn(s2, __dmul_rn((double)p[2], w));
        }
        float* q = dst + idx * c;
        q[0] = (float)s0;
        if (c > 1) q[1] = (float)s1;
        if (c > 2) q[2] = (float)s2;
    }
}

int grid_for(int64_t n) {
    const int64_t blocks = (n + kThreads - 1) / kThreads;
    return (int)(blocks < (int64_t)kNumSms * 16 ? blocks : (int64_t)kNumSms * 16);
}

}  // namespace

struct Resizer {
    std::map<std::pair<int, int>, Table> u8_tables, f32_tables;     // keyed by (input size, output size)
    void* tmp = nullptr;
    size_t tmp_cap = 0;
};

Resizer* resizer_create() { return new Resizer(); }

void resizer_destroy(Resizer* r) {
    if (!r) return;
    for (auto* tabs : {&r->u8_tables, &r->f32_tables})
        for (auto& kv : *tabs) { cudaFree(kv.second.bounds); cudaFree(kv.second.weights); }
    if (r->tmp) cudaFree(r->tmp);
    delete r;
}

// The table of one axis, built and uploaded on first use (a synchronous copy), then cached.
static int get_axis(Resizer* r, int u8, int in_size, int out_size, ResizeAxis* out) {
    auto& tabs = u8 ? r->u8_tables : r->f32_tables;
    const auto key = std::make_pair(in_size, out_size);
    auto it = tabs.find(key);
    if (it == tabs.end()) {
        std::vector<int> b, wi;
        std::vector<double> wd;
        Table t;
        if (u8) host_coeffs(in_size, out_size, b, wi, t.ksize);
        else host_float_coeffs(in_size, out_size, b, wd, t.ksize);
        const size_t wbytes = u8 ? wi.size() * sizeof(int) : wd.size() * sizeof(double);
        COTR_CHECK_CUDA(cudaMalloc((void**)&t.bounds, b.size() * sizeof(int)));
        if (cudaMalloc(&t.weights, wbytes) != cudaSuccess) {
            cudaFree(t.bounds);
            COTR_CHECK(false, "cotr_resize: cannot allocate a %d -> %d coefficient table", in_size, out_size);
        }
        COTR_CHECK_CUDA(cudaMemcpy(t.bounds, b.data(), b.size() * sizeof(int), cudaMemcpyHostToDevice));
        COTR_CHECK_CUDA(cudaMemcpy(t.weights, u8 ? (const void*)wi.data() : (const void*)wd.data(), wbytes, cudaMemcpyHostToDevice));
        it = tabs.emplace(key, t).first;
    }
    out->ksize = it->second.ksize;
    out->bounds = it->second.bounds;
    out->weights = it->second.weights;
    return 0;
}

int resize_plan(Resizer* r, int u8, int h, int w, int c, int oh, int ow, ResizePlan* p) {
    *p = ResizePlan();
    p->u8 = u8; p->h = h; p->w = w; p->c = c; p->oh = oh; p->ow = ow;
    p->need_h = ow != w;
    p->need_v = oh != h;
    if (p->need_h && get_axis(r, u8, w, ow, &p->horiz)) return 1;
    if (p->need_v && get_axis(r, u8, h, oh, &p->vert)) return 1;
    if (p->need_h && p->need_v) {
        const size_t need = (size_t)h * ow * c * (u8 ? 1 : sizeof(float));
        if (need > r->tmp_cap) {
            COTR_CHECK_CUDA(cudaDeviceSynchronize());
            if (r->tmp) cudaFree(r->tmp);
            r->tmp = nullptr;
            r->tmp_cap = 0;
            COTR_CHECK_CUDA(cudaMalloc(&r->tmp, need));
            r->tmp_cap = need;
        }
        p->tmp = r->tmp;
    }
    return 0;
}

int resize_pass(const ResizePlan& p, int pass, const void* src, void* dst, cudaStream_t s) {
    const ResizeAxis& a = pass ? p.vert : p.horiz;
    const int rows = pass ? p.oh : p.h, cols = p.ow, row_len = pass ? p.ow : p.w;
    const int grid = grid_for((int64_t)rows * cols);
    if (p.u8) {
        const unsigned char* in = static_cast<const unsigned char*>(src);
        unsigned char* out = static_cast<unsigned char*>(dst);
        const int* k = static_cast<const int*>(a.weights);
        if (pass) image_pass_kernel<true><<<grid, kThreads, 0, s>>>(in, row_len, rows, cols, a.bounds, k, a.ksize, out);
        else image_pass_kernel<false><<<grid, kThreads, 0, s>>>(in, row_len, rows, cols, a.bounds, k, a.ksize, out);
    } else {
        const float* in = static_cast<const float*>(src);
        float* out = static_cast<float*>(dst);
        const double* k = static_cast<const double*>(a.weights);
        if (pass) map_pass_kernel<true><<<grid, kThreads, 0, s>>>(in, row_len, rows, cols, p.c, a.bounds, k, a.ksize, out);
        else map_pass_kernel<false><<<grid, kThreads, 0, s>>>(in, row_len, rows, cols, p.c, a.bounds, k, a.ksize, out);
    }
    COTR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace cotr
