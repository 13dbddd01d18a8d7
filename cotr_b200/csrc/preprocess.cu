// Device-side replacement of the host work of RefinementTask.get_task (refinement_task.py:105-120): crop two square
// patches out of the uint8 source images, resize each to 256 x 256 with Pillow's antialiased bilinear filter
// (bit-exact: same 22-bit fixed-point coefficient tables, same two passes with uint8 rounding in between), lay them side
// by side and apply to_tensor + ImageNet normalisation -> (n,3,256,512) fp32 canvases ready for cotr_forward.
// The source images are uploaded once per engine call; per batch only n x 6 integers cross PCIe instead of 50 MB of
// fp32 canvases, and ~4 ms of single-threaded PIL work per task disappears from the host loop.
#include <algorithm>
#include <cmath>
#include <map>
#include <vector>

#include "common.cuh"

namespace cotr {

namespace {

constexpr int kOut = 256;
constexpr int kPrecisionBits = 32 - 8 - 2;

struct CoeffTable {
    int ksize = 0;
    int* bounds = nullptr;    // device [256][2]: first source index, tap count
    int* weights = nullptr;   // device [256][ksize]
};

}  // namespace

// libImaging/Resample.c precompute_coeffs + normalize_coeffs_8bpc for the bilinear filter (support 1.0), box = the whole
// input, any output size.  Plain double arithmetic on the host (no FMA contraction on x86-64 baseline), so the integers
// match Pillow's.  Shared with the image resize of cotr_resize_image (resize.cu).
void host_coeffs(int in_size, int out_size, std::vector<int>& bounds, std::vector<int>& weights, int& ksize) {
    const double scale = (double)((float)in_size - 0.0f) / out_size;
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = 1.0 * filterscale;
    ksize = (int)std::ceil(support) * 2 + 1;
    bounds.assign((size_t)out_size * 2, 0);
    weights.assign((size_t)out_size * ksize, 0);
    std::vector<double> k(ksize);
    const double ss = 1.0 / filterscale;
    for (int xx = 0; xx < out_size; ++xx) {
        const double center = 0.0 + (xx + 0.5) * scale;
        double ww = 0.0;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in_size) xmax = in_size;
        xmax -= xmin;
        for (int x = 0; x < xmax; ++x) {
            double w = (x + xmin - center + 0.5) * ss;
            if (w < 0.0) w = -w;
            w = w < 1.0 ? 1.0 - w : 0.0;
            k[x] = w;
            ww += w;
        }
        for (int x = 0; x < xmax; ++x)
            if (ww != 0.0) k[x] /= ww;
        for (int x = 0; x < ksize; ++x) {
            const double v = x < xmax ? k[x] : 0.0;
            weights[(size_t)xx * ksize + x] = v < 0 ? (int)(-0.5 + v * (1 << kPrecisionBits)) : (int)(0.5 + v * (1 << kPrecisionBits));
        }
        bounds[(size_t)xx * 2] = xmin;
        bounds[(size_t)xx * 2 + 1] = xmax;
    }
}

namespace {

__device__ __forceinline__ unsigned char clip8(int v) {
    v >>= kPrecisionBits;
    return (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// horizontal pass: tmp[side][row][xx][c] for every row of the crop
__global__ void __launch_bounds__(256) resize_h_kernel(const CropSide* __restrict__ sides, unsigned char* __restrict__ tmp) {
    const CropSide s = sides[blockIdx.y];
    if (s.size == kOut) return;                                 // Pillow skips both passes when nothing changes
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int row = idx >> 8, xx = idx & 255;
    if (row >= s.size) return;
    const int x0 = s.bounds[xx * 2], n = s.bounds[xx * 2 + 1];
    const int* w = s.weights + (size_t)xx * s.ksize;
    const unsigned char* src = s.img + ((size_t)(s.y + row) * s.img_w + s.x + x0) * 3;
    int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
    for (int x = 0; x < n; ++x) {
        const int k = w[x];
        a0 += src[3 * x] * k;
        a1 += src[3 * x + 1] * k;
        a2 += src[3 * x + 2] * k;
    }
    unsigned char* dst = tmp + s.tmp_offset + ((size_t)row * kOut + xx) * 3;
    dst[0] = clip8(a0); dst[1] = clip8(a1); dst[2] = clip8(a2);
}

// vertical pass + to_tensor (/255) + normalize ((v - mean) / std), written into the canvas half of this side
__global__ void __launch_bounds__(256) resize_v_normalize_kernel(const CropSide* __restrict__ sides, const unsigned char* __restrict__ tmp,
                                                                 float* __restrict__ canvas) {
    const int side = blockIdx.y;
    const CropSide s = sides[side];
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int yy = idx >> 8, xx = idx & 255;
    unsigned char px[3];
    if (s.size == kOut) {
        const unsigned char* src = s.img + ((size_t)(s.y + yy) * s.img_w + s.x + xx) * 3;
        px[0] = src[0]; px[1] = src[1]; px[2] = src[2];
    } else {
        const int y0 = s.bounds[yy * 2], n = s.bounds[yy * 2 + 1];
        const int* w = s.weights + (size_t)yy * s.ksize;
        const unsigned char* src = tmp + s.tmp_offset + ((size_t)y0 * kOut + xx) * 3;
        int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
        for (int y = 0; y < n; ++y) {
            const int k = w[y];
            a0 += src[(size_t)y * kOut * 3] * k;
            a1 += src[(size_t)y * kOut * 3 + 1] * k;
            a2 += src[(size_t)y * kOut * 3 + 2] * k;
        }
        px[0] = clip8(a0); px[1] = clip8(a1); px[2] = clip8(a2);
    }
    // torchvision: to_tensor = uint8 -> float32 / 255; normalize = (t - mean) / std, all in float32
    const float mean[3] = {0.485f, 0.456f, 0.406f};
    const float stdv[3] = {0.229f, 0.224f, 0.225f};
    const int task = side >> 1, half = side & 1;
    float* out = canvas + (size_t)task * 3 * kOut * 2 * kOut + (size_t)yy * 2 * kOut + half * kOut + xx;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float v = __fdiv_rn((float)px[c], 255.0f);
        out[(size_t)c * kOut * 2 * kOut] = __fdiv_rn(__fsub_rn(v, mean[c]), stdv[c]);
    }
}

}  // namespace

struct Preprocessor {
    std::map<int, CoeffTable> tables;
    CropSide* sides_dev = nullptr;
    int sides_cap = 0;
    unsigned char* tmp = nullptr;
    size_t tmp_cap = 0;
    std::vector<CropSide> sides_host;
};

Preprocessor* preprocessor_create() { return new Preprocessor(); }

void preprocessor_destroy(Preprocessor* p) {
    if (!p) return;
    for (auto& kv : p->tables) { cudaFree(kv.second.bounds); cudaFree(kv.second.weights); }
    if (p->sides_dev) cudaFree(p->sides_dev);
    if (p->tmp) cudaFree(p->tmp);
    delete p;
}

static int get_table(Preprocessor* p, int size, CoeffTable* out) {
    auto it = p->tables.find(size);
    if (it == p->tables.end()) {
        std::vector<int> b, w;
        CoeffTable t;
        host_coeffs(size, kOut, b, w, t.ksize);
        COTR_CHECK_CUDA(cudaMalloc((void**)&t.bounds, b.size() * sizeof(int)));
        COTR_CHECK_CUDA(cudaMalloc((void**)&t.weights, w.size() * sizeof(int)));
        COTR_CHECK_CUDA(cudaMemcpy(t.bounds, b.data(), b.size() * sizeof(int), cudaMemcpyHostToDevice));
        COTR_CHECK_CUDA(cudaMemcpy(t.weights, w.data(), w.size() * sizeof(int), cudaMemcpyHostToDevice));
        it = p->tables.emplace(size, t).first;
    }
    *out = it->second;
    return 0;
}

// rects: n x 6 host ints [x_from, y_from, size_from, x_to, y_to, size_to]; canvas: (n,3,256,512) fp32 device.
int preprocess_launch(Preprocessor* p, const unsigned char* img_from, int hf, int wf, const unsigned char* img_to, int ht, int wt,
                      const int* rects, int n, float* canvas, cudaStream_t s) {
    COTR_CHECK(p && img_from && img_to && rects && canvas && n > 0, "cotr_preprocess: bad arguments");
    p->sides_host.resize((size_t)n * 2);
    size_t tmp_bytes = 0;
    int max_size = kOut;
    for (int i = 0; i < n; ++i) {
        for (int side = 0; side < 2; ++side) {
            const int* r = rects + i * 6 + side * 3;
            const int H = side ? ht : hf, W = side ? wt : wf;
            COTR_CHECK(r[2] >= 2 && r[0] >= 0 && r[1] >= 0 && r[0] + r[2] <= W && r[1] + r[2] <= H,
                       "cotr_preprocess: crop %d/%d (x=%d y=%d size=%d) leaves the %dx%d image", i, side, r[0], r[1], r[2], W, H);
            CropSide& c = p->sides_host[(size_t)i * 2 + side];
            c.img = side ? img_to : img_from;
            c.img_w = W;
            c.x = r[0]; c.y = r[1]; c.size = r[2];
            CoeffTable t;
            if (get_table(p, r[2], &t)) return 1;
            c.ksize = t.ksize; c.bounds = t.bounds; c.weights = t.weights;
            c.tmp_offset = tmp_bytes;
            if (r[2] != kOut) tmp_bytes += (size_t)r[2] * kOut * 3;
            if (r[2] > max_size) max_size = r[2];
        }
    }
    if (2 * n > p->sides_cap) {
        COTR_CHECK_CUDA(cudaDeviceSynchronize());
        if (p->sides_dev) cudaFree(p->sides_dev);
        COTR_CHECK_CUDA(cudaMalloc((void**)&p->sides_dev, (size_t)2 * n * sizeof(CropSide)));
        p->sides_cap = 2 * n;
    }
    if (tmp_bytes > p->tmp_cap) {
        COTR_CHECK_CUDA(cudaDeviceSynchronize());
        if (p->tmp) cudaFree(p->tmp);
        COTR_CHECK_CUDA(cudaMalloc((void**)&p->tmp, tmp_bytes));
        p->tmp_cap = tmp_bytes;
    }
    // the table is small (a few KB): a synchronous-with-respect-to-host staged copy keeps sides_host reusable
    COTR_CHECK_CUDA(cudaMemcpyAsync(p->sides_dev, p->sides_host.data(), (size_t)2 * n * sizeof(CropSide), cudaMemcpyHostToDevice, s));
    COTR_CHECK_CUDA(cudaStreamSynchronize(s));
    const dim3 grid_h((unsigned)(((size_t)max_size * kOut + 255) / 256), (unsigned)(2 * n));
    resize_h_kernel<<<grid_h, 256, 0, s>>>(p->sides_dev, p->tmp);
    COTR_CHECK_CUDA(cudaGetLastError());
    const dim3 grid_v(kOut * kOut / 256, (unsigned)(2 * n));
    resize_v_normalize_kernel<<<grid_v, 256, 0, s>>>(p->sides_dev, p->tmp, canvas);
    COTR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int preprocess_coeffs(Preprocessor* p, int size, CropSide* side) {
    CoeffTable t;
    if (get_table(p, size, &t)) return 1;
    side->size = size;
    side->ksize = t.ksize; side->bounds = t.bounds; side->weights = t.weights;
    return 0;
}

int launch_resize_h(const CropSide* sides, int n_sides, int max_size, unsigned char* tmp, cudaStream_t s) {
    const dim3 grid_h((unsigned)(((size_t)std::max(max_size, kOut) * kOut + 255) / 256), (unsigned)n_sides);
    resize_h_kernel<<<grid_h, 256, 0, s>>>(sides, tmp);
    COTR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_resize_v(const CropSide* sides, int n_sides, const unsigned char* tmp, float* canvas, cudaStream_t s) {
    const dim3 grid_v(kOut * kOut / 256, (unsigned)n_sides);
    resize_v_normalize_kernel<<<grid_v, 256, 0, s>>>(sides, tmp, canvas);
    COTR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace cotr
