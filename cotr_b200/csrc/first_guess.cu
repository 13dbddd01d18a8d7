// First guesses of the forced zoom-in (cotr_dense_first_guess, include/cotr_b200.h): the `force` branch of
// SparseEngine.gen_tasks (COTR/inference/sparse_engine.py:224-258) on the merged dense maps of one direction, without
// bringing the maps to the host.
//   * the co-visible area counts: pixels whose cycle confidence, widened to fp64 as the reference's float64 arrays hold
//     it, is below THRESHOLD_AREA = 0.02 (fp64; float32(0.02) lies below 0.02, so an fp32 compare would count it).
//     NaN compares false.  Integer atomics: the counts do not depend on the schedule.
//   * per keypoint the dense prediction at the clipped, truncated pixel, mapped to pixels of the other image:
//     (double(flow) * 0.5 + 0.5) * (W_to, H_to) with separate multiply and add (no contraction).
// cotr_dense_first_guess_f32 is the same branch on float32 maps, which is what 'stretching' mode hands gen_tasks when
// an image had to be stretched (float_image_resize returns float32): numpy then compares `conf < 0.02` in float32, so
// float32(0.02) itself is not counted, and computes `corr * 0.5 + 0.5` in float32 before the multiply by the int64
// image size widens it to fp64.
#include <algorithm>

#include "../../include/cotr_b200.h"
#include "common.cuh"

namespace cotr {
namespace {

constexpr double kThresholdArea = 0.02;   // inference_helper.THRESHOLD_AREA
constexpr float kThresholdAreaF32 = 0.02f;
constexpr int kThreads = 256;

struct FirstGuessArgs {
    const float* flow;          // (h_from, w_from, 2)
    const float* conf_from;     // (h_from, w_from)
    const float* conf_to;       // (h_to, w_to)
    const void* kpts;           // (n, 2) float32 or float64 (x, y)
    int64_t px_from, px_to;
    int h_from, w_from, h_to, w_to, n, f32;
    int f32_maps;               // float32 semantics of the maps (cotr_dense_first_guess_f32)
    double* loc_to;             // (n, 2)
    unsigned long long* counts; // [from, to], zeroed before the launch
};

__global__ void __launch_bounds__(kThreads) dense_first_guess_kernel(const FirstGuessArgs a) {
    const int64_t tid = blockIdx.x * (int64_t)kThreads + threadIdx.x, stride = (int64_t)gridDim.x * kThreads;
    for (int64_t i = tid; i < a.n; i += stride) {
        // pos = (clip(y, 0, H-1), clip(x, 0, W-1)) in the keypoint's dtype, then int(): the bounds are exact in both
        // dtypes and clipping rounds nothing, so the truncation sees the value numpy sees (finite keypoints only)
        int r, c;
        if (a.f32) {
            const float* k = static_cast<const float*>(a.kpts) + 2 * i;
            r = (int)fminf(fmaxf(k[1], 0.f), (float)(a.h_from - 1));
            c = (int)fminf(fmaxf(k[0], 0.f), (float)(a.w_from - 1));
        } else {
            const double* k = static_cast<const double*>(a.kpts) + 2 * i;
            r = (int)fmin(fmax(k[1], 0.0), (double)(a.h_from - 1));
            c = (int)fmin(fmax(k[0], 0.0), (double)(a.w_from - 1));
        }
        const float* f = a.flow + ((int64_t)r * a.w_from + c) * 2;
        if (a.f32_maps) {
            a.loc_to[2 * i] = __dmul_rn((double)__fadd_rn(__fmul_rn(f[0], 0.5f), 0.5f), (double)a.w_to);
            a.loc_to[2 * i + 1] = __dmul_rn((double)__fadd_rn(__fmul_rn(f[1], 0.5f), 0.5f), (double)a.h_to);
        } else {
            a.loc_to[2 * i] = __dmul_rn(__dadd_rn(__dmul_rn((double)f[0], 0.5), 0.5), (double)a.w_to);
            a.loc_to[2 * i + 1] = __dmul_rn(__dadd_rn(__dmul_rn((double)f[1], 0.5), 0.5), (double)a.h_to);
        }
    }
    unsigned int below_from = 0, below_to = 0;      // at most ceil(65536^2 / (132 * 8 * 256)) per thread
    if (a.f32_maps) {
        for (int64_t p = tid; p < a.px_from; p += stride) below_from += a.conf_from[p] < kThresholdAreaF32 ? 1u : 0u;
        for (int64_t p = tid; p < a.px_to; p += stride) below_to += a.conf_to[p] < kThresholdAreaF32 ? 1u : 0u;
    } else {
        for (int64_t p = tid; p < a.px_from; p += stride) below_from += (double)a.conf_from[p] < kThresholdArea ? 1u : 0u;
        for (int64_t p = tid; p < a.px_to; p += stride) below_to += (double)a.conf_to[p] < kThresholdArea ? 1u : 0u;
    }
    below_from = __reduce_add_sync(0xffffffffu, below_from);
    below_to = __reduce_add_sync(0xffffffffu, below_to);
    if ((threadIdx.x & 31) == 0) {
        if (below_from) atomicAdd(a.counts, (unsigned long long)below_from);
        if (below_to) atomicAdd(a.counts + 1, (unsigned long long)below_to);
    }
}

int first_guess_impl(const char* fn, int f32_maps, int device, const float* flow_dev, const float* conf_from_dev, int h_from, int w_from,
                     const float* conf_to_dev, int h_to, int w_to, const void* kpts_dev, int kpt_is_f32, int n, double* loc_to_dev,
                     int64_t* counts_dev, void* cuda_stream) {
    COTR_CHECK(h_from >= 1 && w_from >= 1 && h_to >= 1 && w_to >= 1 && h_from <= 65536 && w_from <= 65536 && h_to <= 65536 && w_to <= 65536,
               "%s: image sizes %d x %d and %d x %d must lie in 1 .. 65536", fn, h_from, w_from, h_to, w_to);
    COTR_CHECK(n >= 0, "%s: n = %d keypoints", fn, n);
    COTR_CHECK(kpt_is_f32 == 0 || kpt_is_f32 == 1, "%s: kpt_is_f32 must be 0 or 1, got %d", fn, kpt_is_f32);
    COTR_CHECK(flow_dev && conf_from_dev && conf_to_dev && counts_dev, "%s: null flow_dev, conf_from_dev, conf_to_dev or counts_dev", fn);
    COTR_CHECK(n == 0 || (kpts_dev && loc_to_dev), "%s: null kpts_dev or loc_to_dev with %d keypoints", fn, n);
    COTR_CHECK(((uintptr_t)flow_dev & 3) == 0 && ((uintptr_t)conf_from_dev & 3) == 0 && ((uintptr_t)conf_to_dev & 3) == 0,
               "%s: flow_dev, conf_from_dev or conf_to_dev is not 4-byte aligned", fn);
    COTR_CHECK(((uintptr_t)kpts_dev & (kpt_is_f32 ? 3 : 7)) == 0, "%s: kpts_dev is not %d-byte aligned", fn, kpt_is_f32 ? 4 : 8);
    COTR_CHECK(((uintptr_t)loc_to_dev & 7) == 0 && ((uintptr_t)counts_dev & 7) == 0, "%s: loc_to_dev or counts_dev is not 8-byte aligned", fn);
    COTR_CHECK_CUDA(cudaSetDevice(device));
    cudaStream_t s = (cudaStream_t)cuda_stream;
    FirstGuessArgs a;
    a.flow = flow_dev; a.conf_from = conf_from_dev; a.conf_to = conf_to_dev; a.kpts = kpts_dev;
    a.px_from = (int64_t)h_from * w_from; a.px_to = (int64_t)h_to * w_to;
    a.h_from = h_from; a.w_from = w_from; a.h_to = h_to; a.w_to = w_to; a.n = n; a.f32 = kpt_is_f32;
    a.f32_maps = f32_maps;
    a.loc_to = loc_to_dev;
    a.counts = reinterpret_cast<unsigned long long*>(counts_dev);
    const int64_t work = std::max<int64_t>(std::max(a.px_from, a.px_to), n);
    const int grid = (int)std::min<int64_t>((work + kThreads - 1) / kThreads, (int64_t)kNumSms * 8);
    COTR_CHECK_CUDA(cudaMemsetAsync(counts_dev, 0, 2 * sizeof(int64_t), s));
    dense_first_guess_kernel<<<grid, kThreads, 0, s>>>(a);
    COTR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace
}  // namespace cotr

int cotr_dense_first_guess(int device, const float* flow_dev, const float* conf_from_dev, int h_from, int w_from, const float* conf_to_dev,
                           int h_to, int w_to, const void* kpts_dev, int kpt_is_f32, int n, double* loc_to_dev, int64_t* counts_dev,
                           void* cuda_stream) {
    return cotr::first_guess_impl("cotr_dense_first_guess", 0, device, flow_dev, conf_from_dev, h_from, w_from, conf_to_dev, h_to, w_to,
                                  kpts_dev, kpt_is_f32, n, loc_to_dev, counts_dev, cuda_stream);
}

int cotr_dense_first_guess_f32(int device, const float* flow_dev, const float* conf_from_dev, int h_from, int w_from,
                               const float* conf_to_dev, int h_to, int w_to, const void* kpts_dev, int kpt_is_f32, int n, double* loc_to_dev,
                               int64_t* counts_dev, void* cuda_stream) {
    return cotr::first_guess_impl("cotr_dense_first_guess_f32", 1, device, flow_dev, conf_from_dev, h_from, w_from, conf_to_dev, h_to, w_to,
                                  kpts_dev, kpt_is_f32, n, loc_to_dev, counts_dev, cuda_stream);
}
