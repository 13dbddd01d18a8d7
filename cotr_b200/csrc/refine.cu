// The zoom-in walks of cotr_refine and cotr_refine_grouped (include/cotr_b200.h): the per-task arithmetic of
// RefinementTask with converge_iters = 1 (refinement_task.py, inference_helper.py:79-96) - crop geometry, canvas query,
// scale_to_loc and conclude() - as numpy / Python evaluate it, bit for bit.  The functions below are __host__ __device__:
// the kernels use them with explicit round-to-nearest intrinsics (no contraction), and cotr_test_refine_math runs the
// same code on the host (plain IEEE double / float arithmetic, no FMA on the x86-64 baseline) so that it can be checked
// against Python.
#include <cmath>

#include "../../include/cotr_b200.h"
#include "common.cuh"

namespace cotr {
namespace {

__host__ __device__ inline double d_add(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ inline double d_sub(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
__host__ __device__ inline double d_mul(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ inline double d_div(double a, double b) {
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}
__host__ __device__ inline double d_sqrt(double a) {
#ifdef __CUDA_ARCH__
    return __dsqrt_rn(a);
#else
    return std::sqrt(a);
#endif
}
__host__ __device__ inline float f_sub(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}
__host__ __device__ inline float f_mul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ inline float to_f32(double a) {
#ifdef __CUDA_ARCH__
    return __double2float_rn(a);
#else
    return (float)a;
#endif
}

// Top (or left) corner of a crop of side `size` around `pos` in an image of extent `limit` (get_patch_centered_at):
// int(pos - size // 2) truncates toward zero, then max(., 0) and the shift back inside.  Python raises on NaN and
// +-inf; here they are clamped explicitly (NaN and -inf to 0, +inf to limit - size) and flagged.  A finite position
// is clamped in fp64 before any conversion, so 1e300 lands at limit - size as it does in Python.
__host__ __device__ inline int patch_corner(double pos, int size, int limit, int* flag) {
    const double d = d_sub(pos, (double)(size / 2));
    if (d != d) { *flag = 1; return 0; }
    if (d == INFINITY || d == -INFINITY) { *flag = 1; return d < 0 ? 0 : limit - size; }
    const double t = trunc(d);
    if (t < 0.0) return 0;
    if (t > (double)(limit - size)) return limit - size;
    return (int)t;
}

// Canvas query of the source point: x over the two-patch-wide canvas, both divisions in fp64, rounded once to fp32.
__host__ __device__ inline float2 query_in(double lx, double ly, int px, int py, int size) {
    return make_float2(to_f32(d_div(d_sub(lx, (double)px), (double)(2 * size))), to_f32(d_div(d_sub(ly, (double)py), (double)size)));
}

// scale_to_loc: raw[0] = (raw[0] - 0.5) * 2 in fp32 (a float32 array), then the fp64 products and sums with the ints.
__host__ __device__ inline double2 scale_to_loc(float p, float q, int px, int py, int size) {
    const float xs = f_mul(f_sub(p, 0.5f), 2.0f);
    return make_double2(d_add(d_mul((double)xs, (double)size), (double)px), d_add(d_mul((double)q, (double)size), (double)py));
}

// conclude() without force: max(np.std(history, axis=0)) >= thr is "bad".  np.std of n <= 8 rows sums sequentially;
// Python's max keeps the first column unless the second is strictly greater (so a NaN first column wins).
__host__ __device__ inline bool conclude_good(const double* h, int n, double thr) {
    double s[2];
    for (int c = 0; c < 2; ++c) {
        double sum = h[c];
        for (int r = 1; r < n; ++r) sum = d_add(sum, h[2 * r + c]);
        const double mean = d_div(sum, (double)n);
        double x = d_sub(h[c], mean);
        double ss = d_mul(x, x);
        for (int r = 1; r < n; ++r) {
            x = d_sub(h[2 * r + c], mean);
            ss = d_add(ss, d_mul(x, x));
        }
        s[c] = d_sqrt(d_div(ss, (double)n));
    }
    const double mx = s[1] > s[0] ? s[1] : s[0];
    return !(mx >= thr);
}

__device__ inline unsigned long long status_key(const RefineLevel& lv, int code) {
    return ((unsigned long long)lv.chunk * 8 + (unsigned long long)lv.level) * 4 + (unsigned long long)code;
}

// ---- grouped walk (cotr_refine_grouped): FasterSparseEngine's squads at one level ----------------------------------

// Corner of a candidate's pilot box as FasterSparseEngine._pilot_boxes computes it: np.trunc(pos - size // 2) cast to
// int64, max(., 0), shifted back inside.  numpy's cast gives INT64_MIN on x86-64 for NaN, +-inf and |x| >= 2**63, which
// max(., 0) turns into 0; for those positions get_patch_centered_at's int() raises (NaN, inf) or is exact (huge finite
// values land at limit - size), so only the box follows numpy here.  A NaN or infinite position only matters in a box
// when its task becomes a pilot, and then the host loop raises at the pilot's crop anyway.
__device__ inline int box_corner(double pos, int size, int limit) {
    const double d = d_sub(pos, (double)(size / 2));
    if (!(fabs(trunc(d)) < 9223372036854775808.0)) return 0;
    int flag = 0;
    return patch_corner(pos, size, limit, &flag);
}

// Python's order of failure at a pilot's crops: get_patch_centered_at takes top (y) before left (x), and the "from"
// crop before the "to" crop.  1 = int(NaN) (ValueError), 2 = int(+-inf) (OverflowError), 0 = none.
__device__ inline int crop_failure(double x, double y, int prev) {
    if (prev) return prev;
    if (y != y) return 1;
    if (y == INFINITY || y == -INFINITY) return 2;
    if (x != x) return 1;
    if (x == INFINITY || x == -INFINITY) return 2;
    return 0;
}

// Per candidate i (task ids[i], list order): its end points [loc_from, location at this level], the central-half boxes
// of the crops it would impose as a pilot (form_squad's safe_box: centre +- size / 4, all exact in fp64) and the
// exception its crop would raise.
__global__ void __launch_bounds__(128) grouped_candidates_kernel(RefineLevel lv, const int32_t* __restrict__ ids,
                                                                 const double* __restrict__ loc_from, const double* __restrict__ history,
                                                                 double* __restrict__ pts, double* __restrict__ box,
                                                                 int32_t* __restrict__ fail) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= lv.count) return;
    const size_t t = (size_t)ids[i];
    const double* lf = loc_from + 2 * t;
    const double* lt = history + (t * (lv.levels + 1) + lv.level) * 2;
    double* p = pts + (size_t)i * 4;
    p[0] = lf[0]; p[1] = lf[1]; p[2] = lt[0]; p[3] = lt[1];
    const int fs = lv.from.size, ts = lv.to.size;
    const int corner[4] = {box_corner(lf[0], fs, lv.w_from), box_corner(lf[1], fs, lv.h_from),
                           box_corner(lt[0], ts, lv.w_to), box_corner(lt[1], ts, lv.h_to)};
    double* b = box + (size_t)i * 8;
#pragma unroll
    for (int side = 0; side < 2; ++side) {
        const double size = side ? ts : fs;
        const double half = d_mul(d_div(size, 2.0), 0.5);
        const double cx = d_add((double)corner[2 * side], d_div(size, 2.0)), cy = d_add((double)corner[2 * side + 1], d_div(size, 2.0));
        b[4 * side + 0] = d_sub(cx, half);
        b[4 * side + 1] = d_add(cx, half);
        b[4 * side + 2] = d_sub(cy, half);
        b[4 * side + 3] = d_add(cy, half);
    }
    fail[i] = crop_failure(lt[0], lt[1], crop_failure(lf[0], lf[1], 0));
}

// ---- one level of either walk: entry i is task lv.task0 + ids[i] in squad squad[i] at rank rank[i] -----------------
// cotr_refine's tasks are squads of one (ids = squad = 0 .. count-1, rank = 0, longest = 1, task0 = the chunk's first
// task); cotr_refine_grouped's are the candidates of one batch (task0 = 0, squad -1 for the ones left out).

// One CTA per squad: the pilot's crops (get_patch_centered_at) become CropSide 2s / 2s+1 and the rect of this level of
// every member (the pilot's two patches, as get_task_pilot submits them), and each member's canvas query is its own
// loc_from in the pilot's "from" patch, at row s * longest + rank (pilot first, then the members in list order).
// Non-finite pilot positions flag `status`; cotr_refine_grouped never gets there, since it stops at such a pilot.
__global__ void __launch_bounds__(256) refine_geometry_kernel(RefineLevel lv, const int32_t* __restrict__ ids,
                                                              const int32_t* __restrict__ squad, const int32_t* __restrict__ rank,
                                                              int n_squads, int longest, const double* __restrict__ loc_from,
                                                              const double* __restrict__ history, CropSide* __restrict__ sides,
                                                              int32_t* __restrict__ rects, float* __restrict__ queries,
                                                              unsigned long long* __restrict__ status) {
    __shared__ int s_rect[4];
    const int s = blockIdx.x;
    const int fs = lv.from.size, ts = lv.to.size;
    for (int i = threadIdx.x; i < lv.count; i += blockDim.x) {
        if (squad[i] != s || rank[i] != 0) continue;
        const size_t t = (size_t)lv.task0 + ids[i];
        const double* lf = loc_from + 2 * t;
        const double* lt = history + (t * (lv.levels + 1) + lv.level) * 2;
        int flag = 0;
        CropSide a = lv.from, b = lv.to;
        a.x = patch_corner(lf[0], fs, lv.w_from, &flag);
        a.y = patch_corner(lf[1], fs, lv.h_from, &flag);
        b.x = patch_corner(lt[0], ts, lv.w_to, &flag);
        b.y = patch_corner(lt[1], ts, lv.h_to, &flag);
        // horizontal-pass bytes: the level's "from" crops first, then its "to" crops
        a.tmp_offset = (size_t)s * fs * 256 * 3;
        b.tmp_offset = (size_t)n_squads * fs * 256 * 3 + (size_t)s * ts * 256 * 3;
        sides[2 * s] = a;
        sides[2 * s + 1] = b;
        s_rect[0] = a.x; s_rect[1] = a.y; s_rect[2] = b.x; s_rect[3] = b.y;
        if (flag) atomicMin(status, status_key(lv, 2));
    }
    __syncthreads();
    const int ax = s_rect[0], ay = s_rect[1], bx = s_rect[2], by = s_rect[3];
    for (int i = threadIdx.x; i < lv.count; i += blockDim.x) {
        if (squad[i] != s) continue;
        const size_t t = (size_t)lv.task0 + ids[i];
        int32_t* r = rects + (t * lv.levels + lv.level) * 6;
        r[0] = ax; r[1] = ay; r[2] = fs; r[3] = bx; r[4] = by; r[5] = ts;
        const float2 q = query_in(loc_from[2 * t], loc_from[2 * t + 1], ax, ay, fs);
        float* out = queries + ((size_t)s * longest + rank[i]) * 2;
        out[0] = q.x;
        out[1] = q.y;
    }
}

// RefinementTask.step for every member: scale_to_loc with its pilot's "to" patch into history row level + 1; at the
// last level conclude(), the good flag and *good_count += 1.  A NaN prediction flags `status`.
__global__ void __launch_bounds__(128) refine_step_kernel(RefineLevel lv, const int32_t* __restrict__ ids, const int32_t* __restrict__ squad,
                                                          const int32_t* __restrict__ rank, int longest, const float* __restrict__ pred,
                                                          const int32_t* __restrict__ rects, double* __restrict__ history,
                                                          int32_t* __restrict__ good, int32_t* __restrict__ good_count,
                                                          unsigned long long* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= lv.count || squad[i] < 0) return;
    const size_t t = (size_t)lv.task0 + ids[i];
    const float* p = pred + ((size_t)squad[i] * longest + rank[i]) * 2;
    if (p[0] != p[0] || p[1] != p[1]) atomicMin(status, status_key(lv, 1));
    const int32_t* r = rects + (t * lv.levels + lv.level) * 6;
    const double2 loc = scale_to_loc(p[0], p[1], r[3], r[4], r[5]);
    double* h = history + t * (lv.levels + 1) * 2;
    h[2 * (lv.level + 1)] = loc.x;
    h[2 * (lv.level + 1) + 1] = loc.y;
    if (lv.level == lv.levels - 1) {
        const bool g = conclude_good(h, lv.levels + 1, lv.thr);
        good[t] = g ? 1 : 0;
        if (g) atomicAdd(good_count, 1);
    }
}

constexpr int kRefineThreads = 128;

}  // namespace

int refine_crop_size(int h, int w, double scale) {
    // Python: min(max(scale, 0.0), 1.0) keeps scale unless the other operand compares strictly greater / smaller
    if (0.0 > scale) scale = 0.0;
    if (1.0 < scale) scale = 1.0;
    if (scale != scale) return -1;                               // int(nan) raises in Python
    const double size = (double)(h < w ? h : w) * scale;
    return (int)(std::floor(size / 2.0) * 2.0);                  // int((size // 2) * 2), exact for size >= 0
}

double refine_threshold(double rel, int h_to, int w_to) {
    int mx = h_to > w_to ? h_to : w_to;
    if (3 > mx) mx = 3;                                          // max(*image_to.shape) includes the 3 channels
    return rel * (double)mx;
}

int launch_grouped_candidates(const RefineLevel& lv, const int32_t* ids, const double* loc_from, const double* history, double* pts,
                              double* box, int32_t* fail, cudaStream_t s) {
    grouped_candidates_kernel<<<(lv.count + kRefineThreads - 1) / kRefineThreads, kRefineThreads, 0, s>>>(lv, ids, loc_from, history,
                                                                                                         pts, box, fail);
    COTR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_refine_geometry(const RefineLevel& lv, const int32_t* ids, const int32_t* squad, const int32_t* rank, int n_squads,
                           int longest, const double* loc_from, const double* history, CropSide* sides, int32_t* rects,
                           float* queries, unsigned long long* status, cudaStream_t s) {
    refine_geometry_kernel<<<n_squads, 256, 0, s>>>(lv, ids, squad, rank, n_squads, longest, loc_from, history, sides, rects, queries,
                                                    status);
    COTR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int launch_refine_step(const RefineLevel& lv, const int32_t* ids, const int32_t* squad, const int32_t* rank, int longest,
                       const float* pred, const int32_t* rects, double* history, int32_t* good, int32_t* good_count,
                       unsigned long long* status, cudaStream_t s) {
    refine_step_kernel<<<(lv.count + kRefineThreads - 1) / kRefineThreads, kRefineThreads, 0, s>>>(lv, ids, squad, rank, longest, pred,
                                                                                                  rects, history, good, good_count, status);
    COTR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace cotr

extern "C" int cotr_test_refine_math(int op, int n, int levels, double rel_threshold, const double* in, const int32_t* in_i,
                                     double* out, int32_t* out_i) {
    using namespace cotr;
    COTR_CHECK(n >= 0 && (n == 0 || (in && in_i)), "cotr_test_refine_math: bad arguments");
    for (int k = 0; k < n; ++k) {
        switch (op) {
        case 0: {   // [pos_x, pos_y, scale] + [h, w] -> [left, top, size, flag]
            COTR_CHECK(out_i, "cotr_test_refine_math: null out_i");
            const double* a = in + 3 * k;
            const int h = in_i[2 * k], w = in_i[2 * k + 1];
            const int size = refine_crop_size(h, w, a[2]);
            int flag = 0, x = 0, y = 0;
            if (size >= 0) {
                x = patch_corner(a[0], size, w, &flag);
                y = patch_corner(a[1], size, h, &flag);
            }
            int32_t* o = out_i + 4 * k;
            o[0] = x; o[1] = y; o[2] = size; o[3] = flag;
            break;
        }
        case 1: {   // [x, y] + [px, py, size] -> the fp32 canvas query (as doubles)
            COTR_CHECK(out, "cotr_test_refine_math: null out");
            const float2 q = query_in(in[2 * k], in[2 * k + 1], in_i[3 * k], in_i[3 * k + 1], in_i[3 * k + 2]);
            out[2 * k] = q.x; out[2 * k + 1] = q.y;
            break;
        }
        case 2: {   // [p_x, p_y] (fp32 values) + [px, py, size] -> pixel location
            COTR_CHECK(out, "cotr_test_refine_math: null out");
            const double2 l = scale_to_loc((float)in[2 * k], (float)in[2 * k + 1], in_i[3 * k], in_i[3 * k + 1], in_i[3 * k + 2]);
            out[2 * k] = l.x; out[2 * k + 1] = l.y;
            break;
        }
        case 3: {   // history (levels + 1, 2) + [h_to, w_to] -> good
            COTR_CHECK(out_i && levels >= 1 && levels <= 7, "cotr_test_refine_math: bad conclude arguments");
            out_i[k] = conclude_good(in + (size_t)k * (levels + 1) * 2, levels + 1,
                                     refine_threshold(rel_threshold, in_i[2 * k], in_i[2 * k + 1])) ? 1 : 0;
            break;
        }
        default:
            COTR_CHECK(false, "cotr_test_refine_math: unknown op %d", op);
        }
    }
    return 0;
}
