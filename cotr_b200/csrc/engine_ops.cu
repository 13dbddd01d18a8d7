// Device-side pieces of the zoom-in engine around the network (SURVEY.md section 8f rows 2-4):
//   * rasterize_triangles: the rendering half of triangulate_corr (inference_helper.py:293-308) - the reference draws
//     the Delaunay triangles of the source points with OpenGL, vertex colour = target coordinates; here one thread
//     block per triangle walks the triangle's bounding box and writes the barycentric interpolation at every pixel
//     centre it covers (top-left fill rule, so shared edges are written exactly once and the result is deterministic).
#include <cmath>
#include <map>
#include <vector>

#include "common.cuh"

namespace cotr {

namespace {

struct Vtx { float x, y, u, v; };

// edge function of (a -> b) at p, in double: the coordinates are fp32 pixel positions, so the products are exact
__device__ __forceinline__ double edge_fn(double ax, double ay, double bx, double by, double px, double py) {
    return (bx - ax) * (py - ay) - (by - ay) * (px - ax);
}
// top-left rule for a counter-clockwise triangle in a y-down image: an edge owns the pixels exactly on it when it is a
// "left" edge (going down) or a horizontal "top" edge (going left)
__device__ __forceinline__ bool owns_edge(double ax, double ay, double bx, double by) {
    const double dx = bx - ax, dy = by - ay;
    return dy > 0.0 || (dy == 0.0 && dx < 0.0);
}

__global__ void __launch_bounds__(256) rasterize_triangles_kernel(const Vtx* __restrict__ tris, int n_tri, int H, int W, float2* __restrict__ out) {
    for (int t = blockIdx.x; t < n_tri; t += gridDim.x) {
        Vtx a = tris[3 * t], b = tris[3 * t + 1], c = tris[3 * t + 2];
        double area = edge_fn(a.x, a.y, b.x, b.y, c.x, c.y);
        if (area == 0.0) continue;                         // degenerate
        if (area < 0.0) { const Vtx tmp = b; b = c; c = tmp; area = -area; }
        const float minx = fminf(a.x, fminf(b.x, c.x)), maxx = fmaxf(a.x, fmaxf(b.x, c.x));
        const float miny = fminf(a.y, fminf(b.y, c.y)), maxy = fmaxf(a.y, fmaxf(b.y, c.y));
        // pixel (ix, iy) is sampled at its centre (ix + 0.5, iy + 0.5)
        int x0 = (int)floorf(minx - 0.5f), x1 = (int)ceilf(maxx - 0.5f);
        int y0 = (int)floorf(miny - 0.5f), y1 = (int)ceilf(maxy - 0.5f);
        x0 = max(x0, 0); y0 = max(y0, 0); x1 = min(x1, W - 1); y1 = min(y1, H - 1);
        if (x1 < x0 || y1 < y0) continue;
        const int bw = x1 - x0 + 1, n = bw * (y1 - y0 + 1);
        const bool own_ab = owns_edge(a.x, a.y, b.x, b.y), own_bc = owns_edge(b.x, b.y, c.x, c.y), own_ca = owns_edge(c.x, c.y, a.x, a.y);
        const double inv = 1.0 / area;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const int iy = y0 + i / bw, ix = x0 + i % bw;
            const double px = ix + 0.5, py = iy + 0.5;
            const double wa = edge_fn(b.x, b.y, c.x, c.y, px, py);      // weight of vertex a
            const double wb = edge_fn(c.x, c.y, a.x, a.y, px, py);
            const double wc = edge_fn(a.x, a.y, b.x, b.y, px, py);
            const bool in = (wa > 0.0 || (wa == 0.0 && own_bc)) && (wb > 0.0 || (wb == 0.0 && own_ca)) && (wc > 0.0 || (wc == 0.0 && own_ab));
            if (!in) continue;
            const double la = wa * inv, lb = wb * inv, lc = wc * inv;
            out[(size_t)iy * W + ix] = make_float2((float)(la * a.u + lb * b.u + lc * c.u), (float)(la * a.v + lb * b.v + lc * c.v));
        }
    }
}

}  // namespace

int rasterize_triangles_launch(const float* tris, int n_tri, int H, int W, float* out, cudaStream_t s) {
    COTR_CHECK(out != nullptr && H > 0 && W > 0 && n_tri >= 0 && (n_tri == 0 || tris != nullptr), "cotr_rasterize_triangles: bad arguments");
    COTR_CHECK_CUDA(cudaMemsetAsync(out, 0, (size_t)H * W * 2 * sizeof(float), s));
    if (n_tri == 0) return 0;
    const int grid = n_tri < kNumSms * 8 ? n_tri : kNumSms * 8;
    rasterize_triangles_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const Vtx*>(tris), n_tri, H, W, reinterpret_cast<float2*>(out));
    COTR_CHECK_CUDA(cudaGetLastError());
    return 0;
}


// =====================================================================================================================
// Dense first guess, device-side tail (inference_helper.py:155-160 + :61-75 + COTR/utils/utils.py:69-83):
//   per (tile of a, tile of b) the reference maps the 256 x 256 x [x, y, confidence] answer of the dense pass into
//   full-image coordinates (an affine map of x, y), resizes the three channels to the tile's pixel size with Pillow's
//   mode-'F' bilinear filter (`float_image_resize`) and merges the tiles per pixel by smallest confidence, ties to the
//   later tile (`merge_flow_patches`).  Here that is two kernels per tile on the device: the answers never leave the
//   GPU until the merged (H, W, 2) flow and (H, W) confidence are complete.
// Pillow's float resampler restated exactly (libImaging/Resample.c, ImagingResampleHorizontal/Vertical_32bpc): double
// coefficients (precompute_coeffs), double accumulation `ss += pixel * k` with separate multiply and add (the x86-64
// build has no FMA contraction: __dmul_rn / __dadd_rn), float32 store after each of the two passes.
// =====================================================================================================================
// Shared with the map resize of cotr_resize_maps (resize.cu).
void host_float_coeffs(int in_size, int out_size, std::vector<int>& bounds, std::vector<double>& weights, int& ksize) {
    const double scale = (double)((float)in_size - 0.0f) / out_size;
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = 1.0 * filterscale;
    ksize = (int)std::ceil(support) * 2 + 1;
    bounds.assign((size_t)out_size * 2, 0);
    weights.assign((size_t)out_size * ksize, 0.0);
    const double ss = 1.0 / filterscale;
    for (int xx = 0; xx < out_size; ++xx) {
        const double center = 0.0 + (xx + 0.5) * scale;
        double ww = 0.0;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in_size) xmax = in_size;
        xmax -= xmin;
        double* k = &weights[(size_t)xx * ksize];
        for (int x = 0; x < xmax; ++x) {
            double w = (x + xmin - center + 0.5) * ss;
            if (w < 0.0) w = -w;
            w = w < 1.0 ? 1.0 - w : 0.0;
            k[x] = w;
            ww += w;
        }
        for (int x = 0; x < xmax; ++x)
            if (ww != 0.0) k[x] /= ww;
        bounds[(size_t)xx * 2] = xmin;
        bounds[(size_t)xx * 2 + 1] = xmax;
    }
}

namespace {

struct FloatCoeffs {
    int ksize = 0;
    int* bounds = nullptr;      // device [out][2]
    double* weights = nullptr;  // device [out][ksize]
};

struct TileJob {
    const float* tile;        // (256, 256, 3) [x, y, confidence], row pitch `pitch` floats
    int pitch;
    double a[6];              // x' = a0 x + a1 y + a2,  y' = a3 x + a4 y + a5
    int pw, ph;               // tile size in pixels of the full image
    int px, py, ow, oh;       // tile position and full image size
    int kw, kh;
    const int* bw; const double* ww;      // horizontal tables (256 -> pw)
    const int* bh; const double* wh;      // vertical tables (256 -> ph)
};

constexpr int kTileIn = 256;

// horizontal pass: tmp[r][xx][c], r in [0,256), xx in [0,pw)
__global__ void __launch_bounds__(256) flow_resize_h_kernel(const TileJob j, float* __restrict__ tmp) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= kTileIn * j.pw) return;
    const int r = idx / j.pw, xx = idx - r * j.pw;
    const int x0 = j.bw[2 * xx], n = j.bw[2 * xx + 1];
    const double* k = j.ww + (size_t)xx * j.kw;
    const float* src = j.tile + (size_t)r * j.pitch + (size_t)x0 * 3;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    for (int x = 0; x < n; ++x) {
        const float fx = __ldcg(src + 3 * x), fy = __ldcg(src + 3 * x + 1), fc = __ldcg(src + 3 * x + 2);
        // numpy: (float32 x, y) @ float64 2x2 + float64 t, stored back into the float32 array
        const float ax = (float)__dadd_rn(__dadd_rn(__dmul_rn((double)fx, j.a[0]), __dmul_rn((double)fy, j.a[1])), j.a[2]);
        const float ay = (float)__dadd_rn(__dadd_rn(__dmul_rn((double)fx, j.a[3]), __dmul_rn((double)fy, j.a[4])), j.a[5]);
        s0 = __dadd_rn(s0, __dmul_rn((double)ax, k[x]));
        s1 = __dadd_rn(s1, __dmul_rn((double)ay, k[x]));
        s2 = __dadd_rn(s2, __dmul_rn((double)fc, k[x]));
    }
    float* dst = tmp + (size_t)idx * 3;
    dst[0] = (float)s0; dst[1] = (float)s1; dst[2] = (float)s2;
}

// vertical pass + merge: per pixel keep the candidate with the smallest confidence, ties to the later tile
__global__ void __launch_bounds__(256) flow_resize_v_merge_kernel(const TileJob j, const float* __restrict__ tmp, float* __restrict__ flow,
                                                                  float* __restrict__ conf) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= j.ph * j.pw) return;
    const int yy = idx / j.pw, xx = idx - yy * j.pw;
    const int y0 = j.bh[2 * yy], n = j.bh[2 * yy + 1];
    const double* k = j.wh + (size_t)yy * j.kh;
    const float* src = tmp + ((size_t)y0 * j.pw + xx) * 3;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    for (int y = 0; y < n; ++y) {
        const float* q = src + (size_t)y * j.pw * 3;
        s0 = __dadd_rn(s0, __dmul_rn((double)q[0], k[y]));
        s1 = __dadd_rn(s1, __dmul_rn((double)q[1], k[y]));
        s2 = __dadd_rn(s2, __dmul_rn((double)q[2], k[y]));
    }
    const float c = (float)s2;
    const size_t o = (size_t)(j.py + yy) * j.ow + (j.px + xx);
    if (c <= conf[o]) {
        conf[o] = c;
        flow[2 * o] = (float)s0;
        flow[2 * o + 1] = (float)s1;
    }
}

__global__ void flow_init_kernel(float* __restrict__ flow, float* __restrict__ conf, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        conf[i] = 100.f;
        flow[2 * i] = 0.f;
        flow[2 * i + 1] = 0.f;
    }
}

}  // namespace

struct FlowMerger {
    std::map<int, FloatCoeffs> tables;     // keyed by output size (input is always 256)
    float* tmp = nullptr;
    size_t tmp_cap = 0;
};

FlowMerger* flow_merger_create() { return new FlowMerger(); }

void flow_merger_destroy(FlowMerger* f) {
    if (!f) return;
    for (auto& kv : f->tables) { cudaFree(kv.second.bounds); cudaFree(kv.second.weights); }
    if (f->tmp) cudaFree(f->tmp);
    delete f;
}

static int float_table(FlowMerger* f, int out_size, FloatCoeffs* out) {
    auto it = f->tables.find(out_size);
    if (it == f->tables.end()) {
        std::vector<int> b;
        std::vector<double> w;
        FloatCoeffs t;
        host_float_coeffs(kTileIn, out_size, b, w, t.ksize);
        COTR_CHECK_CUDA(cudaMalloc((void**)&t.bounds, b.size() * sizeof(int)));
        COTR_CHECK_CUDA(cudaMalloc((void**)&t.weights, w.size() * sizeof(double)));
        COTR_CHECK_CUDA(cudaMemcpy(t.bounds, b.data(), b.size() * sizeof(int), cudaMemcpyHostToDevice));
        COTR_CHECK_CUDA(cudaMemcpy(t.weights, w.data(), w.size() * sizeof(double), cudaMemcpyHostToDevice));
        it = f->tables.emplace(out_size, t).first;
    }
    *out = it->second;
    return 0;
}

int flow_tile_merge_launch(FlowMerger* f, const float* tile, int pitch, const double* affine, int px, int py, int pw, int ph, int ow, int oh,
                           float* flow, float* conf, int first, cudaStream_t s) {
    COTR_CHECK(f && tile && affine && flow && conf, "cotr_flow_tile_merge: null argument");
    COTR_CHECK(pw >= 1 && ph >= 1 && px >= 0 && py >= 0 && px + pw <= ow && py + ph <= oh && pitch >= kTileIn * 3,
               "cotr_flow_tile_merge: tile (%d,%d,%d,%d) does not fit the %dx%d image", px, py, pw, ph, ow, oh);
    TileJob j;
    j.tile = tile; j.pitch = pitch;
    for (int i = 0; i < 6; ++i) j.a[i] = affine[i];
    j.pw = pw; j.ph = ph; j.px = px; j.py = py; j.ow = ow; j.oh = oh;
    FloatCoeffs tw, th;
    if (float_table(f, pw, &tw) || float_table(f, ph, &th)) return 1;
    j.kw = tw.ksize; j.bw = tw.bounds; j.ww = tw.weights;
    j.kh = th.ksize; j.bh = th.bounds; j.wh = th.weights;
    const size_t need = (size_t)kTileIn * pw * 3 * sizeof(float);
    if (need > f->tmp_cap) {
        COTR_CHECK_CUDA(cudaDeviceSynchronize());
        if (f->tmp) cudaFree(f->tmp);
        COTR_CHECK_CUDA(cudaMalloc((void**)&f->tmp, need));
        f->tmp_cap = need;
    }
    if (first) {
        flow_init_kernel<<<kNumSms * 4, 256, 0, s>>>(flow, conf, (size_t)ow * oh);
        COTR_CHECK_CUDA(cudaGetLastError());
    }
    flow_resize_h_kernel<<<(kTileIn * pw + 255) / 256, 256, 0, s>>>(j, f->tmp);
    COTR_CHECK_CUDA(cudaGetLastError());
    flow_resize_v_merge_kernel<<<(ph * pw + 255) / 256, 256, 0, s>>>(j, f->tmp, flow, conf);
    COTR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace cotr

// =====================================================================================================================
// Squad formation of the grouped scheduler (FasterSparseEngine.form_grouped_batch / form_squad, sparse_engine.py:295-369)
// on the device.  Tasks arrive in the engine's shuffled order with their two end points and with the central-half boxes
// of the crops they would impose as a pilot.  The reference walks that list once: a task that is still free becomes the
// pilot of the next squad and takes along the first `max_load` free tasks (in list order) whose two end points lie
// strictly inside both of its boxes; it stops after `batch_size` squads.  The walk is sequential over squads (<= 32 per
// batch) but every membership test and the "first max_load in list order" selection are parallel over the n tasks:
// one CTA, each thread owns a contiguous slice of the list, a block-wide scan orders the candidates.
// Doubles throughout, strict comparisons: the decisions are bit-identical to the numpy expressions of the host path.
// =====================================================================================================================
namespace cotr {
namespace {

constexpr int kGroupThreads = 1024;

__global__ void __launch_bounds__(kGroupThreads) group_tasks_kernel(const double* __restrict__ pts, const double* __restrict__ box, int n,
                                                                    int batch_size, int max_load, int* __restrict__ squad,
                                                                    int* __restrict__ rank, int* __restrict__ n_squads) {
    __shared__ int s_scan[kGroupThreads];
    __shared__ int s_pilot;
    __shared__ double s_box[8];
    const int t = threadIdx.x;
    const int per = (n + kGroupThreads - 1) / kGroupThreads;
    const int lo = min(t * per, n), hi = min(lo + per, n);
    for (int i = lo; i < hi; ++i) { squad[i] = -1; rank[i] = -1; }
    __syncthreads();
    int cursor = 0, made = 0;
    while (made < batch_size) {
        // next free task at or after the cursor (list order): block-wide minimum
        int first = n;
        for (int i = max(lo, cursor); i < hi; ++i)
            if (squad[i] < 0) { first = i; break; }
        s_scan[t] = first;
        __syncthreads();
        for (int off = kGroupThreads / 2; off > 0; off >>= 1) {
            if (t < off) s_scan[t] = min(s_scan[t], s_scan[t + off]);
            __syncthreads();
        }
        const int pilot = s_scan[0];
        __syncthreads();
        if (pilot >= n) break;
        if (t == 0) {
            squad[pilot] = made; rank[pilot] = 0;
            s_pilot = pilot;
            for (int k = 0; k < 8; ++k) s_box[k] = box[(size_t)pilot * 8 + k];
        }
        __syncthreads();
        const double fl = s_box[0], fr = s_box[1], fu = s_box[2], fd = s_box[3], tl = s_box[4], tr = s_box[5], tu = s_box[6], td = s_box[7];
        // candidates of this thread's slice (the pilot itself is no longer free)
        int cnt = 0;
        for (int i = lo; i < hi; ++i) {
            const double* p = pts + (size_t)i * 4;
            const bool fits = squad[i] < 0 && p[0] > fl && p[0] < fr && p[1] > fu && p[1] < fd && p[2] > tl && p[2] < tr && p[3] > tu && p[3] < td;
            cnt += fits ? 1 : 0;
        }
        // exclusive scan of the per-thread counts (Hillis-Steele, 1024 entries)
        s_scan[t] = cnt;
        __syncthreads();
        for (int off = 1; off < kGroupThreads; off <<= 1) {
            const int v = t >= off ? s_scan[t - off] : 0;
            __syncthreads();
            s_scan[t] += v;
            __syncthreads();
        }
        int pos = s_scan[t] - cnt;            // members before this thread's slice
        for (int i = lo; i < hi && pos < max_load; ++i) {
            const double* p = pts + (size_t)i * 4;
            const bool fits = squad[i] < 0 && p[0] > fl && p[0] < fr && p[1] > fu && p[1] < fd && p[2] > tl && p[2] < tr && p[3] > tu && p[3] < td;
            if (fits) { squad[i] = made; rank[i] = 1 + pos; ++pos; }
        }
        __syncthreads();
        cursor = s_pilot + 1;
        ++made;
    }
    if (t == 0) *n_squads = made;
}

}  // namespace

int group_tasks_launch(const double* pts, const double* box, int n, int batch_size, int max_load, int* squad, int* rank, int* n_squads, cudaStream_t s) {
    COTR_CHECK(n >= 0 && batch_size >= 1 && max_load >= 0 && squad && rank && n_squads && (n == 0 || (pts && box)), "cotr_group_tasks: bad arguments");
    group_tasks_kernel<<<1, kGroupThreads, 0, s>>>(pts, box, n, batch_size, max_load, squad, rank, n_squads);
    COTR_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace cotr
