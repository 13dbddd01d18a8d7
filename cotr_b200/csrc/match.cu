// Keypoint matching across image pairs (cotr_match_keypoints / cotr_mutual_nearest, include/cotr_b200.h): the query and
// pixel arithmetic of the first zoom level with the whole image as the patch (refinement_task.py:110, :145-151), and
// the mutual-nearest-neighbour rule of demo_guided_matching.py:48-62 (scipy.spatial.distance_matrix + np.argmin + the
// double loop), reproduced bit for bit in fp64 without a K_a x K_b distance matrix.
#include "common.cuh"

namespace cotr {
namespace {

constexpr int kNearestSplit = 4;                                   // candidate lanes per row
constexpr int kNearestThreads = kMatchTileRows * kNearestSplit;    // 256
constexpr int kNearestChunk = 1024;                                // candidates staged per pass: 16 KB
constexpr int kMutualThreads = 1024;

__global__ void __launch_bounds__(kMatchTileRows) match_queries_kernel(const MatchTile* __restrict__ tiles,
                                                                       const double* __restrict__ kpts, float* __restrict__ queries) {
    const MatchTile t = tiles[blockIdx.x];      // written by a copy before the launch
    pdl_wait();
    const int i = threadIdx.x;
    if (i >= t.rows) return;
    const size_t k = (size_t)t.left0 + i, r = (size_t)t.row0 + i;
    queries[2 * r] = __double2float_rn(__ddiv_rn(kpts[2 * k], 2.0 * (double)t.w_left));
    queries[2 * r + 1] = __double2float_rn(__ddiv_rn(kpts[2 * k + 1], (double)t.h_left));
}

__global__ void __launch_bounds__(kMatchTileRows) match_pixels_kernel(const MatchTile* __restrict__ tiles,
                                                                      const float* __restrict__ pred, double* __restrict__ corr) {
    const MatchTile t = tiles[blockIdx.x];
    pdl_wait();
    const int i = threadIdx.x;
    if (i >= t.rows) return;
    const size_t r = (size_t)t.row0 + i;
    // (p.x - 0.5) * 2 in fp32 as the reference's fp32 array does; both products are exact in fp64 for W, H <= 65536
    const float px = __fmul_rn(__fsub_rn(pred[2 * r], 0.5f), 2.0f);
    corr[2 * r] = __dmul_rn((double)px, (double)t.w_right);
    corr[2 * r + 1] = __dmul_rn((double)pred[2 * r + 1], (double)t.h_right);
}

// (d, i) beats (bd, bi) in np.argmin's order: a NaN beats any number, then the smaller distance, then the smaller index;
// i < 0 is an empty partial result.
__device__ __forceinline__ bool nearer(double d, int i, double bd, int bi) {
    if (i < 0) return false;
    if (bi < 0) return true;
    const bool n = d != d, bn = bd != bd;
    if (n != bn) return n;
    if (!n && d != bd) return d < bd;
    return i < bi;
}

// One CTA per tile: thread (g, r) scans candidates j = g, g + 4, ... of the staged chunks for row r in index order,
// keeping the smallest squared sum s, the distance d = sqrt(s) of its best candidate and that candidate's index.  sqrt is
// taken only when s improves on the smallest s so far (sqrt is monotonic, so nothing else can lower d); the candidate
// replaces the best only when its d is strictly smaller, so equal d - including distinct s that round to the same
// sqrt - keeps the earlier index.  The first NaN is final.  The four lanes of a row then merge in `nearer` order.
__global__ void __launch_bounds__(kNearestThreads) nearest_kernel(const MatchTile* __restrict__ tiles, const double* __restrict__ kpts,
                                                                  const double* __restrict__ corr, int* __restrict__ nearest) {
    __shared__ double2 cand[kNearestChunk];
    __shared__ double part_d[kNearestSplit - 1][kMatchTileRows];
    __shared__ int part_i[kNearestSplit - 1][kMatchTileRows];
    const MatchTile t = tiles[blockIdx.x];
    const int r = threadIdx.x % kMatchTileRows, g = threadIdx.x / kMatchTileRows;
    pdl_wait();
    const bool active = r < t.rows;
    double cx = 0.0, cy = 0.0;
    if (active) {
        cx = corr[2 * ((size_t)t.row0 + r)];
        cy = corr[2 * ((size_t)t.row0 + r) + 1];
    }
    double best_s = 0.0, best_d = 0.0;
    int best = -1;
    const double* right = kpts + 2 * (size_t)t.right0;
    for (int c0 = 0; c0 < t.n_right; c0 += kNearestChunk) {
        const int n = min(kNearestChunk, t.n_right - c0);
        __syncthreads();                        // the previous chunk has been read
        for (int j = threadIdx.x; j < n; j += kNearestThreads)
            cand[j] = make_double2(right[2 * (size_t)(c0 + j)], right[2 * (size_t)(c0 + j) + 1]);
        __syncthreads();
        if (!active || (best >= 0 && best_d != best_d)) continue;
        for (int j = g; j < n; j += kNearestSplit) {
            const double2 k = cand[j];
            const double dx = __dsub_rn(k.x, cx), dy = __dsub_rn(k.y, cy);
            const double s = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
            if (s != s) { best_d = s; best = c0 + j; break; }
            if (best < 0 || s < best_s) {
                best_s = s;
                const double d = __dsqrt_rn(s);
                if (best < 0 || d < best_d) { best_d = d; best = c0 + j; }
            }
        }
    }
    if (g > 0) { part_d[g - 1][r] = best_d; part_i[g - 1][r] = best; }
    __syncthreads();
    if (g > 0 || !active) return;
    for (int h = 0; h < kNearestSplit - 1; ++h)
        if (nearer(part_d[h][r], part_i[h][r], best_d, best)) { best_d = part_d[h][r]; best = part_i[h][r]; }
    nearest[(size_t)t.row0 + r] = best;
}

// One CTA per pair: row i of context 2p survives when nearest_ba[nearest_ab[i]] == i; survivors are compacted in
// ascending i with a block scan into the pair's own rows of `match`, and their number goes to count[p].
__global__ void __launch_bounds__(kMutualThreads) mutual_kernel(const int4* __restrict__ pairs, const int* __restrict__ nearest,
                                                                int* __restrict__ match, int* __restrict__ count) {
    __shared__ int warp_excl[kMutualThreads / 32];
    __shared__ int chunk_total;
    const int4 p = pairs[blockIdx.x];
    pdl_wait();
    const int* ab = nearest + p.x;
    const int* ba = ab + p.y;
    int* out = match + 2 * (size_t)p.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int base = 0;
    for (int i0 = 0; i0 < p.y; i0 += kMutualThreads) {
        const int i = i0 + threadIdx.x;
        int j = -1;
        bool keep = false;
        if (i < p.y) {
            j = ab[i];
            keep = j >= 0 && j < p.z && ba[j] == i;
        }
        const unsigned ballot = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) warp_excl[warp] = __popc(ballot);
        __syncthreads();
        if (warp == 0) {
            const int v = warp_excl[lane];
            int incl = v;
            for (int o = 1; o < 32; o <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += u;
            }
            warp_excl[lane] = incl - v;
            if (lane == 31) chunk_total = incl;
        }
        __syncthreads();
        if (keep) {
            const int k = base + warp_excl[warp] + __popc(ballot & ((1u << lane) - 1u));
            out[2 * k] = i;
            out[2 * k + 1] = j;
        }
        base += chunk_total;
        __syncthreads();                        // warp_excl / chunk_total are rewritten by the next chunk
    }
    if (threadIdx.x == 0) count[blockIdx.x] = base;
}

}  // namespace

int launch_match_queries(const MatchTile* tiles, int n_tiles, const double* kpts, float* queries, cudaStream_t s) {
    if (n_tiles == 0) return 0;
    COTR_CHECK_CUDA(launch_kernel(match_queries_kernel, dim3(n_tiles), dim3(kMatchTileRows), 0, s, tiles, kpts, queries));
    return 0;
}

int launch_match_pixels(const MatchTile* tiles, int n_tiles, const float* pred, double* corr, cudaStream_t s) {
    if (n_tiles == 0) return 0;
    COTR_CHECK_CUDA(launch_kernel(match_pixels_kernel, dim3(n_tiles), dim3(kMatchTileRows), 0, s, tiles, pred, corr));
    return 0;
}

int launch_nearest(const MatchTile* tiles, int n_tiles, const double* kpts, const double* corr, int* nearest, cudaStream_t s) {
    if (n_tiles == 0) return 0;
    COTR_CHECK_CUDA(launch_kernel(nearest_kernel, dim3(n_tiles), dim3(kNearestThreads), 0, s, tiles, kpts, corr, nearest));
    return 0;
}

int launch_mutual(const int4* pairs, int B, const int* nearest, int* match, int* count, cudaStream_t s) {
    COTR_CHECK_CUDA(launch_kernel(mutual_kernel, dim3(B), dim3(kMutualThreads), 0, s, pairs, nearest, match, count));
    return 0;
}

}  // namespace cotr
