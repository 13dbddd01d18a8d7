// Shared declarations of the cotr_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <vector>

namespace cotr {

void set_error(const char* fmt, ...);

#define COTR_CHECK_CUDA(expr)                                                                      \
    do {                                                                                           \
        cudaError_t e_ = (expr);                                                                   \
        if (e_ != cudaSuccess) {                                                                   \
            ::cotr::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e_)); \
            return 1;                                                                              \
        }                                                                                          \
    } while (0)

#define COTR_CHECK(cond, ...)                                                                      \
    do {                                                                                           \
        if (!(cond)) {                                                                             \
            ::cotr::set_error(__VA_ARGS__);                                                        \
            return 1;                                                                              \
        }                                                                                          \
    } while (0)

// ---------------------------------------------------------------------------------------------------------------
// Programmatic dependent launch.  Every kernel of the forward is launched with the programmatic-stream-serialization
// attribute: it may start (barrier init, weight prefetch by TMA) while its predecessor in the
// stream / graph is still draining, and calls pdl_wait() before it first touches memory the predecessor produces
// (or still reads).  At batch 1 the forward is ~135 latency-bound launches, so hiding launch + prologue matters.
// ---------------------------------------------------------------------------------------------------------------
extern int g_use_pdl;
extern int g_tc_variant;
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#endif

// Function attributes (opt-in dynamic shared memory) are per device, and one process may hold one handle per device:
// remember per kernel on which devices it has been configured.  (Racing first uses merely set the attribute twice.)
inline bool first_use_on_device(unsigned long long* configured_mask) {
    int dev = 0;
    cudaGetDevice(&dev);
    const unsigned long long bit = 1ull << (dev & 63);
    if (*configured_mask & bit) return false;
    *configured_mask |= bit;
    return true;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = g_use_pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// Same, with a thread-block cluster of (1, 1, cluster_z) CTAs (grid.z must be a multiple of cluster_z).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                                         int cluster_z, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[2];
    int n = 0;
    if (g_use_pdl) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    if (cluster_z > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = 1;
        attr[n].val.clusterDim.y = 1;
        attr[n].val.clusterDim.z = (unsigned)cluster_z;
        ++n;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// Streaming multiprocessors of an H100 SXM: grid-stride kernels launch at most 16 blocks per SM.
constexpr int kNumSms = 132;

constexpr int kDModel = 256;
constexpr int kHeads = 8;
constexpr int kHeadDim = 32;
constexpr int kTokens = 512;   // 16 x 32 context grid
constexpr int kFF = 1024;
constexpr int kEncLayers = 6;
constexpr int kDecLayers = 6;

// Attention operand images (tensor-core path).  The keys and values of one (pair, slot, head) - slot = decoder layer, or 0
// for the encoder's own layer - are stored in HBM exactly as the attention kernel wants them in shared memory, so that
// staging them is two bulk-TMA copies issued by one thread (cp.async.bulk -> UBLKCP) instead of 8 192 16-byte cp.async
// (a CTA that owns a slice of the keys copies 8 runs of K and one of V):
//   K image  [plane hi | lo][4 groups of 8 head dims][512 keys][16 B]           = 2 x 32 KB  (wgmma K-major canonical layout)
//   V image  [64 groups of 8 keys][hi: 32 head dims x 16 B | lo: 32 x 16 B | 16 B pad]  = 64 x 1040 B
// written in that form by the epilogue of the projection GEMM (split16.cuh::store16).
constexpr size_t kAttnKPlaneBytes = 4 * 512 * 16;                         // 32 KB
constexpr size_t kAttnKImgBytes = 2 * kAttnKPlaneBytes;                   // 64 KB
constexpr size_t kAttnVGroupBytes = 2 * 32 * 16 + 16;                     // 1040 B
constexpr size_t kAttnVImgBytes = 64 * kAttnVGroupBytes;                  // 66 560 B
constexpr size_t kAttnHeadImgBytes = kAttnKImgBytes + kAttnVImgBytes;     // 132 096 B per (pair, slot, head)

// ---------------------------------------------------------------------------------------------------------------
// "split16" activations.  Every activation between kernels is stored as TWO fp16 planes, x ~= hi + lo (22 mantissa
// bits, same bytes as fp32): the tensor-core kernels need their operands in exactly that form (gemm_tc.cu), so the
// producer's epilogue splits once and every consumer stages its operand with plain asynchronous 16-byte copies.
// hi + lo is exactly representable in fp32, so reconstruct -> split round-trips are lossless.
// ---------------------------------------------------------------------------------------------------------------
struct Split16 {          // plain aggregates: they travel inside kernel parameter structs
    __half* hi;
    __half* lo;
};
struct CSplit16 {
    const __half* hi;
    const __half* lo;
};
inline CSplit16 cs(const Split16& s) { return CSplit16{s.hi, s.lo}; }
inline Split16 offset(const Split16& s, size_t elems) { return Split16{s.hi + elems, s.lo + elems}; }
inline CSplit16 offset(const CSplit16& s, size_t elems) { return CSplit16{s.hi + elems, s.lo + elems}; }

// The stem's input.  The network input is an fp32 (B,3,256,512) NCHW canvas, two 256x256 images side by side.  The 7x7
// stride-2 convolution reads it through a split16 copy made by one small kernel per forward (launch_stem_canvas): image
// n = 2*pair + half as [kStemCanvasRows][kStemCanvasPitch] pixels of 4 halves (r, g, b, 0), the image at rows / columns
// 3.., everything else zero (the convolution's padding, written once when the buffer is allocated).  A filter row of
// output pixel (oh, ow) is then 8 consecutive pixels = 64 contiguous, 16-byte aligned bytes per plane starting at pixel
// (2 oh + kh, 2 ow): no bounds checks, plain 16-byte cp.async like every other operand.  K = 7 rows x 8 pixel slots x 4
// channels = 224, the weights carry zeros for slot 7 and channel 3.
constexpr int kStemCanvasRows = 262, kStemCanvasPitch = 264;
constexpr size_t kStemCanvasElems = (size_t)kStemCanvasRows * kStemCanvasPitch * 4;      // halves per image and plane
constexpr int kStemK = 7 * 32;

// How a GEMM finds row m, column k of its A operand.
enum AMode : int {
    A_ROWMAJOR = 0,   // A[m * lda + k]
    A_CONV_NHWC = 1,  // implicit im2col over an NHWC activation: m -> (n, oh, ow), k -> (kh, kw, c)
    A_STEM_NHWC4 = 2, // 7x7 stride-2 stem: implicit im2col over the zero-bordered split16 NHWC4 copy of the canvas (below)
    A_TOKENS = 3,     // m = pair*512 + i*32 + j gathers row ((a_pairs[2*pair + (j>>4)])*16 + i)*16 + (j&15)
};

// D[M,N] = epilogue( A[M,K] * W[N,K]^T ).
struct GemmParams {
    int M, N, K;
    // A operand: split16 activation (A_STEM_NHWC4: the stem canvas)
    CSplit16 a;
    int a_mode;
    int lda;
    // A_TOKENS: [pairs][2] device table, the (left, right) image of each pair among the (n,16,16,1024) images of `a`.
    // Written before the launch by a copy, never by a kernel, so the loaders may read it before the dependency wait.
    const int* a_pairs;
    int H, W, C;      // convolution geometry: input height / width / channels (per image)
    int OH, OW;       // output height / width
    int KH, KW, stride, pad;
    // weights: fp32 row-major [N, K] (K ordered (kh, kw, c) for convolutions) for the SIMT path; for the tensor-core
    // path the same matrix pre-scaled by a power of two, pre-split into fp16 hi/lo and pre-tiled (gemm_tc.cu).
    const float* Wt;
    const void* Wtc;
    float acc_scale;  // undoes the power of two on the accumulator
    // epilogue: v = acc * acc_scale + bias[n] + addmat[(m % add_period) * ld_add + n] + residual[m * ldr + n]; relu; LN
    const float* bias;
    const float* addmat;
    int add_period, ld_add;
    CSplit16 res;
    int ldr;
    int relu;
    const float* ln_gamma;   // optional LayerNorm over the N = 256 columns of each row (after the residual)
    const float* ln_beta;
    // Deferred LayerNorm (tensor-core path, row-major A).  A LayerNorm output is never stored: the GEMM that produces the
    // PRE-norm rows x (N = 256) also leaves, per row and 16-column chunk, the chunk's (mean, M2) in `ln_part_out`
    // [M][16] float2 (from the fp32 values in its epilogue registers); every consumer merges the 16 pairs into the row's
    // (mean, rstd) in its own epilogue prologue and applies the norm on the fly:
    //   * as the A operand (K = 256): the weights carry gamma (W' = W diag(gamma), packed at model creation) and
    //         y[n] = rstd * (acc[n] - mean * a_ln_cs[n]) + bias[n],   a_ln_cs[n] = sum_k W'[n,k],  bias = beta W^T + b;
    //   * as the residual operand: res[n] = (r[n] - mean) rstd res_ln_gamma[n] + res_ln_beta[n].
    const float* a_ln_cs;          // [N]; null = A is used as it is stored
    const float2* a_ln_part;       // [M][16] partial statistics of the A rows
    const float2* res_ln_part;     // [M][16] partial statistics of the residual rows; null = plain residual
    const float* res_ln_gamma;
    const float* res_ln_beta;
    float2* ln_part_out;           // [M][16]; null = no statistics wanted
    // outputs
    float* out_f32;          // when non-null: plain fp32 row-major output (the final prediction, N = 2)
    Split16 out;             // otherwise split16, row-major with leading dimension ldc ...
    int ldc;
    // ... except that 256-column blocks of N can be redirected (K/V projections): blk_map[b] >= 0 -> the block is
    // stored at column offset blk_map[b] of `out`; blk_map[b] = -(v+1) -> the block is a value projection and is
    // stored TRANSPOSED as vt[((pair * n_vt + v) * 256 + c) * 512 + key] (row = pair*512 + key), the K-major B operand
    // the attention kernels need.
    // With kv_img set (tensor-core path) the key / value blocks go into the attention operand images instead:
    // blk_map[b] = -(v+1) -> value block of slot v, blk_map[b] = -1000 - s -> key block of slot s; the image of
    // (pair, slot, head) starts at kv_img + ((pair * n_vt + slot) * 8 + head) * kAttnHeadImgBytes.
    int remap;
    int blk_map[12];
    Split16 vt;
    int n_vt;
    unsigned char* kv_img;
};

// Query rows per CTA of the two attention kernels, and the fewest rows of one pair that go to the tensor-core kernel
// (fewer: a 128-row MMA tile would be more than 75% padding, the SIMT kernel runs them).
constexpr int kAttnTcTileRows = 128;
constexpr int kAttnSimtTileRows = 64;
constexpr int kAttnTcMinRows = 32;

// softmax(q k^T) v per head; q already carries the head_dim^-0.5 scale.
struct AttnParams {
    CSplit16 q; int ldq;         // rows: local row r = pair_local * nq + i (see tiles below)
    CSplit16 k; int ldk;         // rows: (pair0 + pair_local) * 512 + key
    CSplit16 vt;                 // [(pair0 + pair_local) * vt_pair_stride + (head*32 + d) * 512 + key]
    size_t vt_pair_stride;
    // tensor-core path: keys and values as operand images (see kAttnHeadImgBytes); k / vt above are then unused.
    // image of (pair0 + pair_local, head) = kv_img + (pair0 + pair_local) * img_pair_stride + head * kAttnHeadImgBytes
    const unsigned char* kv_img;
    size_t img_pair_stride;
    Split16 out; int ldo;
    int nq;                      // query rows per pair in this launch
    int npairs;
    int pair0;
    // Ragged decode (cotr_decode_ragged): when non-null, CTA blockIdx.x owns the rows of tile tiles[blockIdx.x] =
    // (pair_local, first q / out row, row count) - at most one CTA tile of rows of one pair - and nq / npairs are unused:
    // the grid is (n_tiles, heads, key split).  Written before the launch by a copy, never by a kernel, so the kernels
    // may read it before the dependency wait.  null: row r = pair_local * nq + i as above.
    const int4* tiles;
    int n_tiles;
};

// Head-averaged attention weights (attention_weights.cu): out[pair_local][i][key] = (1/8) sum_h softmax(q_h k_h^T)[i][key],
// the map nn.MultiheadAttention returns with need_weights.  q / k / kv_img / nq / npairs / pair0 as in AttnParams: the
// tensor-core kernel reads the keys from the operand images, the fp32 SIMT one from the row-major k.
struct AttnWeightsParams {
    CSplit16 q; int ldq;
    CSplit16 k; int ldk;
    const unsigned char* kv_img;
    size_t img_pair_stride;
    float* out;                  // fp32, row i of local pair p at out + p * out_pair_stride + i * 512
    size_t out_pair_stride;
    int nq;
    int npairs;
    int pair0;
};

// A transformer feed-forward block with its residual and post-LayerNorm (mlp_tc.cu):
//   out = LN(x + W2 relu(W1 x + b1) + b2), then optionally a second LayerNorm (g2 / be2);  x, out: [M][256], may alias.
struct MlpParams {
    int M;
    CSplit16 x;
    Split16 out;
    const void* w1;      // tensor-core image of linear1 [1024][256] (gemm_tc.cu tc_pack_weight)
    float w1_scale;
    const float* b1;
    const void* w2;      // tensor-core image of linear2 [256][1024]
    float w2_scale;
    const float* b2;
    const float *g, *be;
    const float *g2, *be2;     // null: no second LayerNorm
};

int launch_gemm_simt(const GemmParams& p, cudaStream_t s);
int launch_mlp_tc(const MlpParams& p, cudaStream_t s);
int launch_gemm_simt_raw(const GemmParams& p, float* raw_out_f32, cudaStream_t s);   // result as plain fp32 [M,N]
int launch_layernorm_f32(const float* x, const float* gamma, const float* beta, Split16 out, int rows, cudaStream_t s);
int launch_gemm_tc(const GemmParams& p, cudaStream_t s);
// The plan of a tensor-core GEMM launch (gemm_tc.cu): tile width (16, 32, 64, or 256 with the LayerNorm epilogue), A
// loader (0 row-major / token gather, 1 implicit im2col, 2 stem, 3 halo), deferred-LayerNorm instantiation, split-K
// (CTAs per cluster) and grid.  launch_gemm_tc chooses it by the launch rules; launch_gemm_tc_forced takes the tile width
// and split-K given (0 = the rule), checks them against the same constraints, and reports the plan it launched.  Test hook.
struct GemmPlan {
    int bn, loader, dln, ksplit, grid_x, grid_y;
};
int launch_gemm_tc_forced(const GemmParams& p, int bn, int ksplit, GemmPlan* used, cudaStream_t s);
int launch_attention_simt(const AttnParams& p, cudaStream_t s);
int launch_attention_tc(const AttnParams& p, cudaStream_t s);
// launch_mlp_tc / launch_attention_tc with the hidden split (S = 4 or 8 CTAs per row tile) / key split (ks = 1 or 2)
// given instead of chosen; the tensor-core attention then also runs launches of fewer than kAttnTcMinRows rows per
// pair.  Test hooks.
int launch_mlp_tc_split(const MlpParams& p, int S, cudaStream_t s);
int launch_attention_tc_split(const AttnParams& p, int ks, cudaStream_t s);
int launch_attention_weights_tc(const AttnWeightsParams& p, cudaStream_t s);
int launch_attention_weights_simt(const AttnWeightsParams& p, cudaStream_t s);
int launch_maxpool_3x3s2_nhwc(CSplit16 in, Split16 out, int N, int H, int W, int C, cudaStream_t s);
int launch_layernorm(CSplit16 x, const float* gamma, const float* beta, Split16 out, int rows, cudaStream_t s);
// out = LN2(LN1(x)): the last decoder layer's norm3 followed by decoder.norm (transformer.py:110-111) in one pass
// part[row][c] = (mean, M2) of channels [16c, 16c+16) of a [rows][256] tensor (what GemmParams::ln_part_out holds)
int launch_ln_partials(CSplit16 x, float2* part, int rows, cudaStream_t s);
int launch_layernorm_twice(CSplit16 x, const float* g1, const float* b1, const float* g2, const float* b2, Split16 out, int rows, cudaStream_t s);
int launch_query_encode(const float* queries, Split16 qpos, int rows, cudaStream_t s);
// n_img fp32 256x256 images -> the stem's bordered split16 NHWC4 operand (kStemCanvasElems halves per image and plane).
// halves: img is a (n_img/2,3,256,512) canvas, image n = 2*pair + half; otherwise a (n_img,3,256,256) batch.
int launch_stem_canvas(const float* img, bool halves, Split16 canvas, int n_img, cudaStream_t s);
int launch_f32_to_split16(const float* in, Split16 out, size_t n, cudaStream_t s);
int launch_split16_to_f32(CSplit16 in, float* out, size_t n, cudaStream_t s);

// Keypoint matching (match.cu, cotr_match_keypoints / cotr_mutual_nearest).  Rows are packed in context order; context
// 2p = [a_p | b_p] owns the rows of a_p's keypoints, context 2p+1 = [b_p | a_p] those of b_p's.  A tile is up to
// kMatchTileRows rows of one context; the per-row kernels run one CTA per tile.
constexpr int kMatchTileRows = 64;
struct MatchTile {
    int row0, rows;           // packed rows row0 .. row0 + rows - 1
    int left0;                // packed keypoint of row row0 (the left image's keypoints are the rows, in order)
    int right0, n_right;      // the right image's keypoints: the candidates of nearest
    int w_left, h_left, w_right, h_right;    // image sizes in pixels (match_queries / match_pixels only)
    int pad[3];
};
static_assert(sizeof(MatchTile) == 3 * sizeof(int4), "match tiles travel in an int4 table");
// queries[r] = fp32(kp.x / (2 W_left)), fp32(kp.y / H_left), divisions in fp64
int launch_match_queries(const MatchTile* tiles, int n_tiles, const double* kpts, float* queries, cudaStream_t s);
// corr[r] = fp64(fp32((p.x - 0.5) * 2)) * W_right, fp64(p.y) * H_right
int launch_match_pixels(const MatchTile* tiles, int n_tiles, const float* pred, double* corr, cudaStream_t s);
// nearest[r] = argmin over the right image's keypoints of the fp64 Euclidean distance to corr[r] (-1: no keypoints)
int launch_nearest(const MatchTile* tiles, int n_tiles, const double* kpts, const double* corr, int* nearest, cudaStream_t s);
// pairs[p] = (first row of context 2p, rows of context 2p, rows of context 2p+1, 0); one CTA per pair
int launch_mutual(const int4* pairs, int B, const int* nearest, int* match, int* count, cudaStream_t s);

// Device-side post-processing of the dense pass (dense_post.cu)
int dense_post_launch(const float* pred, float* out, int n, cudaStream_t s);

// Barycentric triangle rasteriser of triangulate_corr (engine_ops.cu)
int rasterize_triangles_launch(const float* tris, int n_tri, int H, int W, float* out, cudaStream_t s);

// Squad formation of the grouped scheduler (engine_ops.cu)
int group_tasks_launch(const double* pts, const double* box, int n, int batch_size, int max_load, int* squad, int* rank, int* n_squads, cudaStream_t s);

// Dense first guess: affine + Pillow-exact float resize + confidence merge of one tile (engine_ops.cu)
struct FlowMerger;
FlowMerger* flow_merger_create();
void flow_merger_destroy(FlowMerger* f);
int flow_tile_merge_launch(FlowMerger* f, const float* tile, int pitch, const double* affine, int px, int py, int pw, int ph, int ow, int oh,
                           float* flow, float* conf, int first, cudaStream_t s);

// Device-side crop + Pillow-exact resize + normalise (preprocess.cu)
struct Preprocessor;
Preprocessor* preprocessor_create();
void preprocessor_destroy(Preprocessor* p);
int preprocess_launch(Preprocessor* p, const unsigned char* img_from, int hf, int wf, const unsigned char* img_to, int ht, int wt,
                      const int* rects_host, int n, float* canvas_dev, cudaStream_t s);
// One crop of the resize kernels: side 2i is task i's "from" crop, 2i+1 its "to" crop.
struct CropSide {
    const unsigned char* img;   // HWC uint8, 3 channels
    int img_w;
    int x, y, size;
    int ksize;
    const int* bounds;
    const int* weights;
    size_t tmp_offset;          // into the horizontal-pass buffer (bytes)
};
// The Pillow coefficient table of a crop side length (built and uploaded on first use, then cached): fills ksize,
// bounds and weights of `side`.
int preprocess_coeffs(Preprocessor* p, int size, CropSide* side);
// The two resize passes over n_sides prepared sides (device table) of side length <= max_size.
int launch_resize_h(const CropSide* sides, int n_sides, int max_size, unsigned char* tmp, cudaStream_t s);
int launch_resize_v(const CropSide* sides, int n_sides, const unsigned char* tmp, float* canvas, cudaStream_t s);

// Pillow's bilinear coefficient tables for an in_size -> out_size axis: 22-bit fixed point for 8-bit images
// (preprocess.cu) and double for mode 'F' (engine_ops.cu).  bounds: out_size x [first source index, tap count].
void host_coeffs(int in_size, int out_size, std::vector<int>& bounds, std::vector<int>& weights, int& ksize);
void host_float_coeffs(int in_size, int out_size, std::vector<int>& bounds, std::vector<double>& weights, int& ksize);

// Whole-image Pillow-exact resizes of cotr_resize_image / cotr_resize_maps (resize.cu).  resize_plan checks nothing (the
// C ABI does), fetches or builds the two axes' tables and grows the intermediate buffer; resize_pass enqueues one pass.
struct Resizer;
Resizer* resizer_create();
void resizer_destroy(Resizer* r);
struct ResizeAxis {
    int ksize = 0;
    const int* bounds = nullptr;
    const void* weights = nullptr;   // int (8-bit images) or double (float maps)
};
struct ResizePlan {
    int u8;                     // 1: uint8 HWC, c = 3; 0: fp32 HWC, c = 1 .. 3
    int h, w, c, oh, ow;
    int need_h, need_v;         // Pillow skips an axis whose size does not change
    ResizeAxis horiz, vert;
    void* tmp;                  // h x ow x c intermediate of the horizontal pass (when both passes run)
};
int resize_plan(Resizer* r, int u8, int h, int w, int c, int oh, int ow, ResizePlan* p);
// pass 0: horizontal, (h, w) -> (h, ow); pass 1: vertical, (h, ow) -> (oh, ow)
int resize_pass(const ResizePlan& p, int pass, const void* src, void* dst, cudaStream_t s);

// Zoom-in walks of cotr_refine and cotr_refine_grouped (refine.cu).  One level: the crops of `count` entries at one zoom
// level, entry i being task task0 + ids[i].
struct RefineLevel {
    int task0, count;
    int level, levels;          // level l of L
    int chunk;                  // chunk index in cotr_refine's walk order (0 in cotr_refine_grouped)
    CropSide from, to;          // everything but x, y and tmp_offset (set per squad by the geometry kernel)
    int h_from, w_from, h_to, w_to;
    double thr;                 // rel_threshold * max(h_to, w_to, 3): conclude()'s bound on the history's std
};
// get_patch_centered_at's crop side for an h x w image at `scale` (-1 for a NaN scale, where Python raises)
int refine_crop_size(int h, int w, double scale);
double refine_threshold(double rel, int h_to, int w_to);
// squads -> CropSide 2s / 2s+1 of each pilot, every member's rect at this level and its query at row s * longest + rank;
// non-finite pilot positions flag `status`
int launch_refine_geometry(const RefineLevel& lv, const int32_t* ids, const int32_t* squad, const int32_t* rank, int n_squads,
                           int longest, const double* loc_from, const double* history, CropSide* sides, int32_t* rects,
                           float* queries, unsigned long long* status, cudaStream_t s);
// predictions -> history row level+1 of every member; at the last level the good flag and good_count; NaN flags `status`
int launch_refine_step(const RefineLevel& lv, const int32_t* ids, const int32_t* squad, const int32_t* rank, int longest,
                       const float* pred, const int32_t* rects, double* history, int32_t* good, int32_t* good_count,
                       unsigned long long* status, cudaStream_t s);
// Grouped walk of cotr_refine_grouped: lv.count candidates ids[0 ..) at lv.level.  End points (n,4), pilot boxes (n,8) and
// the exception code of each candidate's crop (1 NaN, 2 infinite position) for group_tasks_launch.
int launch_grouped_candidates(const RefineLevel& lv, const int32_t* ids, const double* loc_from, const double* history, double* pts,
                              double* box, int32_t* fail, cudaStream_t s);

// Bytes of the pre-tiled fp16 hi/lo image of an [N,K] weight matrix, and the host-side packer (returns acc_scale).
size_t tc_weight_bytes(int N, int K);
float tc_pack_weight(const float* w, int N, int K, void* dst_host);

}  // namespace cotr
