/*
 * cotr_b200 - C ABI of the H100-native COTR correspondence-inference hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch types.  The
 * reference (ubc-vision/COTR) is pure Python, so "what its FFI would bind" is
 * the L4->L3 call of the inference loop and the model construction protocol:
 *
 *   cotr_create            <- COTR/models/__init__.py:9-10  build_model(args)  +
 *                             COTR/utils/utils.py:164-193   safe_load_weights(model, state_dict)
 *                             (tensors are named by the reference's state_dict keys, SURVEY.md app. C)
 *   cotr_forward           <- COTR/models/cotr_model.py:26-40  COTR.forward(samples, queries)
 *                             as called by sparse_engine.py:52,281 and inference_helper.py:126,134,197-198
 *   cotr_encode_context    <- the query-independent part of COTR.forward: backbone.py:79-92,
 *                             cotr_model.py:37 (input_proj), transformer.py:55 (encoder) and the K/V
 *                             in-projections inside transformer.py:192-195
 *   cotr_decode            <- the per-query part: cotr_model.py:34-36 (query_proj), transformer.py:56-57
 *                             (decoder), cotr_model.py:38-39 (corr_embed, last level only)
 *   cotr_forward_host      <- the same call with HOST buffers, i.e. including the .to(device) /
 *                             .cpu() copies of sparse_engine.py:50-53
 *
 * All device pointers are fp32, contiguous.  Every call returns 0 on success; on failure it returns
 * non-zero and cotr_last_error() describes the problem (the Python wrapper raises the exception type
 * the reference would: AssertionError for a wrong canvas size, RuntimeError otherwise).
 *
 * Threading: one caller thread per model handle; one handle per device.  A model's workspace, staging buffers and
 * internal context are shared by all its entry points: calls may use different streams (each call makes its stream
 * wait for the previous call's work through an internal event), but they execute one after the other, and a
 * cotr_context must not be re-encoded while a decode on it is still in flight on another stream.  No hidden host syncs in the
 * device-pointer calls (work is enqueued on the caller's stream) except when the internal workspace has
 * to grow (first call / larger B or Q than seen before).
 */
#ifndef COTR_B200_H_
#define COTR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define COTR_CANVAS_H 256          /* COTR/utils/constants.py:2  MAX_SIZE            */
#define COTR_CANVAS_W 512          /* backbone.py:80             2 * MAX_SIZE        */
#define COTR_CONTEXT_TOKENS 512    /* 16 x 32 layer3 grid                            */
#define COTR_D_MODEL 256

typedef struct cotr_model cotr_model;       /* opaque: packed weights + workspace, bound to one device */
typedef struct cotr_context cotr_context;   /* opaque: per-pair decoder K/V cache (6 layers)           */

/* One named host tensor of the reference checkpoint (fp32, C-contiguous). */
typedef struct cotr_tensor {
    const char* name;        /* reference state_dict key, e.g. "transformer.encoder.layers.0.linear1.weight" */
    const float* data;       /* host pointer                                                                  */
    int32_t ndim;
    int64_t shape[4];
} cotr_tensor;

/* Build a model on CUDA device `device` from the 381 tensors of the reference state_dict
 * (FrozenBN buffers included; the unused decoder norm1.* entries may be present and are ignored).
 * Folds FrozenBN (backbone.py:46-56) into the conv kernels, repacks everything into kernel-native
 * layouts and uploads.  Fails if a required key is missing or has the wrong shape. */
int cotr_create(int device, const cotr_tensor* tensors, int n_tensors, cotr_model** out);
void cotr_destroy(cotr_model* m);

/* A context holds the K/V projections of all 6 decoder layers for up to `max_pairs` image pairs. */
int cotr_context_create(cotr_model* m, int max_pairs, cotr_context** out);
void cotr_context_destroy(cotr_context* c);

/* img_dev: (B,3,256,512) NCHW fp32, ImageNet-normalised, the two 256x256 images side by side. */
int cotr_encode_context(cotr_model* m, const float* img_dev, int B, cotr_context* ctx, void* cuda_stream);

/* queries_dev: (B,Q,2) fp32 (x over the 512-wide canvas, y over 256, both normalised to [0,1]);
 * pred_dev: (B,Q,2) fp32.  B must equal the B of the last cotr_encode_context on `ctx`. */
int cotr_decode(cotr_model* m, const cotr_context* ctx, const float* queries_dev, int B, int Q,
                float* pred_dev, void* cuda_stream);

/* The same two calls, also returning the head-averaged attention maps of the layers selected by `layer_mask` (bit l =
 * layer l, 0..5): the second output of the reference's nn.MultiheadAttention (need_weights=True), i.e. what a forward
 * hook on transformer.encoder.layers[l].self_attn / transformer.decoder.layers[l].multihead_attn sees as output[1].
 * attn_dev [b][i][j] = (1/8) sum over heads h = 0..7 of softmax_j(q_h[i] . k_h[j]), key j = token row * 32 + col of the
 * 16 x 32 context grid (col < 16: left image), fp32, selected layers stored in ascending order:
 *   cotr_encode_context_attention: attn_dev (popcount(layer_mask), B, 512, 512)
 *   cotr_decode_attention:         attn_dev (popcount(layer_mask), B, Q, 512)
 * layer_mask = 0 is exactly the plain call (attn_dev may be NULL); bits at 6 or above, or a NULL attn_dev with a
 * non-zero mask, fail.  Contexts and predictions are bitwise those of the plain calls: each selected layer adds one
 * launch that only reads.  Both calls run eagerly (no CUDA-graph capture). */
int cotr_encode_context_attention(cotr_model* m, const float* img_dev, int B, cotr_context* ctx, int layer_mask,
                                  float* attn_dev, void* cuda_stream);
int cotr_decode_attention(cotr_model* m, const cotr_context* ctx, const float* queries_dev, int B, int Q, int layer_mask,
                          float* attn_dev, float* pred_dev, void* cuda_stream);

/* ---- image-level feature cache ------------------------------------------------------------------------------------
 * cotr_encode_context runs the backbone over both halves of every canvas, then builds the pair context from the two
 * feature maps.  An image that takes part in many pairs (one query against a database, all ordered pairs of an image
 * set, (a|b) and (b|a)) can go through the backbone once: cotr_encode_images caches its features, and
 * cotr_encode_context_pairs builds contexts from any pairs of cached images.  A context of the pairs (2p, 2p+1) of the
 * halves of B canvases is bitwise the cotr_encode_context of those canvases, and the two calls launch exactly the
 * kernels cotr_encode_context launches (for up to 32 pairs).  Both calls run eagerly (no CUDA-graph capture). */

/* Backbone features of one 256x256 image (backbone.py:81-82: each half of a canvas goes through the ResNet body on its own):
 * the layer3 output in the library's split16 storage, plane-major [hi|lo][N][16][16][1024] fp16 = 1 MiB per image.
 * Valid for the weights of the model that made it; the bytes may be copied to the host and back. */
#define COTR_IMAGE_FEATURE_BYTES (2u * 16u * 16u * 1024u * 2u)

/* img_dev: (N,3,256,256) fp32 NCHW, ImageNet-normalised (one half of a cotr_encode_context canvas); N >= 1.
 * feat_dev: N * COTR_IMAGE_FEATURE_BYTES, 16-byte aligned.  The images go through the backbone 64 at a time, so the
 * workspace does not grow with N. */
int cotr_encode_images(cotr_model* m, const float* img_dev, int N, void* feat_dev, void* cuda_stream);

/* The context of B pairs from cached image features: pair p is the canvas [image pairs_host[2p] | image pairs_host[2p+1]]
 * (left half = the image whose queries have x < 0.5).  pairs_host: B x 2 int32 HOST array, indices in [0, n_images).
 * layer_mask / attn_dev as in cotr_encode_context_attention (0 / NULL: no maps).  The table is copied to the device
 * through a pinned staging buffer, so pairs_host may be reused as soon as the call returns; before it refills that
 * buffer the call waits for the previous call's copy out of it (only a host running a whole call ahead of the device
 * waits).  Indices are checked on the host before anything is enqueued.  The context works with
 * cotr_decode and cotr_decode_attention like one from cotr_encode_context. */
int cotr_encode_context_pairs(cotr_model* m, const void* feat_dev, int n_images, const int32_t* pairs_host, int B,
                              cotr_context* ctx, int layer_mask, float* attn_dev, void* cuda_stream);

/* Ragged decode: a different number of queries for each pair of a context in one call (the keypoints of each image of a
 * set, the surviving predictions of a cycle pass).  queries_dev: (R,2), pred_dev: (R,2), R = offsets_host[B]; pair p's
 * queries are rows offsets_host[p] .. offsets_host[p+1]-1.  B must equal the context's pair count; offsets_host (B+1
 * int64, HOST) starts at 0 and never decreases (empty pairs are allowed).  A pair's predictions do not depend on the
 * other pairs' queries: with the same count Q for every pair the call launches exactly the kernels of cotr_decode and
 * its predictions are bitwise cotr_decode's.  All arguments are checked on the host before anything is enqueued;
 * R == 0 returns 0 without a launch.  The attention tile table of the call goes to the device through a pinned staging
 * buffer, with the same wait as cotr_encode_context_pairs.  No attention maps.  Eager (no CUDA-graph capture). */
int cotr_decode_ragged(cotr_model* m, const cotr_context* ctx, const float* queries_dev, const int64_t* offsets_host,
                       int B, float* pred_dev, void* cuda_stream);

/* ---- keypoint matching across image pairs ------------------------------------------------------------------------
 * Guided matching of demo_guided_matching.py:44-62 with the whole image as the patch, on the device.  Images 0..N-1 with
 * keypoints kpts_dev: fp64 (x, y) pixels, image i's at rows kpt_offsets_host[i] .. kpt_offsets_host[i+1]-1 (N+1 int64,
 * HOST, starting at 0, never decreasing).  Pair p = (a_p, b_p) = pairs_host[2p], pairs_host[2p+1] (B x 2 int32, HOST)
 * uses two contexts: 2p = [a_p | b_p] decodes a_p's keypoints and 2p+1 = [b_p | a_p] decodes b_p's.  These rows are packed
 * in context order, R = sum over p of (K_a + K_b); off_ab[p] = the first row of context 2p.
 *   query (refinement_task.py:110):       q = fp32(x / (2 W_left)), fp32(y / H_left), divisions in fp64
 *   pixel (refinement_task.py:145-151):   c = fp64(fp32((p.x - 0.5) * 2)) * W_right, fp64(p.y) * H_right
 *   nearest (scipy distance_matrix + np.argmin): the index among the right image's keypoints minimising
 *       d = sqrt(dx dx + dy dy), dx = kp.x - c.x, all fp64 without contraction; equal d (also distinct squared sums whose
 *       sqrt rounds equal) -> the lowest index; a NaN d wins over any number and the first NaN wins; no keypoints -> -1
 *   mutual (the demo's double loop): pair p keeps (i, j = nearest_ab[i]) when nearest_ba[j] == i, in ascending i.
 * Outputs, all DEVICE: corr_dev (R,2) fp64, nearest_dev (R) int32 (an index into the right image's keypoints),
 * match_dev (R,2) int32 (pair p's matches are rows off_ab[p] .. off_ab[p] + count[p] - 1, (index into kp_a, index into
 * kp_b)), count_dev (B) int32.  No K_a x K_b buffer exists anywhere.  Every argument is checked on the host before
 * anything is enqueued.  cotr_match_keypoints stages its tables through the model's pinned buffer (waiting only as
 * cotr_encode_context_pairs does) and synchronises the device only when its buffers grow; cotr_mutual_nearest has no
 * model and copies its tables from pageable host memory, so the runtime may wait for the stream while it stages that
 * copy.  Eager (no CUDA-graph capture). */

/* The matching alone, for predictions made elsewhere (the zoom-in engines): corr_dev (R,2) fp64 pixels in the layout
 * above -> nearest_dev, match_dev, count_dev.  `device` is the CUDA device index. */
int cotr_mutual_nearest(int device, const double* kpts_dev, const int64_t* kpt_offsets_host, int n_images,
                        const int32_t* pairs_host, int B, const double* corr_dev, int32_t* nearest_dev, int32_t* match_dev,
                        int32_t* count_dev, void* cuda_stream);

/* Cached image features (cotr_encode_images) + pairs + keypoints -> mutual matches, in one call: the encoder tail of the
 * 2B contexts (as cotr_encode_context_pairs, into ctx, which needs max_pairs >= 2B), the canvas queries, the ragged decode
 * of cotr_decode_ragged, the pixels written to corr_dev, and cotr_mutual_nearest.  sizes_host: N x 2 int32 (W, H), HOST,
 * the original image sizes, 1 .. 65536 (each image was resized whole to 256 x 256 for cotr_encode_images).  It launches
 * the kernels of cotr_encode_context_pairs(2B) + cotr_decode_ragged + 4 (R == 0: + 1, the pair counts). */
int cotr_match_keypoints(cotr_model* m, const void* feat_dev, int n_images, const int32_t* sizes_host, const double* kpts_dev,
                         const int64_t* kpt_offsets_host, const int32_t* pairs_host, int B, cotr_context* ctx,
                         double* corr_dev, int32_t* nearest_dev, int32_t* match_dev, int32_t* count_dev, void* cuda_stream);

/* cotr_encode_context + cotr_decode on an internal context. */
int cotr_forward(cotr_model* m, const float* img_dev, const float* queries_dev, int B, int Q,
                 float* pred_dev, void* cuda_stream);

/* Same with host buffers (pinned or pageable): H2D, forward, D2H, stream synchronised on return. */
int cotr_forward_host(cotr_model* m, const float* img_host, const float* queries_host, int B, int Q,
                      float* pred_host);

/* Device-side replacement of the host work of RefinementTask.get_task (COTR/inference/refinement_task.py:105-120) and
 * of the canvas construction in inference_helper.py:108-113: for each of the n tasks crop a square patch out of the
 * "from" image and one out of the "to" image (uint8 HWC, 3 channels, DEVICE memory, uploaded once per engine call),
 * resize both to 256x256 with Pillow's antialiased bilinear filter (bit-exact), put them side by side and apply
 * to_tensor + normalize(mean (0.485,0.456,0.406), std (0.229,0.224,0.225)).  rects_host: n x 6 int32 HOST array
 * [x_from, y_from, size_from, x_to, y_to, size_to]; canvas_dev: (n,3,256,512) fp32 DEVICE output. */
int cotr_preprocess(cotr_model* m, const uint8_t* img_from_dev, int h_from, int w_from, const uint8_t* img_to_dev, int h_to,
                    int w_to, const int32_t* rects_host, int n, float* canvas_dev, void* cuda_stream);

/* The single-query zoom-in walk of SparseEngine with converge_iters = 1 (COTR/inference/sparse_engine.py:197-211,
 * refinement_task.py) on the device, for n fresh tasks.  A group is the tasks first .. first+count-1 of one
 * (image_from, image_to) pair with one (s_from, s_to); groups are consecutive in task order and cover 0 .. n-1.  The
 * walk takes chunks of at most `batch` consecutive tasks of one group and walks each chunk through all L = n_zoom levels
 * before the next, exactly as the host loop's batches fall: per level the crops of get_patch_centered_at (side
 * min(h, w) * clip(s * zoom_host[l], 0, 1) rounded down to even, known on the host), the canvas query, the Pillow-exact
 * canvases of cotr_preprocess, the forward of cotr_forward at (chunk, Q = 1), and scale_to_loc; after the last level
 * conclude(): good when max(std(history, axis=0)) < rel_threshold * max(h_to, w_to, 3).  All of it bit for bit.
 *   images_host: n_images uint8 HWC (3 channels) DEVICE pointers; hw_host: n_images x 2 (H, W), HOST.
 *   loc_from_dev, loc_to_dev: n x 2 fp64 (x, y) source points and first guesses, DEVICE.
 *   history_dev: n x (L+1) x 2 fp64, row 0 = the first guess, row l+1 = the location after level l.
 *   rects_dev: n x L x 6 int32 [x_from, y_from, size_from, x_to, y_to, size_to] crop of each level.
 *   good_dev: n int32, 1 when the task is good.
 * max_good is the engine's max_corrs stop: chunks run in waves of `wave` chunks; after each wave one small copy reads the
 * good counts (over the whole call, in task order), and the walk ends after the first wave in which they reached
 * max_good.  *walked_host is then exactly the number of tasks the host loop walks: every task up to the end of the chunk
 * in which the count reached max_good (n when it never did, 0 when max_good <= 0); later tasks hold no result.  With
 * max_good >= n the host waits only once, at the end.  status_host: 3 int32 [code, chunk, level]: code 0 ok, 1 a NaN
 * prediction, 2 a NaN or infinite position (clamped, not used); the walk then ends after the wave, *walked_host is the
 * first task of that chunk, and the call still returns 0.  Every argument is checked before anything is enqueued
 * (1 <= L <= 7, every crop side >= 2).  The canvases, crop table, queries and counters are model-owned and grow on demand.
 * Launches per chunk level: refine_geometry, resize_h, resize_v, the forward, refine_step. */
typedef struct cotr_refine_group {
    int32_t image_from, image_to, first, count;
    double s_from, s_to;
} cotr_refine_group;
int cotr_refine(cotr_model* m, const uint8_t* const* images_host, const int32_t* hw_host, int n_images,
                const cotr_refine_group* groups_host, int n_groups, const double* zoom_host, int n_zoom, int batch, int wave,
                int64_t max_good, double rel_threshold, const double* loc_from_dev, const double* loc_to_dev,
                double* history_dev, int32_t* rects_dev, int32_t* good_dev, int64_t* walked_host, int32_t* status_host,
                void* cuda_stream);

/* One grouped batch of FasterSparseEngine's zoom-in with converge_iters = 1 (COTR/inference/sparse_engine.py:339-369
 * form_grouped_batch and form_squad, :383-399 the batch loop of cotr_corr_multiscale, refinement_task.py:71-85
 * get_task_pilot) on the device, bit for bit.  The caller keeps the open tasks of each level and draws the permutation:
 * ids_host holds the n_ids open tasks of level `level` in the engine's shuffled order (distinct, in [0, n_tasks)).
 *   1. Candidate i gets its end points [loc_from, history row `level`] and the central-half boxes of the crops it would
 *      impose as a pilot (get_patch_centered_at, with _pilot_boxes' int64 cast); squads form as in cotr_group_tasks.
 *   2. One small copy brings back the squads: squad_host[i] = squad of candidate i or -1.  result_host: 5 int32
 *      [n_squads, longest squad, members (num_steps), stepped, status].  status 1 / 2: the crop of a pilot raises in
 *      Python (int() of a NaN / infinite position: ValueError / OverflowError); the call then stops there.
 *   3. The squads are submitted: row `level` of rects_dev of every member is its pilot's crop pair.  When max_good <= 0,
 *      or good_dev[n_tasks] >= max_good (read in the same copy, only when max_good <= n_tasks), the batch stops here
 *      (stepped 0): the engine's max_corrs stop, which comes after the batch is formed.
 *   4. Otherwise (stepped 1) the pilots' canvases, the forward of cotr_forward at (n_squads, longest) with each member's
 *      query (its own loc_from in the pilot's "from" patch; rows pilot first, then the members in list order; zero
 *      padded) and, per member, scale_to_loc with the pilot's "to" patch into history row level + 1; at the last level
 *      conclude() into good_dev[t] and the count good_dev[n_tasks].  No wait after step 2.
 *   img_*_dev: uint8 HWC (3 channels) DEVICE images; crop sides min(h, w) * clip(s * zoom_host[level], 0, 1) rounded down
 *   to even must be >= 2.  loc_from_dev: n_tasks x 2 fp64; history_dev: n_tasks x (L+1) x 2 fp64 (row 0 = first guesses,
 *   filled by the caller); rects_dev: n_tasks x L x 6 int32 as in cotr_refine; good_dev: n_tasks + 1 int32 (the caller
 *   zeroes the count before the first batch).  L = n_zoom, 1 .. 7.  Every argument is checked before anything is
 *   enqueued; the candidate tables, canvases, queries and predictions are model-owned, shared with cotr_refine, and grow
 *   on demand.  Launches: grouped_candidates, group_tasks, then refine_geometry, and when stepped resize_h, resize_v,
 *   the forward, refine_step: the level launches of cotr_refine, with squads in place of single tasks. */
int cotr_refine_grouped(cotr_model* m, const uint8_t* img_from_dev, int h_from, int w_from, const uint8_t* img_to_dev, int h_to,
                        int w_to, double s_from, double s_to, const double* zoom_host, int n_zoom, int level, const int32_t* ids_host,
                        int n_ids, int n_tasks, int batch_size, int max_load, int64_t max_good, double rel_threshold,
                        const double* loc_from_dev, double* history_dev, int32_t* rects_dev, int32_t* good_dev, int32_t* squad_host,
                        int32_t* result_host, void* cuda_stream);

/* Device-side post-processing of the dense first guess (COTR/inference/inference_helper.py:131-145, the host work of
 * cotr_patch_flow_exhaustive after the 131 072-query forward): pred_dev holds n x (256*512) x 2 fp32 predictions for the
 * grid queries (j/512, i/256) in row-major (i, j) order; out_dev receives n x 256 x 512 x 3 fp32
 * [x in the other image's [-1,1] frame, y in [-1,1], cycle-consistency confidence] exactly as the reference's
 * `corr` array before it is split into its two halves (grid_sample: bilinear, zero padding, align_corners = False). */
int cotr_dense_postprocess(cotr_model* m, const float* pred_dev, int n, float* out_dev, void* cuda_stream);

/* Device-side tail of the dense first guess for ONE (tile of a, tile of b) answer (inference_helper.py:155-160, :61-75,
 * COTR/utils/utils.py:69-83): tile_dev is a 256 x 256 x 3 fp32 block [x, y, confidence] (row pitch `pitch_floats`, e.g.
 * one half of cotr_dense_postprocess' output).  (x, y) are mapped by the 2x3 affine `affine_host` (row-major doubles:
 * x' = a0 x + a1 y + a2, y' = a3 x + a4 y + a5, what cv2.getAffineTransform gives the reference), the three channels are
 * resized to ph x pw with Pillow's mode-'F' bilinear filter (bit-exact restatement) and merged into the oh x ow canvases
 * flow_dev (oh, ow, 2) / conf_dev (oh, ow) at (px, py): a pixel takes the tile's value when the tile's confidence is <=
 * the stored one (ties go to the later tile).  first != 0 initialises the canvases (flow 0, confidence 100) beforehand. */
int cotr_flow_tile_merge(cotr_model* m, const float* tile_dev, int pitch_floats, const double* affine_host, int px, int py, int pw, int ph,
                         int ow, int oh, float* flow_dev, float* conf_dev, int first, void* cuda_stream);

/* The first guesses of the forced zoom-in for ONE direction, from its merged dense maps (the `force` branch of
 * SparseEngine.gen_tasks, COTR/inference/sparse_engine.py:224-258, with the areas of :227-228), bit for bit:
 *   counts_dev[0] = #pixels with (double)conf_from < THRESHOLD_AREA (0.02, compared in fp64: float32(0.02) lies below
 *   0.02), counts_dev[1] the same for conf_to; NaN is not counted.  int64, deterministic (integer atomics).
 *   loc_to_dev[i] = (double(flow[r, c]) * 0.5 + 0.5) * (w_to, h_to), fp64 without contraction, where
 *   r = (int)clip(y_i, 0, h_from - 1), c = (int)clip(x_i, 0, w_from - 1) with the clip in the keypoint's dtype
 *   (sparse_engine.py:255-257, :232-234).
 * flow_dev: h_from x w_from x 2 fp32 [-1,1] prediction in the "to" image; conf_from_dev: h_from x w_from fp32;
 * conf_to_dev: h_to x w_to fp32 (what cotr_flow_tile_merge leaves for the two images of the pass).  kpts_dev: n x 2
 * (x, y), float32 when kpt_is_f32 else float64, finite (the caller refuses others).  loc_to_dev: n x 2 fp64.  All DEVICE.
 * Sizes 1 .. 65536.  Every argument is checked before anything is enqueued; one memset and one kernel, no wait.
 * `device` is the CUDA device index. */
int cotr_dense_first_guess(int device, const float* flow_dev, const float* conf_from_dev, int h_from, int w_from, const float* conf_to_dev,
                           int h_to, int w_to, const void* kpts_dev, int kpt_is_f32, int n, double* loc_to_dev, int64_t* counts_dev,
                           void* cuda_stream);

/* cotr_dense_first_guess on float32 maps: the same branch with the dtype rule of 'stretching' mode, where gen_tasks
 * receives the maps from utils.float_image_resize as float32 whenever an image of the pair was stretched, bit for bit:
 *   counts_dev[0] / [1] = #pixels with conf < 0.02f, compared in float32 (float32(0.02) is NOT counted; NaN is not).
 *   loc_to_dev[i] = (double)(flow[r, c] * 0.5f + 0.5f) * (w_to, h_to): the scale and offset in float32 with separate
 *   multiply and add, then one fp64 multiply by the int64 image size (numpy's promotion).
 * Arguments, checks, pixel choice and launches as cotr_dense_first_guess. */
int cotr_dense_first_guess_f32(int device, const float* flow_dev, const float* conf_from_dev, int h_from, int w_from,
                               const float* conf_to_dev, int h_to, int w_to, const void* kpts_dev, int kpt_is_f32, int n, double* loc_to_dev,
                               int64_t* counts_dev, void* cuda_stream);

/* Whole-image resizes with Pillow's bilinear filter, bit for bit, on the device (what 'stretching' mode does on the host:
 * stretch_to_square_np and utils.float_image_resize).  An axis whose size does not change is not resampled, as in Pillow
 * (an identity pass would turn a NaN or infinite neighbour into NaN); with neither changing the output is a copy.
 *   cotr_resize_image: src_dev h x w x 3 uint8 (RGB, HWC) -> dst_dev out_h x out_w x 3 uint8, equal to
 *     PIL.Image.fromarray(src).resize((out_w, out_h), BILINEAR): 22-bit fixed-point tables, horizontal pass first with
 *     uint8 rounding and clipping in between.
 *   cotr_resize_maps: src_dev h x w x c fp32 (c = 1 .. 3, channels interleaved) -> dst_dev out_h x out_w x c fp32, equal to
 *     utils.float_image_resize (Pillow mode 'F' per channel): double coefficients and accumulation, float32 after each pass.
 * All sizes 1 .. 65536; src and dst DEVICE memory that must not overlap (maps 4-byte aligned).  Every argument is checked
 * before anything is enqueued.  The coefficient tables (per input and output size, built and uploaded on first use) and
 * the intermediate buffer are model-owned; once sizes have been seen, a call enqueues at most two kernels and never waits. */
int cotr_resize_image(cotr_model* m, const uint8_t* src_dev, int h, int w, uint8_t* dst_dev, int out_h, int out_w, void* cuda_stream);
int cotr_resize_maps(cotr_model* m, const float* src_dev, int h, int w, int c, float* dst_dev, int out_h, int out_w, void* cuda_stream);

/* Squad formation of the grouped scheduler (FasterSparseEngine.form_grouped_batch / form_squad,
 * COTR/inference/sparse_engine.py:295-369) on the device.  pts_dev: n x 4 fp64 [x_from, y_from, x_to, y_to] of the open
 * tasks of one zoom level in the engine's (already shuffled) order; box_dev: n x 8 fp64, the central-half boxes
 * [f_l, f_r, f_u, f_d, t_l, t_r, t_u, t_d] of the two crops task i would impose as a pilot.  In list order every still
 * free task becomes the pilot of a new squad and takes along the first max_load free tasks strictly inside both of its
 * boxes, until batch_size squads exist.  squad_dev[i] = squad of task i or -1, rank_dev[i] = position inside the squad
 * (0 = pilot, members in list order), *n_squads_dev = squads formed.  All arrays DEVICE memory. */
int cotr_group_tasks(int device, const double* pts_dev, const double* box_dev, int n, int batch_size, int max_load, int32_t* squad_dev,
                     int32_t* rank_dev, int32_t* n_squads_dev, void* cuda_stream);

/* The rendering half of triangulate_corr (COTR/inference/inference_helper.py:293-308; the reference rasterises the
 * Delaunay triangles of the source points with OpenGL through vispy, vertex colour = target coordinates).
 * tris_dev: n_tri x 3 vertices x 4 fp32 [x, y, u, v] (DEVICE; x, y in pixels of the H x W source image, u, v the values
 * to interpolate); out_dev: H x W x 2 fp32 (DEVICE) = barycentric interpolation of (u, v) at every pixel centre
 * (x + 0.5, y + 0.5) covered by a triangle (top-left fill rule), zero elsewhere.  `device` is the CUDA device index. */
int cotr_rasterize_triangles(int device, const float* tris_dev, int n_tri, int H, int W, float* out_dev, void* cuda_stream);

/* ---- result exchange between the GPUs of one node over NVLink peer memory -------------------------------------------
 * The reference has no multi-GPU inference; its closest call site is the loop over independent pairs of
 * demo_reconstruction.py:44-49, which BASELINE.json configs[3] / configs[4] spread over 8 GPUs.  Pairs shard, weights are
 * replicated, and the only exchange is the all-gather of every rank's block of predictions.  cotr_exchange does that
 * gather with this library's own kernels instead of a collective: a push writes the block straight into every peer's
 * symmetric buffer (nobody waits in order to send), a wait polls the local arrival flags of one step and copies the
 * gathered blocks out.  One process per GPU:
 *     cotr_exchange_create(dev, rank, world, block_bytes, slots, &ex);  cotr_exchange_handle(ex, my_handle);
 *     <all-gather the 64-byte handles with whatever the host program has: torch.distributed, MPI, a file>
 *     cotr_exchange_connect(ex, all_handles);
 *     seq = cotr_exchange_push(ex, pred_dev, bytes, stream);  ...  cotr_exchange_wait(ex, seq, gathered_dev, NULL, stream);
 * Every rank must push the same sequence of steps.  `slots` (2..64) steps are kept; a wait for a step that a faster
 * peer has meanwhile overwritten is detected (cotr_exchange_status == 2), a peer that never publishes the step within
 * ~3 s gives status 1 instead of a hang.  A rank that alternates push and wait can never be overwritten.  Sizes and device
 * addresses are multiples of 16 bytes.  One stream at a time per exchange. */
typedef struct cotr_exchange cotr_exchange;
#define COTR_EXCHANGE_HANDLE_BYTES 64
int cotr_exchange_create(int device, int rank, int world, size_t block_bytes, int slots, cotr_exchange** out);
/* handle_out: COTR_EXCHANGE_HANDLE_BYTES bytes (a cudaIpcMemHandle_t of this rank's buffer) */
int cotr_exchange_handle(cotr_exchange* ex, void* handle_out);
/* handles: world x COTR_EXCHANGE_HANDLE_BYTES bytes in rank order (the own entry is ignored) */
int cotr_exchange_connect(cotr_exchange* ex, const void* handles);
/* the same for exchanges that live in ONE process (one thread per GPU, or tests): all[r] = the exchange of rank r */
int cotr_exchange_connect_local(cotr_exchange* ex, cotr_exchange* const* all);
/* returns the step number (1, 2, ...) or -1 */
long long cotr_exchange_push(cotr_exchange* ex, const void* block_dev, size_t bytes, void* cuda_stream);
/* gathered_dev: the blocks of step `seq` concatenated in rank order (NULL: only wait); bytes_per_rank: world entries
 * (HOST), NULL = every rank pushed block_bytes */
int cotr_exchange_wait(cotr_exchange* ex, long long seq, void* gathered_dev, const size_t* bytes_per_rank, void* cuda_stream);
/* 0 ok, 1 a peer never arrived, 2 a waited step was overwritten; meaningful after the stream of the wait synchronised */
int cotr_exchange_status(const cotr_exchange* ex);
void cotr_exchange_destroy(cotr_exchange* ex);

/* cotr_forward / cotr_forward_host replay a CUDA graph per (B,Q) shape (captured on the second call with that shape;
 * inputs / outputs pass through internal staging buffers so the graph's addresses stay fixed).  0 disables it. */
int cotr_set_graph_mode(cotr_model* m, int enabled);

/* Bytes of device workspace a (B,Q) call needs (activations only, excluding weights and contexts). */
size_t cotr_workspace_bytes(int B, int Q);

/* Number of kernels the last cotr_forward / encode / decode call launched (for bench.py's gpu_launches). */
int cotr_last_launch_count(const cotr_model* m);

/* Per-launch profiler.  Between cotr_profile_begin and cotr_profile_end every kernel the library launches is bracketed
 * by two CUDA events recorded on the launching stream.  cotr_profile_end synchronises the device, fills `out` with
 * one record per launch in launch order and returns -(count + 1) on success (so 0 records -> -1), > 0 on failure.
 * kernel ids: 0 gemm_tc (wgmma), 1 gemm_simt, 2 attention_tc, 3 attention_simt, 4 layernorm, 5 maxpool,
 * 6 query_encode, 7 stem_canvas, 8 gemm_mlp (fused feed-forward block), 9 attention_weights_tc, 10 attention_weights_simt
 * (the maps of cotr_*_attention), 11 match_queries, 12 match_pixels, 13 nearest, 14 mutual (cotr_match_keypoints),
 * 15 refine_geometry, 16 resize_h, 17 resize_v, 18 refine_step (cotr_refine and cotr_refine_grouped),
 * 19 grouped_candidates, 20 group_tasks (cotr_refine_grouped), 21 dense_first_guess (reserved: cotr_dense_first_guess
 * takes no model, so its launch has no profiler to record it), 22 resize_image (cotr_resize_image), 23 resize_maps
 * (cotr_resize_maps).  For GEMMs M,N,K are the problem size; for attention and
 * attention weights M = query rows, N = 512, K = 256; for 11-13 M = rows, N = 2; for 14 M = pairs; for 15 and 18
 * M = tasks of the launch (cotr_refine_grouped: its candidates), N = level; for 16-17 M = crops; for 19-20
 * M = candidates, N = level; for 22-23 M = output rows of the pass, N = output columns, K = 0 horizontal / 1 vertical. */
typedef struct cotr_launch_record {
    int32_t kernel;
    int32_t M, N, K;
    float ms;
} cotr_launch_record;
int cotr_profile_begin(cotr_model* m, int max_records);
int cotr_profile_end(cotr_model* m, cotr_launch_record* out, int max_records);

/* Test hook: copy an intermediate of the LAST forward to the host.  name is one of
 * "feat" (2B,16,16,1024 NHWC, image n = 2*pair + half), "src" / "mem" (B*512,256 token-major),
 * "hs" (B*Q,256, final decoder LayerNorm output; only valid if B*Q fits in one decode chunk).
 * "feat" is written by cotr_encode_context only (not by cotr_encode_images / cotr_encode_context_pairs).
 * Returns the element count copied, or -1. */
int64_t cotr_debug_read(cotr_model* m, const char* name, float* out_host, int64_t max_elems);

/* Select the matrix-multiply path: 0 = wgmma tensor-core kernels (default), 1 = fp32 SIMT kernels
 * (debug / numerical cross-check only). */
int cotr_set_gemm_path(cotr_model* m, int path);

/* ---- kernel-level test hooks (used by tests/ only) ------------------------------------------------------ */
typedef struct cotr_test_gemm_desc {
    int32_t path;                 /* 0 = wgmma, 1 = fp32 SIMT                                                 */
    int32_t M, N, K;
    int32_t a_mode;               /* 0 row-major [M,K]; 1 implicit im2col over NHWC; 2 7x7/2 stem (A_dev = the fp32 (B,3,256,512) canvas, w_host [N][7][7][3]); 3 token gather */
    int32_t lda;
    int32_t H, W, C, OH, OW, KH, KW, stride, pad;   /* convolution geometry for a_mode 1 / 2                  */
    int32_t relu;
    int32_t add_period, ld_add, ldr, ldc;
    int32_t a_ln;                 /* 1: A holds PRE-LayerNorm rows (K = 256); ln_gamma / ln_beta are the norm of A,
                                     applied on the fly (deferred LayerNorm, wgmma path only)   instead of an output norm */
    int32_t res_ln;               /* 1: the residual (ldr = N = 256) is a deferred LayerNorm too, same gamma / beta   */
    int32_t emit_part;            /* 1: also write the [M][16] (mean, M2) partial row statistics of the output (N = 256) */
    int32_t reserved;
    int64_t a_elems;              /* element count of the whole A buffer, all of it converted (a_mode 0 / 1 / 3)    */
    int32_t out_rows;             /* out is (out_rows >= M, ldc >= N), 0 = M; converted in: what the launch does not write comes back */
    int32_t res_rows, res_col0;   /* residual buffer (res_rows >= M, 0 = M; ldr); the launch reads columns res_col0 ..      */
    int32_t n_pairs, n_images;    /* a_mode 3: pairs_host [n_pairs][2] images of A = (n_images,16,16,lda) features, M = 512 n_pairs */
    int32_t redirect;             /* GemmParams::blk_map: 0 none; 1 values transposed into vt_dev (vt_pairs,n_vt,256,512) fp32,
                                     converted in and out; 2 keys / values into the operand images img_dev (path 0), raw bytes */
    int32_t n_vt, vt_pairs;
    int32_t blk_map[12];
    int32_t force_bn, force_ksplit;   /* path 0: tile width (16 / 32 / 64 / 256) and split-K (1 / 2 / 4), 0 = launch rule */
    int32_t plan_bn, plan_loader, plan_dln, plan_ksplit;   /* set by the call on path 0: the plan it launched (loader
                                     0 gather, 1 im2col, 2 stem, 3 halo; dln: deferred-LayerNorm instantiation)          */
    int32_t plan_grid_x, plan_grid_y;
    int32_t plan_ln_defused;      /* 1: the LayerNorm ran as its own kernel after a narrow-tile GEMM (run_gemm's rule)   */
    int32_t reserved2;
} cotr_test_gemm_desc;
/* out = epilogue(A * W^T): A/bias/addmat/residual/ln_* /out/vt are fp32 DEVICE pointers (may be NULL where optional) -
 * the hook converts activations to / from the library's split16 storage around the kernel under test; w_host is a HOST
 * [N,K] matrix (packed for the tensor-core path internally), pairs_host a HOST int32 table.  Every argument is checked
 * before anything is launched. */
int cotr_test_gemm(cotr_test_gemm_desc* d, const float* A_dev, const float* w_host, const float* bias_dev,
                   const float* addmat_dev, const float* residual_dev, const float* ln_gamma_dev,
                   const float* ln_beta_dev, float* out_dev, float* part_out_dev /* [M][16][2] or NULL */,
                   const int32_t* pairs_host, float* vt_dev, unsigned char* img_dev);
typedef struct cotr_test_attention_desc {
    int32_t path;                 /* 0 = wgmma (attention_tc.cu), 1 = fp32 SIMT (attention_simt.cu)                */
    int32_t nq, npairs;           /* uniform layout: local pair p owns q / out rows p*nq .. p*nq+nq-1             */
    int32_t operands;             /* 0: K row-major, V transposed (fp32 SIMT schedule); 1: attention operand images,
                                     written by the tensor-core K/V projection epilogue (tensor-core schedule)        */
    int32_t slots, slot;          /* k / v hold `slots` layers side by side, as a context does; the launch reads `slot` */
    int32_t ctx_pairs, pair0;     /* k / v hold ctx_pairs pairs; the launch reads pairs pair0 ..                       */
    int32_t q_rows, ldq, q_col0;  /* q (q_rows, ldq), the launch reads its columns q_col0 .. q_col0+255; out (q_rows,256) */
    int32_t n_tiles;              /* > 0: tiles_host holds n_tiles (pair, first row, row count) triples (ragged decode) */
    int32_t key_split;            /* path 0: 0 = the launch rule, 1 or 2 = that key split                             */
    int32_t maps_rows;            /* maps_dev != NULL: maps_dev is (maps_rows, 512) ...                                 */
    int32_t maps_row0;            /* ... and local pair p, query i of the launch goes to its row maps_row0 + p*nq + i    */
    int32_t reserved;
} cotr_test_attention_desc;
/* out[r, h*32+d] = softmax(q k^T) v per head for the rows the launch owns; every other row of out is left as it was
 * passed.  q (q_rows,ldq), k / v (ctx_pairs*512, slots*256), out (q_rows,256): fp32 DEVICE; tiles_host int32 HOST or NULL.
 * maps_dev (fp32 DEVICE, or NULL: no maps): after the attention launch, the head-averaged attention maps of the same
 * operands, launched as the model launches them for cotr_*_attention (attention_weights.cu): the tensor-core kernel
 * (path 0, image operands) or the fp32 SIMT one (path 1, row-major operands); not with a tile table.  Map rows the launch
 * does not own are left as they were passed.  Every argument is checked before anything is launched. */
int cotr_test_attention(const cotr_test_attention_desc* d, const float* q_dev, const float* k_dev, const float* v_dev,
                        float* out_dev, const int32_t* tiles_host, float* maps_dev);
typedef struct cotr_test_mlp_desc {
    int32_t M;                    /* rows of the launch                                                             */
    int32_t rows;                 /* rows of x and out (>= M)                                                        */
    int32_t split;                /* 0 = the launch rule, 4 or 8 = CTAs per row tile                                  */
    int32_t in_place;             /* 1: the launch writes into x (out == x, as the decoder runs it); out receives x after */
} cotr_test_mlp_desc;
/* The fused feed-forward block (mlp_tc.cu): out = LN(x + relu(x W1^T + b1) W2^T + b2) [then LN2 when g2 / be2 are given]
 * on rows < M; rows >= M of out are left as they were passed.  x / out (rows,256), b1 (1024), b2 / g / be / g2 / be2 (256):
 * fp32 DEVICE; w1 [1024,256], w2 [256,1024]: fp32 HOST. */
int cotr_test_mlp(const cotr_test_mlp_desc* d, const float* x_dev, const float* w1_host, const float* b1_dev,
                  const float* w2_host, const float* b2_dev, const float* g_dev, const float* be_dev,
                  const float* g2_dev, const float* be2_dev, float* out_dev);
/* Row kernels: op 0 LayerNorm of a split16 input, 1 LayerNorm of an fp32 input, 2 LN2(LN1(x)) (g2 / b2),
 * 3 lin_sine query encoding of (rows,2) points in [0,1] (in; g1 .. b2 unused).  in (rows,256), out (rows,256): DEVICE. */
int cotr_test_rowwise(int op, int rows, const float* in_dev, const float* g1_dev, const float* b1_dev,
                      const float* g2_dev, const float* b2_dev, float* out_dev);
/* The per-task arithmetic of cotr_refine run on the HOST (the same __host__ __device__ functions), n rows:
 * op 0 crop: in [pos_x, pos_y, scale], in_i [h, w] -> out_i [left, top, size, flag] (size -1: NaN scale; flag 1: NaN or
 * infinite position, clamped); op 1 query: in [x, y], in_i [px, py, size] -> out fp32 [qx, qy]; op 2 scale_to_loc:
 * in fp32 [p_x, p_y], in_i [px, py, size] -> out [x, y]; op 3 conclude: in (levels+1) x 2 history, in_i [h_to, w_to]
 * -> out_i good. */
int cotr_test_refine_math(int op, int n, int levels, double rel_threshold, const double* in, const int32_t* in_i,
                          double* out, int32_t* out_i);
/* The candidate kernel of cotr_refine_grouped on n candidates: pts_host n x 4 fp64 [x_from, y_from, x_to, y_to] (HOST),
 * geom_host [h_from, w_from, h_to, w_to, size_from, size_to] -> box_host n x 8 fp64 pilot boxes, fail_host n int32
 * (0, 1 NaN, 2 infinite position: the exception the pilot's crop raises in Python).  `device` is the CUDA device index. */
int cotr_test_pilot_boxes(int device, const double* pts_host, int n, const int32_t* geom_host, double* box_host, int32_t* fail_host);
/* bring-up / A-B switches (0 = production): bit 8 (256) disables programmatic dependent launch, bit 9 (512) disables
 * split-K, bits 10-11 move the CTA-count threshold of the 64-wide GEMM tile, bits 14-15 lower the
 * minimum K of split-K (16 >> n chunks of 64).  Schedule: by default a transformer section with >= 2048 rows runs the
 * deferred-LayerNorm schedule (no LayerNorm launches), smaller ones the explicit one, in which each feed-forward block
 * (linear1, linear2, its LayerNorm) is one fused launch on the tensor-core path; bit 19 forces deferred everywhere,
 * bit 16 never and runs every feed-forward block as separate linear1 / linear2 / LayerNorm launches.  Bit 20 (1048576)
 * runs the 3x3 stride-1 convolutions on the implicit-im2col loader instead of the halo loader (same launches).
 * Process-wide; graphs captured under another value are NOT dropped (call cotr_set_gemm_path twice to drop them). */
void cotr_debug_set_variant(int variant);

const char* cotr_last_error(void);
const char* cotr_version(void);

#ifdef __cplusplus
}
#endif
#endif /* COTR_B200_H_ */
