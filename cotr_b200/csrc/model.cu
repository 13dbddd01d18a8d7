// Model state, weight packing, workspace and the forward schedule behind the C ABI (include/cotr_b200.h).
//
// Reference lines restated by each stage are cited inline (paths relative to the reference root).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "../../include/cotr_b200.h"
#include "common.cuh"

namespace cotr {

extern int g_tc_variant;
static thread_local char g_error[1024] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

namespace {

constexpr int kDecodeChunkRows = 32768;   // decoder rows processed per pass (rows are independent, so chunking is exact)
constexpr int kKCols = kDecLayers * kDModel;         // 1536: K of all decoder layers, [layer][256]
constexpr int kQpCols = kDecLayers * kDModel;        // 1536
constexpr size_t kVtLayer = (size_t)kDModel * kTokens;   // one transposed value projection [256][512]

struct DevConv {
    float* w = nullptr;    // [cout][kh][kw][cin], FrozenBN scale folded in
    void* wtc = nullptr;   // tensor-core image of w
    float wtc_scale = 1.f; // accumulator scale that undoes the image's power-of-two pre-scaling
    float* b = nullptr;    // FrozenBN shift
    int cout = 0, cin = 0, kh = 1, kw = 1, stride = 1, pad = 0;
    bool stem = false;     // 7x7/2 stem over the bordered NHWC4 canvas: kw = 8 pixel slots, cin = 4 (common.cuh)
};

struct DevLinear {
    float* w = nullptr;    // [N][K]
    void* wtc_plain = nullptr;       // tensor-core image of W (explicit-LayerNorm schedule)
    float wtc_plain_scale = 1.f;
    void* wtc = nullptr;             // image of the deferred-LayerNorm schedule: wtc_plain unless built by make_linear_ln
    float wtc_scale = 1.f;
    float* b = nullptr;    // [N] or null
    int n = 0, k = 0;
    // Deferred LayerNorm on the input (tensor-core path, GemmParams::a_ln_cs): wtc then holds W diag(gamma),
    // cs its column sums and b_tc = beta W^T + b; w / b stay the checkpoint's values for the fp32 SIMT path.
    float* cs = nullptr;
    float* b_tc = nullptr;
};

struct Block {
    DevConv c1, c2, c3, ds;
    bool has_ds = false;
};

struct EncLayer {
    DevLinear qkv;         // [768][256]; q rows pre-scaled by head_dim^-0.5; bias folded into add_qkv
    float* add_qkv = nullptr;   // [512][768] = [ (pos Wq^T + bq) s | pos Wk^T + bk | bv ]
    float* add_qkv_tc = nullptr;   // + beta W^T of the previous layer's norm2 (deferred LayerNorm, layers > 0)
    DevLinear o, l1, l2;
    float *ln1_g, *ln1_b, *ln2_g, *ln2_b;
};
static_assert(sizeof(float2) == 8, "row statistics are (mean, rstd) pairs");

struct DecLayer {
    DevLinear q;           // [256][256] pre-scaled, no bias (bias lives in the qpos projection)
    DevLinear o, l1, l2;
    float *ln2_g, *ln2_b, *ln3_g, *ln3_b;
};

const Split16 kNoSplit = {nullptr, nullptr};

// Sizes of the zoom-in walks' workspace: crop pairs (squads) of one level, its query rows, the entries of one level
// launch, horizontal-pass bytes and cotr_refine's chunks.
struct RefineCaps {
    int64_t squads = 0, rows = 0, ids = 0, chunks = 0;
    size_t tmp = 0;
};

struct Workspace {
    int cap_pairs = 0;
    int cap_rows = 0;
    // backbone (per image sizes x 2*cap_pairs), all split16
    Split16 canvas = kNoSplit, stem = kNoSplit, bx = kNoSplit, by = kNoSplit, bt1 = kNoSplit, bt2 = kNoSplit, bds = kNoSplit;
    // encoder
    Split16 src = kNoSplit, xa = kNoSplit, xb = kNoSplit, qk = kNoSplit, vt = kNoSplit, ao = kNoSplit, ffh = kNoSplit;
    int* pair_id = nullptr;              // [pairs][2] = (2p, 2p+1): input_proj's image table for canvases (constant, graph-safe)
    unsigned char* kvimg = nullptr;      // [pairs][8 heads] attention operand images of the encoder's own k / v
    float* ln_tmp = nullptr;      // fp32 [tokens][256]: pre-LayerNorm rows of the SIMT cross-check path
    float2 *enc_st_a = nullptr, *enc_st_b = nullptr;     // [tokens][16] partial row statistics of xa / xb (deferred LayerNorms)
    // decoder
    Split16 qpos = kNoSplit, qp = kNoSplit, t = kNoSplit, qb = kNoSplit, dao = kNoSplit, dh = kNoSplit, hs = kNoSplit,
            hd1 = kNoSplit, hd2 = kNoSplit, t2 = kNoSplit;
    float* dln_tmp = nullptr;
    float2 *dec_st_a = nullptr, *dec_st_b = nullptr;
    // host-buffer entry point staging
    float *img_stage = nullptr, *q_stage = nullptr, *pred_stage = nullptr;
    size_t img_stage_elems = 0, q_stage_elems = 0;
    // keypoint matching (cotr_match_keypoints): the (rows,2) canvas queries and predictions of one call
    int64_t cap_match_rows = 0;
    float *match_q = nullptr, *match_pred = nullptr;
    // zoom-in walks (cotr_refine, cotr_refine_grouped): one level's canvases, crop table, horizontal-pass bytes and
    // (squads, longest) queries and predictions; the status word followed by cotr_refine's per-chunk good counts; the
    // squad tables of cotr_refine's squads of one (0 .. ids-1 and zeros); cotr_refine_grouped's candidate end points and
    // pilot boxes and its table [n_squads | squad | fail | rank]
    RefineCaps cap_refine;
    float *refine_canvas = nullptr, *refine_q = nullptr, *refine_pred = nullptr;
    CropSide* refine_sides = nullptr;
    unsigned char* refine_tmp = nullptr;
    unsigned long long* refine_counts = nullptr;
    int32_t *refine_iota = nullptr, *refine_zeros = nullptr;
    double *grouped_pts = nullptr, *grouped_box = nullptr;
    int32_t* grouped_tab = nullptr;
};

// A host table that reaches the device with one asynchronous copy per call, staged through pinned memory.  `copied` is
// recorded after each copy out of `stage`; the host rewrites `stage` only once that copy has completed, which it has
// long done unless the host runs a whole call ahead of the device.
template <class T>
struct PinnedTable {
    T* dev = nullptr;
    T* stage = nullptr;
    size_t cap = 0;
    cudaEvent_t copied = nullptr;
    ~PinnedTable() {
        if (dev) cudaFree(dev);
        if (stage) cudaFreeHost(stage);
        if (copied) cudaEventDestroy(copied);
    }
    int upload(const T* src, size_t n, cudaStream_t s) {
        if (n > cap) {
            COTR_CHECK_CUDA(cudaDeviceSynchronize());
            cap = 0;      // a failed allocation below leaves no capacity behind, so the next call allocates again
            if (dev) { cudaFree(dev); dev = nullptr; }
            if (stage) { cudaFreeHost(stage); stage = nullptr; }
            COTR_CHECK_CUDA(cudaMalloc((void**)&dev, n * sizeof(T)));
            COTR_CHECK_CUDA(cudaMallocHost((void**)&stage, n * sizeof(T)));
            cap = n;
        }
        if (!copied) COTR_CHECK_CUDA(cudaEventCreateWithFlags(&copied, cudaEventDisableTiming));
        COTR_CHECK_CUDA(cudaEventSynchronize(copied));
        memcpy(stage, src, n * sizeof(T));
        COTR_CHECK_CUDA(cudaMemcpyAsync(dev, stage, n * sizeof(T), cudaMemcpyHostToDevice, s));
        COTR_CHECK_CUDA(cudaEventRecord(copied, s));
        return 0;
    }
};

}  // namespace
}  // namespace cotr

struct cotr_context {
    cotr_model* model = nullptr;
    cotr::Split16 k = cotr::kNoSplit;    // [max_pairs * 512][6 * 256]
    cotr::Split16 vt = cotr::kNoSplit;   // [max_pairs][6][256][512]  (value projections stored transposed)
    unsigned char* img = nullptr;        // [max_pairs][6][8 heads] attention operand images (common.cuh kAttnHeadImgBytes)
    bool holds_img = false;              // what the last encode wrote: images (tensor-core path) or k / vt (fp32 SIMT path)
    int max_pairs = 0;
    int pairs = 0;                       // pairs encoded by the last cotr_encode_context
};

struct cotr_model {
    int device = 0;
    int gemm_path = 0;          // 0 = tensor cores (wgmma), 1 = fp32 SIMT
    int launches = 0;
    std::vector<void*> allocs;
    cotr::DevConv stem;
    std::vector<cotr::Block> blocks;
    cotr::DevLinear proj;
    cotr::EncLayer enc[cotr::kEncLayers];
    cotr::DevLinear kv_all;     // [3072][256] rows [l*512, l*512+256) = Wk_l, [l*512+256, l*512+512) = Wv_l
    float* add_kv = nullptr;    // [512][3072]
    float* add_kv_tc = nullptr; // + beta W^T of the last encoder norm2 (deferred LayerNorm)
    cotr::DevLinear qpos_all;   // [1536][256] pre-scaled, bias pre-scaled
    cotr::DecLayer dec[cotr::kDecLayers];
    float *dec_norm_g = nullptr, *dec_norm_b = nullptr;
    cotr::DevLinear head[3];
    float* pos = nullptr;       // [512][256] grid position embedding (fp32, debug / tests)
    cotr::Workspace ws;
    cotr_context* own_ctx = nullptr;
    cudaStream_t host_stream = nullptr;
    cotr::Split16 last_feat = cotr::kNoSplit;
    cotr::Split16 last_mem = cotr::kNoSplit;
    bool last_mem_pre_ln = false;   // tensor-core path: last_mem holds the rows BEFORE the last encoder norm2
    int last_pairs = 0, last_rows = 0;
    // per-launch profiler (cotr_profile_begin / cotr_profile_end): CUDA event pairs on the launching stream
    // CUDA-graph replay of cotr_forward, one executable graph per (B, Q) shape (captured on the second call)
    bool graph_mode = true;
    std::map<long long, cudaGraphExec_t> graphs;
    std::map<long long, int> graph_launches;
    std::set<long long> shapes_seen;
    cotr::PinnedTable<int> pair_tab;     // cotr_encode_context_pairs: the caller's (B,2) image table
    cotr::PinnedTable<int4> tile_tab;    // cotr_decode_ragged: the attention tile tables of all chunks of a call (AttnParams::tiles)
    cotr::PinnedTable<int4> match_tab;   // cotr_match_keypoints: the match tiles and pair table of a call (MatchPlan::tab)
    cotr::PinnedTable<int32_t> grouped_ids;   // cotr_refine_grouped: the batch's permuted candidate task ids
    cotr::Preprocessor* pre = nullptr;         // device-side crop / resize / normalise (cotr_preprocess)
    cotr::FlowMerger* merger = nullptr;        // device-side tail of the dense first guess (cotr_flow_tile_merge)
    cotr::Resizer* resizer = nullptr;          // whole-image resizes (cotr_resize_image, cotr_resize_maps)
    bool prof_on = false;
    std::vector<cudaEvent_t> prof_events;      // 2 per record
    std::vector<cotr_launch_record> prof_records;
    int prof_max = 0;
    // The workspace, the staging buffers and own_ctx are shared by every entry point: consecutive calls on different
    // streams are ordered with this event (recorded at the end of each call, waited for by the next call's stream).
    cudaEvent_t order_event = nullptr;
    cudaStream_t order_stream = nullptr;
    bool order_valid = false;
};

namespace cotr {
namespace {

// ----------------------------------------------------------------------------------------------
// weight lookup / upload helpers
// ----------------------------------------------------------------------------------------------
struct TensorMap {
    std::map<std::string, const cotr_tensor*> m;
    const cotr_tensor* get(const std::string& name, std::initializer_list<int64_t> shape) const {
        auto it = m.find(name);
        if (it == m.end()) { set_error("cotr_create: missing tensor '%s'", name.c_str()); return nullptr; }
        const cotr_tensor* t = it->second;
        if (t->ndim != (int)shape.size()) { set_error("cotr_create: '%s' has ndim %d, expected %zu", name.c_str(), t->ndim, shape.size()); return nullptr; }
        int i = 0;
        for (int64_t s : shape) {
            if (t->shape[i] != s) { set_error("cotr_create: '%s' dim %d is %lld, expected %lld", name.c_str(), i, (long long)t->shape[i], (long long)s); return nullptr; }
            ++i;
        }
        if (!t->data) { set_error("cotr_create: '%s' has a null data pointer", name.c_str()); return nullptr; }
        return t;
    }
};

int dev_alloc(cotr_model* m, void** p, size_t bytes) {
    COTR_CHECK_CUDA(cudaMalloc(p, bytes ? bytes : 4));
    m->allocs.push_back(*p);
    return 0;
}

int upload(cotr_model* m, const std::vector<float>& h, float** d) {
    if (dev_alloc(m, (void**)d, h.size() * sizeof(float))) return 1;
    COTR_CHECK_CUDA(cudaMemcpy(*d, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice));
    return 0;
}

int upload_tc(cotr_model* m, const std::vector<float>& w, int N, int K, void** d, float* acc_scale) {
    const size_t bytes = tc_weight_bytes(N, K);
    std::vector<uint8_t> img(bytes);
    *acc_scale = tc_pack_weight(w.data(), N, K, img.data());
    if (dev_alloc(m, d, bytes)) return 1;
    COTR_CHECK_CUDA(cudaMemcpy(*d, img.data(), bytes, cudaMemcpyHostToDevice));
    return 0;
}

int make_linear(cotr_model* m, const std::vector<float>& w, const std::vector<float>* b, int N, int K, DevLinear* out) {
    out->n = N; out->k = K;
    if (upload(m, w, &out->w)) return 1;
    if (upload_tc(m, w, N, K, &out->wtc_plain, &out->wtc_plain_scale)) return 1;
    out->wtc = out->wtc_plain; out->wtc_scale = out->wtc_plain_scale;
    if (b) { if (upload(m, *b, &out->b)) return 1; }
    return 0;
}

// A linear layer W [N][K] + b (b may be null) whose input is a deferred LayerNorm (gamma, beta): the tensor-core GEMM
// multiplies by w = W diag(gamma), its epilogue takes the column sums cs of w and the folded bias b = beta W^T + b
// (see GemmParams::a_ln_cs).  The sums are taken in double.
struct LnFold {
    std::vector<float> w, cs, b;
};
LnFold fold_ln(const float* w, const float* b, int N, int K, const float* gamma, const float* beta) {
    LnFold f;
    f.w.resize((size_t)N * K); f.cs.resize(N); f.b.resize(N);
    for (int n = 0; n < N; ++n) {
        double s = 0.0, c = b ? (double)b[n] : 0.0;
        for (int k = 0; k < K; ++k) {
            const float v = w[(size_t)n * K + k] * gamma[k];
            f.w[(size_t)n * K + k] = v;
            s += (double)v;
            c += (double)w[(size_t)n * K + k] * (double)beta[k];
        }
        f.cs[n] = (float)s;
        f.b[n] = (float)c;
    }
    return f;
}

// Linear layer whose input is a deferred LayerNorm (gamma, beta): wtc holds the folded image (fold_ln), wtc_plain the
// image of W itself.
int make_linear_ln(cotr_model* m, const std::vector<float>& w, const std::vector<float>* b, int N, int K,
                   const float* gamma, const float* beta, DevLinear* out, std::vector<float>* folded_bias = nullptr) {
    out->n = N; out->k = K;
    if (upload(m, w, &out->w)) return 1;
    if (b) { if (upload(m, *b, &out->b)) return 1; }
    const LnFold f = fold_ln(w.data(), b ? b->data() : nullptr, N, K, gamma, beta);
    if (upload_tc(m, f.w, N, K, &out->wtc, &out->wtc_scale)) return 1;
    if (upload_tc(m, w, N, K, &out->wtc_plain, &out->wtc_plain_scale)) return 1;
    if (upload(m, f.cs, &out->cs) || upload(m, f.b, &out->b_tc)) return 1;
    if (folded_bias) *folded_bias = f.b;
    return 0;
}

// backbone.py:46-56 folded into the conv: w' = w * s[o], shift = b - rm * s, s = weight * (rv + 1e-5)^-1/2.
// [cout][7][7][3] (kh, kw, c) -> [cout][7][8][4]: the K order of A_STEM_NHWC4 (common.cuh), zero weights for pixel slot 7 / channel 3
std::vector<float> stem_weight_order(const std::vector<float>& w, int cout) {
    std::vector<float> o((size_t)cout * kStemK, 0.f);
    for (int n = 0; n < cout; ++n)
        for (int y = 0; y < 7; ++y)
            for (int x = 0; x < 7; ++x)
                for (int c = 0; c < 3; ++c)
                    o[(size_t)n * kStemK + y * 32 + x * 4 + c] = w[(((size_t)n * 7 + y) * 7 + x) * 3 + c];
    return o;
}

int make_conv(cotr_model* m, const TensorMap& tm, const std::string& conv, const std::string& bn,
              int cout, int cin, int kh, int kw, int stride, int pad, DevConv* out) {
    const cotr_tensor* w = tm.get(conv + ".weight", {cout, cin, kh, kw});
    const cotr_tensor* g = tm.get(bn + ".weight", {cout});
    const cotr_tensor* b = tm.get(bn + ".bias", {cout});
    const cotr_tensor* rm = tm.get(bn + ".running_mean", {cout});
    const cotr_tensor* rv = tm.get(bn + ".running_var", {cout});
    if (!w || !g || !b || !rm || !rv) return 1;
    std::vector<float> wf((size_t)cout * kh * kw * cin), bf(cout);
    for (int o = 0; o < cout; ++o) {
        const double s = (double)g->data[o] / std::sqrt((double)rv->data[o] + 1e-5);
        bf[o] = (float)((double)b->data[o] - (double)rm->data[o] * s);
        for (int c = 0; c < cin; ++c)
            for (int y = 0; y < kh; ++y)
                for (int x = 0; x < kw; ++x)
                    wf[(((size_t)o * kh + y) * kw + x) * cin + c] =
                        (float)((double)w->data[(((size_t)o * cin + c) * kh + y) * kw + x] * s);
    }
    out->cout = cout; out->cin = cin; out->kh = kh; out->kw = kw; out->stride = stride; out->pad = pad;
    if (kh == 7 && cin == 3) {      // the stem reads the bordered NHWC4 canvas: K = (kh, 8 pixel slots, 4 channels), zeros in the padding
        wf = stem_weight_order(wf, cout);
        out->kw = 8; out->cin = 4; out->stem = true;
    }
    if (upload(m, wf, &out->w)) return 1;
    if (upload_tc(m, wf, cout, out->kh * out->kw * out->cin, &out->wtc, &out->wtc_scale)) return 1;
    if (upload(m, bf, &out->b)) return 1;
    return 0;
}

std::vector<float> to_vec(const cotr_tensor* t, size_t n, size_t offset = 0) {
    return std::vector<float>(t->data + offset, t->data + offset + n);
}

int upload_vec(cotr_model* m, const TensorMap& tm, const std::string& name, int n, float** d) {
    const cotr_tensor* t = tm.get(name, {n});
    if (!t) return 1;
    return upload(m, to_vec(t, n), d);
}

// position_encoding.py:60-72 for the all-False mask of the 16x32 grid, evaluated like the reference in fp32.
std::vector<float> grid_position_table() {
    std::vector<float> pos((size_t)kTokens * kDModel);
    for (int i = 0; i < 16; ++i)
        for (int j = 0; j < 32; ++j) {
            const float y = ((float)(i + 1) - 0.5f) / ((float)16 + 1e-6f);
            const float x = ((float)(j + 1) - 0.5f) / ((float)32 + 1e-6f);
            float* row = pos.data() + (size_t)(i * 32 + j) * kDModel;
            for (int k = 1; k <= 64; ++k) {
                const float kpi = (float)((double)k * 3.14159265358979323846);
                const float ax = kpi * x, ay = kpi * y;
                row[2 * (k - 1) + 0] = (float)std::sin((double)ax);
                row[2 * (k - 1) + 1] = (float)std::sin((double)ay);
                row[128 + 2 * (k - 1) + 0] = (float)std::cos((double)ax);
                row[128 + 2 * (k - 1) + 1] = (float)std::cos((double)ay);
            }
        }
    return pos;
}

// ----------------------------------------------------------------------------------------------
// launch helpers (all kernel launches of the forward go through these, so they can be counted / profiled)
// ----------------------------------------------------------------------------------------------
struct Run {
    cotr_model* m;
    cudaStream_t s;
};

enum KernelId { K_GEMM_TC = 0, K_GEMM_SIMT = 1, K_ATTN_TC = 2, K_ATTN_SIMT = 3, K_LAYERNORM = 4, K_MAXPOOL = 5, K_QENC = 6, K_STEM_CANVAS = 7,
                K_GEMM_MLP = 8, K_ATTN_WEIGHTS_TC = 9, K_ATTN_WEIGHTS_SIMT = 10, K_MATCH_QUERIES = 11, K_MATCH_PIXELS = 12,
                K_NEAREST = 13, K_MUTUAL = 14, K_REFINE_GEOMETRY = 15, K_RESIZE_H = 16, K_RESIZE_V = 17, K_REFINE_STEP = 18,
                K_GROUPED_CANDIDATES = 19, K_GROUP_TASKS = 20, K_DENSE_FIRST_GUESS = 21, K_RESIZE_IMAGE = 22, K_RESIZE_MAPS = 23 };

// Counts the launch and, when the profiler is on, brackets it with two events on the launching stream.
struct LaunchScope {
    cotr_model* m;
    cudaStream_t s;
    int slot = -1;
    LaunchScope(const Run& r, int kernel, int M, int N, int K) : m(r.m), s(r.s) {
        m->launches++;
        if (!m->prof_on || (int)m->prof_records.size() >= m->prof_max) return;
        slot = (int)m->prof_records.size();
        while ((int)m->prof_events.size() < 2 * (slot + 1)) {
            cudaEvent_t e;
            if (cudaEventCreate(&e) != cudaSuccess) { slot = -1; return; }
            m->prof_events.push_back(e);
        }
        cotr_launch_record rec;
        rec.kernel = kernel; rec.M = M; rec.N = N; rec.K = K; rec.ms = 0.f;
        m->prof_records.push_back(rec);
        cudaEventRecord(m->prof_events[2 * slot], s);
    }
    ~LaunchScope() {
        if (slot >= 0) cudaEventRecord(m->prof_events[2 * slot + 1], s);
    }
};

GemmParams gemm_base(int M, int N, int K, CSplit16 A, int lda, const float* W, const void* Wtc, float wtc_scale,
                     Split16 out, int ldc) {
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.M = M; p.N = N; p.K = K;
    p.a = A; p.a_mode = A_ROWMAJOR; p.lda = lda;
    p.Wt = W; p.Wtc = Wtc; p.acc_scale = wtc_scale;
    p.out = out; p.ldc = ldc;
    p.add_period = 1;
    return p;
}

// GEMM of linear layer L; folded: with the deferred-LayerNorm schedule's weight image (DevLinear::wtc)
GemmParams gemm_linear(const DevLinear& L, bool folded, int M, CSplit16 A, int lda, Split16 out, int ldc) {
    if (folded) return gemm_base(M, L.n, L.k, A, lda, L.w, L.wtc, L.wtc_scale, out, ldc);
    return gemm_base(M, L.n, L.k, A, lda, L.w, L.wtc_plain, L.wtc_plain_scale, out, ldc);
}

// Redirects the 256-column blocks of a key / value projection (GemmParams::remap): the blocks before kv0 keep their
// columns, then come `slots` (key, value) block pairs.  The keys of slot l go to columns k_col0 + 256 l of the output,
// or into slot l's attention operand images when kv_img is set; the values go transposed to slot l of vt, or into the
// images.
void redirect_kv(GemmParams& p, int kv0, int slots, int k_col0, Split16 vt, unsigned char* kv_img) {
    p.remap = 1;
    for (int b = 0; b < kv0; ++b) p.blk_map[b] = b * kDModel;
    for (int l = 0; l < slots; ++l) {
        p.blk_map[kv0 + 2 * l] = kv_img ? -1000 - l : k_col0 + l * kDModel;
        p.blk_map[kv0 + 2 * l + 1] = -(l + 1);
    }
    p.vt = vt; p.n_vt = slots;
    p.kv_img = kv_img;
}

// The fused LayerNorm epilogue needs the whole 256-wide row in one CTA (128 x 256 tile): with few rows that is a
// handful of CTAs doing a long serial epilogue while the other SMs idle.  Below 64 row tiles the GEMM runs with narrow
// tiles across many SMs and LayerNorm follows as its own (in-place, one warp per row) kernel.
inline bool ln_defused(int M) { return (M + 127) / 128 < 64; }

int launch_tc(const Run& r, const GemmParams& p) {
    LaunchScope scope(r, K_GEMM_TC, p.M, p.N, p.K);
    return launch_gemm_tc(p, r.s);
}

// ln_scratch: fp32 [M][256] staging for the SIMT path (the tensor-core GEMM fuses LayerNorm into its epilogue).
int run_gemm(const Run& r, GemmParams p, float* ln_scratch) {
    if (r.m->gemm_path == 0 && p.ln_gamma == nullptr) return launch_tc(r, p);
    if (r.m->gemm_path == 0) {
        const bool defuse = p.ln_gamma != nullptr && ln_defused(p.M);
        const float* g = p.ln_gamma;
        const float* b = p.ln_beta;
        if (defuse) { p.ln_gamma = nullptr; p.ln_beta = nullptr; }
        if (launch_tc(r, p)) return 1;
        if (defuse) {
            LaunchScope scope(r, K_LAYERNORM, p.M, kDModel, 0);
            if (launch_layernorm(cs(p.out), g, b, p.out, p.M, r.s)) return 1;
        }
        return 0;
    }
    const float* g = p.ln_gamma;
    const float* b = p.ln_beta;
    if (g) {
        COTR_CHECK(p.N == kDModel && ln_scratch != nullptr, "run_gemm: LayerNorm epilogue needs N = 256");
        p.ln_gamma = nullptr; p.ln_beta = nullptr;
    }
    {
        LaunchScope scope(r, K_GEMM_SIMT, p.M, p.N, p.K);
        if (launch_gemm_simt_raw(p, g ? ln_scratch : nullptr, r.s)) return 1;
    }
    if (g) {
        LaunchScope scope(r, K_LAYERNORM, p.M, kDModel, 0);
        if (launch_layernorm_f32(ln_scratch, g, b, Split16{p.out.hi, p.out.lo}, p.M, r.s)) return 1;
    }
    return 0;
}

int run_linear(const Run& r, const DevLinear& L, int M, CSplit16 A, int lda, Split16 out, int ldc, bool relu,
               CSplit16 residual = CSplit16{nullptr, nullptr}, int ldr = 0, const float* ln_g = nullptr,
               const float* ln_b = nullptr, float* ln_scratch = nullptr) {
    GemmParams p = gemm_linear(L, false, M, A, lda, out, ldc);
    p.bias = L.b;
    p.relu = relu ? 1 : 0;
    p.res = residual; p.ldr = ldr;
    p.ln_gamma = ln_g; p.ln_beta = ln_b;
    return run_gemm(r, p, ln_scratch);
}

// Tensor-core path only: out = LN(x + linear2(relu(linear1(x)))) [-> LN(g2, b2)] in one launch (mlp_tc.cu).  Recorded as
// M = rows, N = 1024, K = 512, so that 2 M N K is the FLOP count of both GEMMs.
int run_mlp(const Run& r, const DevLinear& l1, const DevLinear& l2, int M, CSplit16 x, Split16 out, const float* g, const float* b,
            const float* g2 = nullptr, const float* b2 = nullptr) {
    MlpParams p;
    memset(&p, 0, sizeof(p));
    p.M = M; p.x = x; p.out = out;
    p.w1 = l1.wtc_plain; p.w1_scale = l1.wtc_plain_scale; p.b1 = l1.b;
    p.w2 = l2.wtc_plain; p.w2_scale = l2.wtc_plain_scale; p.b2 = l2.b;
    p.g = g; p.be = b; p.g2 = g2; p.be2 = b2;
    LaunchScope scope(r, K_GEMM_MLP, M, kFF, 2 * kDModel);
    return launch_mlp_tc(p, r.s);
}

// Tensor-core path only: linear layer with deferred LayerNorms (GemmParams::a_ln_cs / res_ln_part / ln_part_out).
//   a_part     non-null: A holds pre-LayerNorm rows with these partial statistics; L was built by make_linear_ln
//   part_out   non-null: the output rows are pre-LayerNorm rows of a later norm - leave their partial statistics here
//   res_part   non-null: the residual operand is a deferred LayerNorm (res_g, res_b) of the stored rows
int run_linear_dln(const Run& r, const DevLinear& L, int M, CSplit16 A, int lda, Split16 out, int ldc, bool relu,
                   const float2* a_part, float2* part_out, CSplit16 residual = CSplit16{nullptr, nullptr}, int ldr = 0,
                   const float2* res_part = nullptr, const float* res_g = nullptr, const float* res_b = nullptr) {
    GemmParams p = gemm_linear(L, true, M, A, lda, out, ldc);
    p.bias = a_part ? L.b_tc : L.b;
    p.relu = relu ? 1 : 0;
    p.res = residual; p.ldr = ldr;
    if (a_part) { p.a_ln_cs = L.cs; p.a_ln_part = a_part; }
    p.ln_part_out = part_out;
    p.res_ln_part = res_part; p.res_ln_gamma = res_g; p.res_ln_beta = res_b;
    return launch_tc(r, p);
}

int run_conv(const Run& r, const DevConv& c, int n_img, CSplit16 in, int H, int W, Split16 out, bool relu, CSplit16 residual) {
    const int OH = c.stem ? H / 2 : (H + 2 * c.pad - c.kh) / c.stride + 1;
    const int OW = c.stem ? W / 2 : (W + 2 * c.pad - c.kw) / c.stride + 1;
    GemmParams p = gemm_base(n_img * OH * OW, c.cout, c.kh * c.kw * c.cin, in, c.cin, c.w, c.wtc, c.wtc_scale, out, c.cout);
    if (c.stem) {
        p.a_mode = A_STEM_NHWC4;        // `in` is the bordered canvas (launch_stem_canvas)
    } else if (c.kh == 1 && c.kw == 1 && c.stride == 1) {
        p.a_mode = A_ROWMAJOR;          // NHWC 1x1 convolution is a plain GEMM over pixels
    } else {
        p.a_mode = A_CONV_NHWC;
    }
    p.H = H; p.W = W; p.C = c.cin; p.OH = OH; p.OW = OW;
    p.KH = c.kh; p.KW = c.kw; p.stride = c.stride; p.pad = c.pad;
    p.bias = c.b;
    p.relu = relu ? 1 : 0;
    p.res = residual; p.ldr = c.cout;
    return run_gemm(r, p, nullptr);
}

// The attention tiles of one ragged decode chunk (cotr_decode_ragged): a device table of n_tc tensor-core tiles
// (kAttnTcTileRows rows of a pair with >= kAttnTcMinRows rows in the chunk) followed by n_simt SIMT tiles
// (kAttnSimtTileRows rows: the other pairs, or every pair on the fp32 SIMT path), see AttnParams::tiles.
struct ChunkTiles {
    const int4* tab = nullptr;
    int n_tc = 0, n_simt = 0;
    int rows_tc = 0, rows_simt = 0;
};

// Recorded as M = query rows, N = 512 keys, K = 32 x 8 heads.  Without tiles: one launch over nq rows of each of npairs
// pairs.  With the tiles of a ragged chunk: one launch per kind of tile present; the two launches write disjoint rows
// of the output.
int run_attention(const Run& r, AttnParams a, const ChunkTiles* t = nullptr) {
    if (!t) {
        LaunchScope scope(r, r.m->gemm_path == 0 ? K_ATTN_TC : K_ATTN_SIMT, a.nq * a.npairs, kTokens, kDModel);
        if (r.m->gemm_path != 0) return launch_attention_simt(a, r.s);
        return launch_attention_tc(a, r.s);
    }
    if (t->n_tc > 0) {
        a.tiles = t->tab; a.n_tiles = t->n_tc;
        LaunchScope scope(r, K_ATTN_TC, t->rows_tc, kTokens, kDModel);
        if (launch_attention_tc(a, r.s)) return 1;
    }
    if (t->n_simt > 0) {
        a.tiles = t->tab + t->n_tc; a.n_tiles = t->n_simt;
        LaunchScope scope(r, K_ATTN_SIMT, t->rows_simt, kTokens, kDModel);
        if (launch_attention_simt(a, r.s)) return 1;
    }
    return 0;
}

// Where the head-averaged attention maps of the selected layers go (cotr_encode_context_attention /
// cotr_decode_attention): bit l of `mask` selects layer l, selected layers are stored one after the other in ascending
// order, `base` is the first row of this call in the first selected layer's map.  mask = 0: no maps, no launches.
struct AttnMaps {
    unsigned mask = 0;
    float* base = nullptr;
    size_t layer_stride = 0;     // elements between the maps of consecutive selected layers
    size_t pair_stride = 0;      // elements between the first rows of consecutive pairs
    float* layer(int l) const {
        if (!((mask >> l) & 1u)) return nullptr;
        return base + (size_t)__builtin_popcount(mask & ((1u << l) - 1u)) * layer_stride;
    }
    AttnMaps at(size_t elems) const { AttnMaps a = *this; if (a.base) a.base += elems; return a; }
};

// The maps of a call over B pairs with `rows` query rows each, into the caller's (n_sel, B, rows, 512) buffer
AttnMaps attn_maps(int layer_mask, float* attn_dev, int B, size_t rows) {
    AttnMaps maps;
    maps.mask = (unsigned)layer_mask;
    maps.base = attn_dev;
    maps.layer_stride = (size_t)B * rows * kTokens;
    maps.pair_stride = rows * kTokens;
    return maps;
}

// The maps launch over the operands the attention launch `a` reads, local pair p's rows from out + p * out_pair_stride
AttnWeightsParams attention_weights_params(const AttnParams& a, float* out, size_t out_pair_stride) {
    AttnWeightsParams p{};
    p.q = a.q; p.ldq = a.ldq;
    p.k = a.k; p.ldk = a.ldk;
    p.kv_img = a.kv_img; p.img_pair_stride = a.img_pair_stride;
    p.out = out; p.out_pair_stride = out_pair_stride;
    p.nq = a.nq; p.npairs = a.npairs; p.pair0 = a.pair0;
    return p;
}

// The maps of one layer from the operands its attention launch `a` just read (attention_weights.cu); recorded like the
// attention launch (M = query rows, N = 512 keys, K = 32 x 8 heads).
int run_attention_weights(const Run& r, const AttnParams& a, const AttnMaps& maps, int layer) {
    float* out = maps.layer(layer);
    if (!out) return 0;
    const AttnWeightsParams p = attention_weights_params(a, out, maps.pair_stride);
    const bool tc = r.m->gemm_path == 0;
    LaunchScope scope(r, tc ? K_ATTN_WEIGHTS_TC : K_ATTN_WEIGHTS_SIMT, a.nq * a.npairs, kTokens, kDModel);
    return tc ? launch_attention_weights_tc(p, r.s) : launch_attention_weights_simt(p, r.s);
}

// ----------------------------------------------------------------------------------------------
// workspace
// ----------------------------------------------------------------------------------------------
constexpr size_t kStemElems = 128 * 128 * 64;      // per image
constexpr size_t kBigElems = 64 * 64 * 256;        // largest block input / output per image
constexpr size_t kT1Elems = 64 * 64 * 128;         // largest conv1 output per image (layer2.0)
constexpr size_t kT2Elems = 64 * 64 * 64;          // largest conv2 output per image (layer1)

// split16 buffer of `elems` elements: one allocation, hi plane first (elems is always a multiple of 8)
int ws_alloc(Split16* t, size_t elems) {
    __half* base = nullptr;
    COTR_CHECK_CUDA(cudaMalloc((void**)&base, elems * 2 * sizeof(__half)));
    t->hi = base;
    t->lo = base + elems;
    return 0;
}
void ws_free(Split16* t) { if (t->hi) { cudaFree(t->hi); } t->hi = nullptr; t->lo = nullptr; }
int ws_alloc_f32(float** p, size_t elems) {
    COTR_CHECK_CUDA(cudaMalloc((void**)p, elems * sizeof(float)));
    return 0;
}
void ws_free_f32(float** p) { if (*p) { cudaFree(*p); *p = nullptr; } }

// One workspace buffer: a split16 tensor (allocated as ws_alloc does) or a plain device array, and its size.
struct WsBuf {
    Split16* split;
    void** raw;
    size_t bytes;
};
WsBuf ws_split(Split16* t, size_t elems) { return {t, nullptr, elems * 2 * sizeof(__half)}; }
template <class T>
WsBuf ws_raw(T** p, size_t elems) { return {nullptr, reinterpret_cast<void**>(p), elems * sizeof(T)}; }

// Every buffer of a section's workspace with its size, listed once: allocation, release and cotr_workspace_bytes all
// walk these lists.  Encoder: the backbone of 2B images and the transformer of B pairs.
std::vector<WsBuf> encode_ws_bufs(Workspace& w, int B) {
    const size_t img = 2 * (size_t)B, tok = (size_t)B * kTokens;
    return {ws_split(&w.canvas, img * kStemCanvasElems), ws_split(&w.stem, img * kStemElems),
            ws_split(&w.bx, img * kBigElems), ws_split(&w.by, img * kBigElems), ws_split(&w.bds, img * kBigElems),
            ws_split(&w.bt1, img * kT1Elems), ws_split(&w.bt2, img * kT2Elems),
            ws_split(&w.src, tok * kDModel), ws_split(&w.xa, tok * kDModel), ws_split(&w.xb, tok * kDModel),
            ws_split(&w.qk, tok * 2 * kDModel), ws_split(&w.vt, (size_t)B * kVtLayer), ws_split(&w.ao, tok * kDModel),
            ws_split(&w.ffh, tok * kFF), ws_raw(&w.ln_tmp, tok * kDModel),
            ws_raw(&w.enc_st_a, tok * 16), ws_raw(&w.enc_st_b, tok * 16),
            ws_raw(&w.kvimg, (size_t)B * kHeads * kAttnHeadImgBytes), ws_raw(&w.pair_id, img)};
}
// Decoder: `rows` query rows, rounded up to a multiple of 8 (ws_alloc's condition).
std::vector<WsBuf> decode_ws_bufs(Workspace& w, int rows) {
    const size_t R = ((size_t)rows + 7) & ~(size_t)7;
    return {ws_split(&w.qpos, R * kDModel), ws_split(&w.qp, R * kQpCols), ws_split(&w.t, R * kDModel),
            ws_split(&w.qb, R * kDModel), ws_split(&w.dao, R * kDModel), ws_split(&w.dh, R * kFF),
            ws_split(&w.hs, R * kDModel), ws_split(&w.hd1, R * kDModel), ws_split(&w.hd2, R * kDModel),
            ws_split(&w.t2, R * kDModel), ws_raw(&w.dln_tmp, R * kDModel),
            ws_raw(&w.dec_st_a, R * 16), ws_raw(&w.dec_st_b, R * 16)};
}

// Keypoint matching: the canvas queries and predictions of `rows` packed rows.
std::vector<WsBuf> match_ws_bufs(Workspace& w, int64_t rows) {
    return {ws_raw(&w.match_q, (size_t)rows * 2), ws_raw(&w.match_pred, (size_t)rows * 2)};
}

// Zoom-in walks: the per-chunk counters are 2 per u64, after the status word.
std::vector<WsBuf> refine_ws_bufs(Workspace& w, const RefineCaps& c) {
    return {ws_raw(&w.refine_canvas, (size_t)c.squads * 3 * COTR_CANVAS_H * COTR_CANVAS_W), ws_raw(&w.refine_sides, (size_t)c.squads * 2),
            ws_raw(&w.refine_tmp, c.tmp), ws_raw(&w.refine_q, (size_t)c.rows * 2), ws_raw(&w.refine_pred, (size_t)c.rows * 2),
            ws_raw(&w.refine_counts, 1 + ((size_t)c.chunks + 1) / 2), ws_raw(&w.refine_iota, (size_t)c.ids),
            ws_raw(&w.refine_zeros, (size_t)c.ids), ws_raw(&w.grouped_pts, (size_t)c.ids * 4), ws_raw(&w.grouped_box, (size_t)c.ids * 8),
            ws_raw(&w.grouped_tab, 1 + (size_t)c.ids * 3)};
}

void ws_release(const std::vector<WsBuf>& bufs) {
    for (const WsBuf& b : bufs) {
        if (b.split) ws_free(b.split);
        else if (*b.raw) { cudaFree(*b.raw); *b.raw = nullptr; }
    }
}
int ws_allocate(const std::vector<WsBuf>& bufs) {
    for (const WsBuf& b : bufs) {
        void* base = nullptr;
        COTR_CHECK_CUDA(cudaMalloc(&base, b.bytes));
        if (b.split) {
            b.split->hi = static_cast<__half*>(base);
            b.split->lo = b.split->hi + b.bytes / (2 * sizeof(__half));
        } else {
            *b.raw = base;
        }
    }
    return 0;
}
size_t ws_bytes(const std::vector<WsBuf>& bufs) {
    size_t n = 0;
    for (const WsBuf& b : bufs) n += b.bytes;
    return n;
}

// Temporaries of one call (model construction, test hooks), freed on every return (cudaFree waits for the work queued
// on them).
struct DevAllocs {
    std::vector<void*> ptrs;
    ~DevAllocs() { for (void* p : ptrs) cudaFree(p); }
    int alloc(void** out, size_t bytes) {
        COTR_CHECK_CUDA(cudaMalloc(out, bytes));
        ptrs.push_back(*out);
        return 0;
    }
    int upload(void** out, const void* host, size_t bytes) {
        if (alloc(out, bytes)) return 1;
        COTR_CHECK_CUDA(cudaMemcpy(*out, host, bytes, cudaMemcpyHostToDevice));
        return 0;
    }
};

struct TmpSplit {
    Split16 t = kNoSplit;
    ~TmpSplit() { ws_free(&t); }
    int from_f32(const float* src, size_t n) {
        const size_t padded = (n + 7) & ~(size_t)7;
        if (ws_alloc(&t, padded)) return 1;
        return launch_f32_to_split16(src, t, n, 0);
    }
    int empty(size_t n) { return ws_alloc(&t, (n + 7) & ~(size_t)7); }
};

// Schedule selection.
// Deferred LayerNorm (no LayerNorm launches; consumers normalise on the fly) removes 12 launches from the encoder and
// 12 from each decoder chunk but makes its consumer GEMMs a little longer: it pays off only once a section has
// thousands of rows (the launches saved then outweigh the longer epilogues), so each section picks it by its row count.
// cotr_debug_set_variant overrides: bit 19 = always deferred, bit 16 = never.
constexpr int kDeferredLnMinRows = 2048;
inline bool deferred_ln_enabled(const cotr_model* m, int rows) {
    if (m->gemm_path != 0 || (g_tc_variant & (1 << 16))) return false;
    return (g_tc_variant & (1 << 19)) != 0 || rows >= kDeferredLnMinRows;
}
// In the explicit-LayerNorm schedule on the tensor-core path each feed-forward block (linear1, linear2, norm) is one
// fused launch (run_mlp); bit 16 keeps the separate launches.
inline bool fused_mlp_enabled(const cotr_model* m) {
    return m->gemm_path == 0 && !(g_tc_variant & (1 << 16));
}

// Captured graphs embed workspace / staging / context addresses: whenever one of those is reallocated every graph is
// stale.  The shapes stay "seen", so the next call of each shape re-captures against the new buffers.
void drop_graphs(cotr_model* m) {
    for (auto& kv : m->graphs) cudaGraphExecDestroy(kv.second);
    m->graphs.clear();
    m->graph_launches.clear();
}

// Cross-stream ordering of the entry points (see cotr_model::order_event).  Same-stream calls need no wait.
struct CallOrder {
    cotr_model* m;
    cudaStream_t s;
    CallOrder(cotr_model* m_, cudaStream_t s_) : m(m_), s(s_) {
        if (m->order_valid && m->order_stream != s && m->order_event) cudaStreamWaitEvent(s, m->order_event, 0);
    }
    ~CallOrder() {
        if (!m->order_event && cudaEventCreateWithFlags(&m->order_event, cudaEventDisableTiming) != cudaSuccess) {
            m->order_event = nullptr;
            return;
        }
        if (cudaEventRecord(m->order_event, s) == cudaSuccess) { m->order_stream = s; m->order_valid = true; }
    }
};

int ensure_encode_ws(cotr_model* m, int B) {
    Workspace& w = m->ws;
    if (B <= w.cap_pairs) return 0;
    COTR_CHECK_CUDA(cudaDeviceSynchronize());
    drop_graphs(m);
    w.cap_pairs = 0;      // a failed allocation below leaves no capacity behind, so the next call allocates again
    ws_release(encode_ws_bufs(w, 0));
    if (ws_allocate(encode_ws_bufs(w, B))) return 1;
    std::vector<int> ident(2 * (size_t)B);
    for (size_t i = 0; i < ident.size(); ++i) ident[i] = (int)i;
    COTR_CHECK_CUDA(cudaMemcpy(w.pair_id, ident.data(), ident.size() * sizeof(int), cudaMemcpyHostToDevice));
    // the 16 pad bytes of every value key group are copied by the bulk TMA: keep them defined
    COTR_CHECK_CUDA(cudaMemset(w.kvimg, 0, (size_t)B * kHeads * kAttnHeadImgBytes));
    // the border of the stem canvas is the convolution's zero padding: written here, never again
    COTR_CHECK_CUDA(cudaMemset(w.canvas.hi, 0, 2 * (size_t)B * kStemCanvasElems * 2 * sizeof(__half)));
    w.cap_pairs = B;
    return 0;
}

int ensure_decode_ws(cotr_model* m, int rows) {
    Workspace& w = m->ws;
    if (rows <= w.cap_rows) return 0;
    COTR_CHECK_CUDA(cudaDeviceSynchronize());
    drop_graphs(m);
    w.cap_rows = 0;       // as in ensure_encode_ws: no stale capacity after a failed allocation
    ws_release(decode_ws_bufs(w, 0));
    if (ws_allocate(decode_ws_bufs(w, rows))) return 1;
    w.cap_rows = rows;
    return 0;
}

// Never captured in a graph, so growing it drops none.
int ensure_match_ws(cotr_model* m, int64_t rows) {
    Workspace& w = m->ws;
    if (rows <= w.cap_match_rows) return 0;
    COTR_CHECK_CUDA(cudaDeviceSynchronize());
    w.cap_match_rows = 0;     // as in ensure_encode_ws: no stale capacity after a failed allocation
    ws_release(match_ws_bufs(w, 0));
    if (ws_allocate(match_ws_bufs(w, rows))) return 1;
    w.cap_match_rows = rows;
    return 0;
}

// Never captured in a graph either; every capacity only grows.
int ensure_refine_ws(cotr_model* m, RefineCaps need) {
    Workspace& w = m->ws;
    RefineCaps& cap = w.cap_refine;
    if (need.squads <= cap.squads && need.rows <= cap.rows && need.ids <= cap.ids && need.chunks <= cap.chunks && need.tmp <= cap.tmp)
        return 0;
    need.squads = std::max(need.squads, cap.squads);
    need.rows = std::max(need.rows, cap.rows);
    need.ids = std::max(need.ids, cap.ids);
    need.chunks = std::max(need.chunks, cap.chunks);
    need.tmp = std::max(need.tmp, cap.tmp);
    COTR_CHECK_CUDA(cudaDeviceSynchronize());
    cap = RefineCaps();       // as in ensure_encode_ws
    ws_release(refine_ws_bufs(w, cap));
    if (ws_allocate(refine_ws_bufs(w, need))) return 1;
    std::vector<int32_t> iota((size_t)need.ids);
    for (size_t i = 0; i < iota.size(); ++i) iota[i] = (int32_t)i;
    COTR_CHECK_CUDA(cudaMemcpy(w.refine_iota, iota.data(), iota.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
    COTR_CHECK_CUDA(cudaMemset(w.refine_zeros, 0, iota.size() * sizeof(int32_t)));
    COTR_CHECK_CUDA(cudaDeviceSynchronize());     // both tables written before a call on a non-blocking stream reads them
    cap = need;
    return 0;
}

// ----------------------------------------------------------------------------------------------
// forward schedule
// ----------------------------------------------------------------------------------------------
// The backbone of n_img 256x256 images (halves: the two halves of n_img/2 canvases, else a (n_img,3,256,256) batch) up to
// layer3; the last bottleneck writes the (n_img,16,16,1024) NHWC features to `feat`.  The workspace must hold n_img images.
int encode_backbone(cotr_model* m, const float* img, bool halves, int n_img, Split16 feat, cudaStream_t s) {
    Workspace& w = m->ws;
    Run r{m, s};
    const CSplit16 none{nullptr, nullptr};

    // backbone.py:81-82: the two 256x256 halves go through the ResNet body as independent images.
    // Stem: conv 7x7/2 (+FrozenBN folded) + ReLU, then MaxPool 3x3/2  (torchvision resnet.py _forward_impl).
    {
        LaunchScope scope(r, K_STEM_CANVAS, n_img * 256 * 256, 4, 0);
        if (launch_stem_canvas(img, halves, w.canvas, n_img, s)) return 1;
    }
    if (run_conv(r, m->stem, n_img, cs(w.canvas), 256, 256, w.stem, true, none)) return 1;
    {
        LaunchScope scope(r, K_MAXPOOL, n_img * 64 * 64, 64, 0);
        if (launch_maxpool_3x3s2_nhwc(cs(w.stem), w.bx, n_img, 128, 128, 64, s)) return 1;
    }

    Split16 x = w.bx;
    Split16 y = w.by;
    int H = 64, W = 64;
    for (size_t i = 0; i < m->blocks.size(); ++i) {
        const Block& b = m->blocks[i];
        // torchvision Bottleneck (v1.5): 1x1 -> 3x3(stride) -> 1x1, + identity | downsample, ReLU
        if (run_conv(r, b.c1, n_img, cs(x), H, W, w.bt1, true, none)) return 1;
        if (run_conv(r, b.c2, n_img, cs(w.bt1), H, W, w.bt2, true, none)) return 1;
        const int OH = H / b.c2.stride, OW = W / b.c2.stride;
        CSplit16 identity = cs(x);
        if (b.has_ds) {
            if (run_conv(r, b.ds, n_img, cs(x), H, W, w.bds, false, none)) return 1;
            identity = cs(w.bds);
        }
        if (i + 1 == m->blocks.size()) y = feat;
        if (run_conv(r, b.c3, n_img, cs(w.bt2), OH, OW, y, true, identity)) return 1;
        Split16 t = x; x = y; y = t;
        H = OH; W = OW;
    }
    return 0;
}

// Everything of the context after the backbone, for B pairs: pair p is the canvas [image pairs[2p] | image pairs[2p+1]]
// of the (n,16,16,1024) NHWC features `feat` (pairs: [B][2] device table, see GemmParams::a_pairs).
int encode_tail(cotr_model* m, CSplit16 feat, const int* pairs, int B, cotr_context* ctx, cudaStream_t s, const AttnMaps& maps) {
    Workspace& w = m->ws;
    Run r{m, s};

    // cotr_model.py:37 input_proj (1x1 conv 1024 -> 256) fused with the left|right concat (backbone.py:85)
    // and the flatten to token-major (transformer.py:50): row = pair*512 + i*32 + j.
    const int T = B * kTokens;
    {
        GemmParams p = gemm_base(T, kDModel, 1024, feat, 1024, m->proj.w, m->proj.wtc, m->proj.wtc_scale, w.src, kDModel);
        p.a_mode = A_TOKENS;
        p.a_pairs = pairs;
        p.bias = m->proj.b;
        if (run_gemm(r, p, nullptr)) return 1;
    }

    // transformer.py:143-159 x6 (post-LN).  q = k = x + pos is folded into the constant add_qkv matrix.
    // q | k land row-major in qk [T][512]; v lands transposed in vt [pair][256][512] (what P V needs as its B operand).
    // On the tensor-core path keys and values go straight into the attention operand images instead.
    //
    // Deferred LayerNorm (tensor-core path, see deferred_ln_enabled): no LayerNorm kernel and no LayerNorm epilogue.  A
    // LayerNorm output is never stored; its producer writes the pre-norm rows (xa: x + attention, xb: x1 + FFN) and every
    // consumer applies the norm on the fly (GemmParams::a_ln_cs for GEMM inputs, res_ln_part for residual operands) from
    // the partial row statistics the producer's epilogue leaves behind: enc_st_a belongs to xa (norm1), enc_st_b to xb
    // (norm2).  Otherwise (and on the fp32 SIMT cross-check path): explicit LayerNorm launches, the checkpoint's weights
    // as they are.
    const bool dln = deferred_ln_enabled(m, T);
    const bool tc = m->gemm_path == 0;
    const bool fused_mlp = fused_mlp_enabled(m);
    Split16 xin = w.src;      // layer input
    for (int l = 0; l < kEncLayers; ++l) {
        const EncLayer& e = m->enc[l];
        const bool ln_in = dln && l > 0;          // the layer input is LN2_{l-1}(xb), deferred
        {
            GemmParams p = gemm_linear(e.qkv, dln, T, cs(xin), kDModel, w.qk, 2 * kDModel);
            p.addmat = dln ? e.add_qkv_tc : e.add_qkv; p.add_period = kTokens; p.ld_add = 3 * kDModel;
            redirect_kv(p, 1, 1, kDModel, w.vt, tc ? w.kvimg : nullptr);
            if (ln_in) { p.a_ln_cs = e.qkv.cs; p.a_ln_part = w.enc_st_b; }
            if (run_gemm(r, p, nullptr)) return 1;
        }
        AttnParams a{};
        a.q = cs(w.qk); a.ldq = 2 * kDModel;
        a.k = offset(cs(w.qk), kDModel); a.ldk = 2 * kDModel;
        a.vt = cs(w.vt); a.vt_pair_stride = kVtLayer;
        if (tc) { a.kv_img = w.kvimg; a.img_pair_stride = kHeads * kAttnHeadImgBytes; }
        a.out = w.ao; a.ldo = kDModel;
        a.nq = kTokens; a.npairs = B; a.pair0 = 0;
        if (run_attention(r, a)) return 1;
        if (run_attention_weights(r, a, maps, l)) return 1;         // before the next layer overwrites qk / kvimg
        if (dln) {
            // xa = x + out_proj(attn)                                   (transformer.py:149-154, norm1 deferred)
            if (run_linear_dln(r, e.o, T, cs(w.ao), kDModel, w.xa, kDModel, false, nullptr, w.enc_st_a, cs(xin), kDModel,
                               ln_in ? w.enc_st_b : nullptr, ln_in ? m->enc[l - 1].ln2_g : nullptr, ln_in ? m->enc[l - 1].ln2_b : nullptr)) return 1;
            // h = relu(W1 norm1(xa) + b1)                               (transformer.py:155)
            if (run_linear_dln(r, e.l1, T, cs(w.xa), kDModel, w.ffh, kFF, true, w.enc_st_a, nullptr)) return 1;
            // xb = norm1(xa) + W2 h + b2                                (transformer.py:155-157, norm2 deferred)
            if (run_linear_dln(r, e.l2, T, cs(w.ffh), kFF, w.xb, kDModel, false, nullptr, w.enc_st_b, cs(w.xa), kDModel,
                               w.enc_st_a, e.ln1_g, e.ln1_b)) return 1;
        } else {
            // x1 = LN1(x + out_proj(attn))
            if (run_linear(r, e.o, T, cs(w.ao), kDModel, w.xa, kDModel, false, cs(xin), kDModel, e.ln1_g, e.ln1_b, w.ln_tmp)) return 1;
            // x2 = LN2(x1 + W2 relu(W1 x1 + b1) + b2)
            if (fused_mlp) {
                if (run_mlp(r, e.l1, e.l2, T, cs(w.xa), w.xb, e.ln2_g, e.ln2_b)) return 1;
            } else {
                if (run_linear(r, e.l1, T, cs(w.xa), kDModel, w.ffh, kFF, true)) return 1;
                if (run_linear(r, e.l2, T, cs(w.ffh), kFF, w.xb, kDModel, false, cs(w.xa), kDModel, e.ln2_g, e.ln2_b, w.ln_tmp)) return 1;
            }
        }
        xin = w.xb;
    }
    m->last_mem = xin;
    m->last_mem_pre_ln = dln;

    // transformer.py:192-195: K_l = (mem + pos) Wk_l^T + bk_l, V_l = mem Wv_l^T + bv_l for all 6 decoder layers in ONE
    // GEMM (N = 3072): K blocks go row-major into ctx->k [T][1536], V blocks transposed into ctx->vt [pair][6][256][512]
    // (or both into the context's operand images).  Deferred: mem is norm2(xb) of the last encoder layer, applied here.
    {
        GemmParams p = gemm_linear(m->kv_all, dln, T, cs(xin), kDModel, ctx->k, kKCols);
        p.addmat = dln ? m->add_kv_tc : m->add_kv; p.add_period = kTokens; p.ld_add = 2 * kKCols;
        redirect_kv(p, 0, kDecLayers, 0, ctx->vt, tc ? ctx->img : nullptr);
        if (dln) { p.a_ln_cs = m->kv_all.cs; p.a_ln_part = w.enc_st_b; }
        if (run_gemm(r, p, nullptr)) return 1;
    }
    ctx->pairs = B;
    ctx->holds_img = tc;
    m->last_pairs = B;
    return 0;
}

int check_context(cotr_model* m, const char* fn, int B, const cotr_context* ctx) {
    COTR_CHECK(B >= 1, "%s: B must be >= 1 (got %d)", fn, B);
    COTR_CHECK(ctx && ctx->model == m, "%s: context does not belong to this model", fn);
    COTR_CHECK(B <= ctx->max_pairs, "%s: B = %d exceeds the context capacity %d", fn, B, ctx->max_pairs);
    return 0;
}

// A decode's context: this model's, holding exactly B pairs, encoded under the current matrix-multiply path.
int check_decode_context(cotr_model* m, const char* fn, int B, const cotr_context* ctx) {
    COTR_CHECK(ctx && ctx->model == m, "%s: context does not belong to this model", fn);
    COTR_CHECK(B >= 1 && B == ctx->pairs, "%s: B = %d but the context holds %d pairs", fn, B, ctx->pairs);
    COTR_CHECK(ctx->holds_img == (m->gemm_path == 0), "%s: the context was encoded under the other matrix-multiply path "
               "(cotr_set_gemm_path): re-encode it", fn);
    return 0;
}

int encode_impl(cotr_model* m, const float* img, int B, cotr_context* ctx, cudaStream_t s, const AttnMaps& maps = AttnMaps()) {
    if (check_context(m, "cotr_encode_context", B, ctx)) return 1;
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    if (ensure_encode_ws(m, B)) return 1;
    Workspace& w = m->ws;
    if (encode_backbone(m, img, true, 2 * B, w.bx, s)) return 1;
    m->last_feat = w.bx;   // (2B,16,16,1024) NHWC
    return encode_tail(m, cs(w.bx), w.pair_id, B, ctx, s, maps);
}

// Images per backbone pass of cotr_encode_images: the backbone workspace of a 32-pair context.
constexpr int kImageChunk = 64;
constexpr size_t kFeatElems = 16 * 16 * 1024;     // per image and plane (COTR_IMAGE_FEATURE_BYTES / 4)

int encode_images_impl(cotr_model* m, const float* img, int N, void* feat_dev, cudaStream_t s) {
    if (ensure_encode_ws(m, (std::min(N, kImageChunk) + 1) / 2)) return 1;
    __half* hi = static_cast<__half*>(feat_dev);
    __half* lo = hi + (size_t)N * kFeatElems;
    for (int n0 = 0; n0 < N; n0 += kImageChunk) {
        const int n = std::min(kImageChunk, N - n0);
        const Split16 dst{hi + (size_t)n0 * kFeatElems, lo + (size_t)n0 * kFeatElems};
        if (encode_backbone(m, img + (size_t)n0 * 3 * 256 * 256, false, n, dst, s)) return 1;
    }
    return 0;
}

int encode_pairs_impl(cotr_model* m, const void* feat_dev, int n_images, const int32_t* pairs, int B, cotr_context* ctx,
                      cudaStream_t s, const AttnMaps& maps) {
    if (ensure_encode_ws(m, B)) return 1;
    if (m->pair_tab.upload(pairs, 2 * (size_t)B, s)) return 1;
    const __half* hi = static_cast<const __half*>(feat_dev);
    return encode_tail(m, CSplit16{hi, hi + (size_t)n_images * kFeatElems}, m->pair_tab.dev, B, ctx, s, maps);
}

// R query rows (queries / pred: (R,2)).  tiles == nullptr: pair pair0 + p owns rows p * nq .. p * nq + nq - 1, p < npairs;
// otherwise the attention follows the chunk's tile table (a ragged chunk, no maps) and pair0 / npairs / nq are unused.
// maps.base: this chunk's first row (pair pair0, its first query) in the caller's (n_sel, B, Q, 512) buffer
int decode_chunk(cotr_model* m, const cotr_context* ctx, const float* queries, float* pred, int R, const ChunkTiles* tiles,
                 int pair0, int npairs, int nq, cudaStream_t s, const AttnMaps& maps) {
    Workspace& w = m->ws;
    Run r{m, s};
    const CSplit16 none{nullptr, nullptr};
    // cotr_model.py:34-35 query_proj (lin_sine, depth 64)
    {
        LaunchScope scope(r, K_QENC, R, kDModel, 0);
        if (launch_query_encode(queries, w.qpos, R, s)) return 1;
    }
    // q-side of transformer.py:192: ((t + qpos) Wq^T + bq) s  =  t (s Wq)^T + [qpos (s Wq)^T + s bq]; the bracket for
    // all 6 layers is one GEMM.
    if (run_linear(r, m->qpos_all, R, cs(w.qpos), kDModel, w.qp, kQpCols, false)) return 1;

    // Deferred LayerNorm (see encode_tail): w.t = t + attention (norm2 deferred), w.t2 = t1 + FFN (norm3 deferred);
    // dec_st_a = partial row statistics of w.t (norm2), dec_st_b of w.t2 (norm3).  Explicit: every layer ends in w.t.
    const bool dln = deferred_ln_enabled(m, R);
    const bool fused_mlp = fused_mlp_enabled(m);
    const Split16 tin = dln ? w.t2 : w.t;      // the layer input t of layers > 0 (deferred: before norm3_{l-1})
    for (int l = 0; l < kDecLayers; ++l) {
        const DecLayer& d = m->dec[l];
        const bool ln_in = dln && l > 0;
        CSplit16 q = cs(w.qp);      // layer 0: tgt = 0 (transformer.py:54), so q is the qpos projection alone
        int ldq = kQpCols;
        if (l > 0) {
            const CSplit16 qpos_l = offset(cs(w.qp), (size_t)l * kDModel);
            if (dln ? run_linear_dln(r, d.q, R, cs(tin), kDModel, w.qb, kDModel, false, w.dec_st_b, nullptr, qpos_l, kQpCols)
                    : run_linear(r, d.q, R, cs(tin), kDModel, w.qb, kDModel, false, qpos_l, kQpCols)) return 1;
            q = cs(w.qb); ldq = kDModel;
        }
        AttnParams a{};
        a.q = q; a.ldq = ldq;
        a.k = offset(cs(ctx->k), (size_t)l * kDModel); a.ldk = kKCols;
        a.vt = offset(cs(ctx->vt), (size_t)l * kVtLayer); a.vt_pair_stride = kDecLayers * kVtLayer;
        if (ctx->holds_img) { a.kv_img = ctx->img + (size_t)l * kHeads * kAttnHeadImgBytes; a.img_pair_stride = (size_t)kDecLayers * kHeads * kAttnHeadImgBytes; }
        a.out = w.dao; a.ldo = kDModel;
        a.nq = nq; a.npairs = npairs; a.pair0 = pair0;
        if (run_attention(r, a, tiles)) return 1;
        if (run_attention_weights(r, a, maps, l)) return 1;
        const CSplit16 res = l > 0 ? cs(tin) : none;
        if (dln) {
            // transformer.py:196-197: t = t + out_proj(attn)   (norm2 deferred; t = norm3_{l-1}(t2), deferred, or 0)
            if (run_linear_dln(r, d.o, R, cs(w.dao), kDModel, w.t, kDModel, false, nullptr, w.dec_st_a, res, kDModel,
                               ln_in ? w.dec_st_b : nullptr, ln_in ? m->dec[l - 1].ln3_g : nullptr, ln_in ? m->dec[l - 1].ln3_b : nullptr)) return 1;
            // transformer.py:198-200: t2 = norm2(t) + linear2(relu(linear1(norm2(t))))   (norm3 deferred)
            if (run_linear_dln(r, d.l1, R, cs(w.t), kDModel, w.dh, kFF, true, w.dec_st_a, nullptr)) return 1;
            if (run_linear_dln(r, d.l2, R, cs(w.dh), kFF, w.t2, kDModel, false, nullptr, w.dec_st_b, cs(w.t), kDModel,
                               w.dec_st_a, d.ln2_g, d.ln2_b)) return 1;
        } else {
            // transformer.py:196-197: t = norm2(t + out_proj(attn))
            if (run_linear(r, d.o, R, cs(w.dao), kDModel, w.t, kDModel, false, res, kDModel, d.ln2_g, d.ln2_b, w.dln_tmp)) return 1;
            // transformer.py:198-200: t = norm3(t + linear2(relu(linear1(t))))
            if (fused_mlp) {
                // in place; the last layer also applies transformer.py:110-111 decoder.norm and writes hs
                const bool last = l == kDecLayers - 1;
                if (run_mlp(r, d.l1, d.l2, R, cs(w.t), last ? w.hs : w.t, d.ln3_g, d.ln3_b,
                            last ? m->dec_norm_g : nullptr, last ? m->dec_norm_b : nullptr)) return 1;
            } else {
                if (run_linear(r, d.l1, R, cs(w.t), kDModel, w.dh, kFF, true)) return 1;
                if (run_linear(r, d.l2, R, cs(w.dh), kFF, w.t, kDModel, false, cs(w.t), kDModel, d.ln3_g, d.ln3_b, w.dln_tmp)) return 1;
            }
        }
    }
    // transformer.py:110-111 decoder.norm on the last level; cotr_model.py:38-39 corr_embed on that level only.
    if (dln) {
        // norm3 of the last layer, then decoder.norm, in one pass over the rows
        const DecLayer& d = m->dec[kDecLayers - 1];
        LaunchScope scope(r, K_LAYERNORM, R, kDModel, 0);
        if (launch_layernorm_twice(cs(w.t2), d.ln3_g, d.ln3_b, m->dec_norm_g, m->dec_norm_b, w.hs, R, s)) return 1;
    } else if (!fused_mlp) {      // (fused: the last feed-forward launch wrote hs)
        LaunchScope scope(r, K_LAYERNORM, R, kDModel, 0);
        if (launch_layernorm(cs(w.t), m->dec_norm_g, m->dec_norm_b, w.hs, R, s)) return 1;
    }
    if (run_linear(r, m->head[0], R, cs(w.hs), kDModel, w.hd1, kDModel, true)) return 1;
    if (run_linear(r, m->head[1], R, cs(w.hd1), kDModel, w.hd2, kDModel, true)) return 1;
    {
        GemmParams p = gemm_base(R, 2, kDModel, cs(w.hd2), kDModel, m->head[2].w, m->head[2].wtc, m->head[2].wtc_scale, kNoSplit, 2);
        p.bias = m->head[2].b;
        p.out_f32 = pred;
        if (run_gemm(r, p, nullptr)) return 1;
    }
    return 0;
}

// maps (optional): base = attn_dev, layer_stride = B * Q * 512, pair_stride = Q * 512
int decode_impl(cotr_model* m, const cotr_context* ctx, const float* queries, int B, int Q, float* pred, cudaStream_t s,
                const AttnMaps& maps = AttnMaps()) {
    if (check_decode_context(m, "cotr_decode", B, ctx)) return 1;
    COTR_CHECK(Q >= 0, "cotr_decode: negative Q");
    if (Q == 0) return 0;
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    const long long total = (long long)B * Q;
    const int cap = (int)(total < kDecodeChunkRows ? total : kDecodeChunkRows);
    if (ensure_decode_ws(m, cap)) return 1;
    if (Q <= kDecodeChunkRows) {
        const int pairs_per = kDecodeChunkRows / Q;
        for (int b0 = 0; b0 < B; b0 += pairs_per) {
            const int nb = (B - b0 < pairs_per) ? B - b0 : pairs_per;
            if (decode_chunk(m, ctx, queries + (size_t)b0 * Q * 2, pred + (size_t)b0 * Q * 2, nb * Q, nullptr, b0, nb, Q, s,
                             maps.at((size_t)b0 * Q * kTokens))) return 1;
        }
    } else {
        for (int b = 0; b < B; ++b)
            for (int q0 = 0; q0 < Q; q0 += kDecodeChunkRows) {
                const int nq = (Q - q0 < kDecodeChunkRows) ? Q - q0 : kDecodeChunkRows;
                const size_t off = ((size_t)b * Q + q0) * 2;
                if (decode_chunk(m, ctx, queries + off, pred + off, nq, nullptr, b, 1, nq, s, maps.at(((size_t)b * Q + q0) * kTokens))) return 1;
            }
    }
    m->last_rows = (total <= kDecodeChunkRows) ? (int)total : 0;
    return 0;
}

// Ragged decode (cotr_decode_ragged): pair p owns the packed rows offsets[p] .. offsets[p+1] - 1.  Whole pairs are packed in
// order into chunks of at most kDecodeChunkRows rows; a pair with more rows than that gets chunks of its own, one per
// slice, as in decode_impl.  A chunk is a contiguous row range, so its queries and predictions are pointer offsets, and
// with the same count Q for every pair the chunks, and so the launches, are exactly those of decode_impl.  Every chunk's
// attention tile table is built on the host and reaches the device with one copy per call.  Arguments are checked by
// the caller.
int decode_ragged_impl(cotr_model* m, const cotr_context* ctx, const float* queries, const int64_t* offsets, int B,
                       float* pred, cudaStream_t s) {
    struct Chunk {
        int64_t row0 = 0;      // first packed row
        int rows = 0;
        size_t tab0 = 0;       // first entry of the chunk's tiles in the call's table
        ChunkTiles t;
    };
    struct Segment { int pair, row0, rows; };     // rows of one pair in a chunk, row0 relative to the chunk
    std::vector<Chunk> chunks;
    std::vector<int4> tab;
    std::vector<Segment> segs;
    const bool tc = m->gemm_path == 0;
    Chunk cur;
    auto close = [&]() {
        if (cur.rows == 0) return;
        cur.tab0 = tab.size();
        // tensor-core tiles first, then the SIMT tiles (see ChunkTiles)
        for (int pass = 0; pass < 2; ++pass) {
            const size_t first = tab.size();
            for (const Segment& g : segs) {
                const bool to_tc = tc && g.rows >= kAttnTcMinRows;
                if (to_tc != (pass == 0)) continue;
                const int step = to_tc ? kAttnTcTileRows : kAttnSimtTileRows;
                for (int i = 0; i < g.rows; i += step) tab.push_back(make_int4(g.pair, g.row0 + i, std::min(step, g.rows - i), 0));
                (to_tc ? cur.t.rows_tc : cur.t.rows_simt) += g.rows;
            }
            (pass == 0 ? cur.t.n_tc : cur.t.n_simt) = (int)(tab.size() - first);
        }
        chunks.push_back(cur);
        const int64_t next = cur.row0 + cur.rows;
        cur = Chunk();
        cur.row0 = next;
        segs.clear();
    };
    for (int p = 0; p < B; ++p) {
        const int64_t n = offsets[p + 1] - offsets[p];
        if (n == 0) continue;
        if (n > kDecodeChunkRows) {
            close();
            for (int64_t q0 = 0; q0 < n; q0 += kDecodeChunkRows) {
                const int rows = (int)std::min<int64_t>(kDecodeChunkRows, n - q0);
                segs.push_back({p, 0, rows});
                cur.rows = rows;
                close();
            }
            continue;
        }
        if (cur.rows + n > kDecodeChunkRows) close();
        segs.push_back({p, cur.rows, (int)n});
        cur.rows += (int)n;
    }
    close();

    int cap = 0;
    for (const Chunk& c : chunks) cap = std::max(cap, c.rows);
    if (ensure_decode_ws(m, cap)) return 1;
    if (m->tile_tab.upload(tab.data(), tab.size(), s)) return 1;
    for (Chunk& c : chunks) {
        c.t.tab = m->tile_tab.dev + c.tab0;
        const size_t off = (size_t)c.row0 * 2;
        if (decode_chunk(m, ctx, queries + off, pred + off, c.rows, &c.t, 0, 0, 0, s, AttnMaps())) return 1;
    }
    m->last_rows = chunks.size() == 1 ? chunks[0].rows : 0;
    return 0;
}

// The rows of a matching call (cotr_match_keypoints / cotr_mutual_nearest): context 2p = [a_p | b_p] owns the rows of
// a_p's keypoints, context 2p+1 = [b_p | a_p] those of b_p's, packed in context order; ctx_off[c] is context c's first
// row.  `tab` holds the n_tiles match tiles (3 int4 each, common.cuh MatchTile) followed by one (first row of context
// 2p, rows of 2p, rows of 2p+1, 0) entry per pair for mutual_kernel.  Every argument is checked here, on the host.
struct MatchPlan {
    std::vector<int4> tab;
    std::vector<int64_t> ctx_off;
    int n_tiles = 0;
    int64_t rows = 0;
};

int plan_match(const char* fn, const int64_t* kpt_off, int n_images, const int32_t* pairs, int B, const int32_t* sizes,
               MatchPlan* plan) {
    COTR_CHECK(n_images >= 1, "%s: n_images must be >= 1 (got %d)", fn, n_images);
    COTR_CHECK(B >= 1, "%s: B must be >= 1 (got %d)", fn, B);
    COTR_CHECK(kpt_off && pairs, "%s: null kpt_offsets_host or pairs_host", fn);
    COTR_CHECK(kpt_off[0] == 0, "%s: kpt_offsets_host[0] = %lld, must be 0", fn, (long long)kpt_off[0]);
    for (int i = 0; i < n_images; ++i)
        COTR_CHECK(kpt_off[i + 1] >= kpt_off[i], "%s: kpt_offsets_host decreases at image %d (%lld -> %lld)", fn, i,
                   (long long)kpt_off[i], (long long)kpt_off[i + 1]);
    COTR_CHECK(kpt_off[n_images] <= INT32_MAX, "%s: %lld keypoints in one call (at most %d)", fn, (long long)kpt_off[n_images], INT32_MAX);
    for (int i = 0; i < 2 * B; ++i)
        COTR_CHECK(pairs[i] >= 0 && pairs[i] < n_images, "%s: pairs[%d][%d] = %d is outside [0, %d)", fn, i / 2, i % 2,
                   (int)pairs[i], n_images);
    if (sizes)
        for (int i = 0; i < 2 * n_images; ++i)
            COTR_CHECK(sizes[i] >= 1 && sizes[i] <= 65536, "%s: sizes[%d][%d] = %d is outside [1, 65536]", fn, i / 2, i % 2,
                       (int)sizes[i]);
    int64_t R = 0;
    for (int p = 0; p < B; ++p) R += (kpt_off[pairs[2 * p] + 1] - kpt_off[pairs[2 * p]]) + (kpt_off[pairs[2 * p + 1] + 1] - kpt_off[pairs[2 * p + 1]]);
    COTR_CHECK(R <= INT32_MAX, "%s: %lld rows in one call (at most %d)", fn, (long long)R, INT32_MAX);

    plan->rows = R;
    plan->ctx_off.assign(2 * (size_t)B + 1, 0);
    plan->tab.clear();
    int64_t row = 0;
    for (int c = 0; c < 2 * B; ++c) {
        const int left = pairs[2 * (c / 2) + (c & 1)], right = pairs[2 * (c / 2) + 1 - (c & 1)];
        const int n_left = (int)(kpt_off[left + 1] - kpt_off[left]);
        plan->ctx_off[c] = row;
        for (int i = 0; i < n_left; i += kMatchTileRows) {
            MatchTile t{};
            t.row0 = (int)(row + i);
            t.rows = std::min(kMatchTileRows, n_left - i);
            t.left0 = (int)kpt_off[left] + i;
            t.right0 = (int)kpt_off[right];
            t.n_right = (int)(kpt_off[right + 1] - kpt_off[right]);
            if (sizes) {
                t.w_left = sizes[2 * left]; t.h_left = sizes[2 * left + 1];
                t.w_right = sizes[2 * right]; t.h_right = sizes[2 * right + 1];
            }
            int4 v[3];
            memcpy(v, &t, sizeof(t));
            plan->tab.insert(plan->tab.end(), v, v + 3);
        }
        row += n_left;
    }
    plan->ctx_off[2 * B] = row;
    plan->n_tiles = (int)(plan->tab.size() / 3);
    for (int p = 0; p < B; ++p)
        plan->tab.push_back(make_int4((int)plan->ctx_off[2 * p], (int)(plan->ctx_off[2 * p + 1] - plan->ctx_off[2 * p]),
                                      (int)(plan->ctx_off[2 * p + 2] - plan->ctx_off[2 * p + 1]), 0));
    return 0;
}

// Output buffers of a matching call with R rows (NULL allowed when R == 0).
int check_match_outputs(const char* fn, int64_t R, const double* kpts, const double* corr, const int32_t* nearest,
                        const int32_t* match, const int32_t* count) {
    COTR_CHECK(count != nullptr, "%s: null count_dev", fn);
    COTR_CHECK(((uintptr_t)count & 3) == 0, "%s: count_dev is not 4-byte aligned", fn);
    if (R == 0) return 0;
    COTR_CHECK(kpts && corr && nearest && match, "%s: null kpts_dev, corr_dev, nearest_dev or match_dev for %lld rows", fn, (long long)R);
    COTR_CHECK(((uintptr_t)kpts & 7) == 0 && ((uintptr_t)corr & 7) == 0, "%s: kpts_dev or corr_dev is not 8-byte aligned", fn);
    COTR_CHECK(((uintptr_t)nearest & 3) == 0 && ((uintptr_t)match & 3) == 0, "%s: nearest_dev or match_dev is not 4-byte aligned", fn);
    return 0;
}

// ----------------------------------------------------------------------------------------------
// model construction
// ----------------------------------------------------------------------------------------------
int build_model(cotr_model* m, const TensorMap& tm) {
    const std::string body = "backbone.0.body";
    if (make_conv(m, tm, body + ".conv1", body + ".bn1", 64, 3, 7, 7, 2, 3, &m->stem)) return 1;
    struct LayerCfg { const char* name; int n, planes, stride; };
    const LayerCfg layers[3] = {{"layer1", 3, 64, 1}, {"layer2", 4, 128, 2}, {"layer3", 6, 256, 2}};
    int inplanes = 64;
    for (const LayerCfg& L : layers) {
        for (int i = 0; i < L.n; ++i) {
            const std::string p = body + "." + L.name + "." + std::to_string(i);
            Block b;
            const int stride = (i == 0) ? L.stride : 1;
            if (make_conv(m, tm, p + ".conv1", p + ".bn1", L.planes, inplanes, 1, 1, 1, 0, &b.c1)) return 1;
            if (make_conv(m, tm, p + ".conv2", p + ".bn2", L.planes, L.planes, 3, 3, stride, 1, &b.c2)) return 1;
            if (make_conv(m, tm, p + ".conv3", p + ".bn3", L.planes * 4, L.planes, 1, 1, 1, 0, &b.c3)) return 1;
            b.has_ds = (i == 0);
            if (b.has_ds && make_conv(m, tm, p + ".downsample.0", p + ".downsample.1", L.planes * 4, inplanes, 1, 1, stride, 0, &b.ds)) return 1;
            m->blocks.push_back(b);
            inplanes = L.planes * 4;
        }
    }
    {
        const cotr_tensor* w = tm.get("input_proj.weight", {kDModel, 1024, 1, 1});
        const cotr_tensor* b = tm.get("input_proj.bias", {kDModel});
        if (!w || !b) return 1;
        std::vector<float> bv = to_vec(b, kDModel);
        if (make_linear(m, to_vec(w, (size_t)kDModel * 1024), &bv, kDModel, 1024, &m->proj)) return 1;
    }
    if (upload(m, grid_position_table(), &m->pos)) return 1;

    const float qscale = 1.0f / std::sqrt((float)kHeadDim);   // F.multi_head_attention_forward: q * head_dim^-0.5
    const size_t DD = (size_t)kDModel * kDModel;

    auto linear_from = [&](const std::string& prefix, int N, int K, DevLinear* out) -> int {
        const cotr_tensor* w = tm.get(prefix + ".weight", {N, K});
        const cotr_tensor* b = tm.get(prefix + ".bias", {N});
        if (!w || !b) return 1;
        std::vector<float> bv = to_vec(b, N);
        return make_linear(m, to_vec(w, (size_t)N * K), &bv, N, K, out);
    };

    // same, for a layer whose input is a deferred LayerNorm `norm` (weight / bias in the checkpoint)
    auto linear_ln_from = [&](const std::string& prefix, int N, int K, const std::string& norm, DevLinear* out) -> int {
        const cotr_tensor* w = tm.get(prefix + ".weight", {N, K});
        const cotr_tensor* b = tm.get(prefix + ".bias", {N});
        const cotr_tensor* g = tm.get(norm + ".weight", {K});
        const cotr_tensor* be = tm.get(norm + ".bias", {K});
        if (!w || !b || !g || !be) return 1;
        std::vector<float> bv = to_vec(b, N);
        return make_linear_ln(m, to_vec(w, (size_t)N * K), &bv, N, K, g->data, be->data, out);
    };

    // constant position-bias matrices, produced with the fp32 SIMT GEMM once per model
    struct PosBiasJob { std::vector<float> w_masked; std::vector<float> bias; int N; float** dst; };
    std::vector<PosBiasJob> jobs;

    for (int l = 0; l < kEncLayers; ++l) {
        const std::string p = "transformer.encoder.layers." + std::to_string(l);
        EncLayer& e = m->enc[l];
        const cotr_tensor* w = tm.get(p + ".self_attn.in_proj_weight", {3 * kDModel, kDModel});
        const cotr_tensor* b = tm.get(p + ".self_attn.in_proj_bias", {3 * kDModel});
        if (!w || !b) return 1;
        std::vector<float> wv = to_vec(w, 3 * DD), bv = to_vec(b, 3 * kDModel);
        for (size_t i = 0; i < DD; ++i) wv[i] *= qscale;
        for (int i = 0; i < kDModel; ++i) bv[i] *= qscale;
        std::vector<float> wm = wv;                               // value rows see x only, not x + pos
        std::fill(wm.begin() + 2 * DD, wm.end(), 0.f);
        jobs.push_back({wm, bv, 3 * kDModel, &e.add_qkv});
        if (l == 0) {
            if (make_linear(m, wv, nullptr, 3 * kDModel, kDModel, &e.qkv)) return 1;
        } else {
            // the layer input is norm2 of the previous layer, applied on the fly by this GEMM (tensor-core path)
            const std::string prev = "transformer.encoder.layers." + std::to_string(l - 1) + ".norm2";
            const cotr_tensor* g = tm.get(prev + ".weight", {kDModel});
            const cotr_tensor* be = tm.get(prev + ".bias", {kDModel});
            if (!g || !be) return 1;
            std::vector<float> cb;
            if (make_linear_ln(m, wv, nullptr, 3 * kDModel, kDModel, g->data, be->data, &e.qkv, &cb)) return 1;
            std::vector<float> bv_tc = bv;
            for (int i = 0; i < 3 * kDModel; ++i) bv_tc[i] += cb[i];
            jobs.push_back({wm, bv_tc, 3 * kDModel, &e.add_qkv_tc});
        }
        if (linear_from(p + ".self_attn.out_proj", kDModel, kDModel, &e.o)) return 1;
        if (linear_ln_from(p + ".linear1", kFF, kDModel, p + ".norm1", &e.l1)) return 1;
        if (linear_from(p + ".linear2", kDModel, kFF, &e.l2)) return 1;
        if (upload_vec(m, tm, p + ".norm1.weight", kDModel, &e.ln1_g) || upload_vec(m, tm, p + ".norm1.bias", kDModel, &e.ln1_b) ||
            upload_vec(m, tm, p + ".norm2.weight", kDModel, &e.ln2_g) || upload_vec(m, tm, p + ".norm2.bias", kDModel, &e.ln2_b))
            return 1;
    }

    const int kKvN = 2 * kKCols;   // 3072
    std::vector<float> kv_w((size_t)kKvN * kDModel), kv_wm((size_t)kKvN * kDModel, 0.f), kv_b(kKvN);
    std::vector<float> qp_w((size_t)kQpCols * kDModel), qp_b(kQpCols);
    for (int l = 0; l < kDecLayers; ++l) {
        const std::string p = "transformer.decoder.layers." + std::to_string(l);
        DecLayer& d = m->dec[l];
        const cotr_tensor* w = tm.get(p + ".multihead_attn.in_proj_weight", {3 * kDModel, kDModel});
        const cotr_tensor* b = tm.get(p + ".multihead_attn.in_proj_bias", {3 * kDModel});
        if (!w || !b) return 1;
        std::vector<float> wq = to_vec(w, DD);
        for (float& v : wq) v *= qscale;
        if (l == 0) {
            if (make_linear(m, wq, nullptr, kDModel, kDModel, &d.q)) return 1;       // (never run: tgt = 0 in layer 0)
        } else {
            const std::string prev = "transformer.decoder.layers." + std::to_string(l - 1) + ".norm3";
            const cotr_tensor* g = tm.get(prev + ".weight", {kDModel});
            const cotr_tensor* be = tm.get(prev + ".bias", {kDModel});
            if (!g || !be) return 1;
            if (make_linear_ln(m, wq, nullptr, kDModel, kDModel, g->data, be->data, &d.q)) return 1;
        }
        memcpy(qp_w.data() + (size_t)l * DD, wq.data(), DD * sizeof(float));
        for (int i = 0; i < kDModel; ++i) qp_b[l * kDModel + i] = b->data[i] * qscale;
        // K rows then V rows of layer l
        memcpy(kv_w.data() + (size_t)l * 2 * DD, w->data + DD, 2 * DD * sizeof(float));
        memcpy(kv_wm.data() + (size_t)l * 2 * DD, w->data + DD, DD * sizeof(float));   // only K sees pos
        memcpy(kv_b.data() + (size_t)l * 2 * kDModel, b->data + kDModel, 2 * kDModel * sizeof(float));
        if (linear_from(p + ".multihead_attn.out_proj", kDModel, kDModel, &d.o)) return 1;
        if (linear_ln_from(p + ".linear1", kFF, kDModel, p + ".norm2", &d.l1)) return 1;
        if (linear_from(p + ".linear2", kDModel, kFF, &d.l2)) return 1;
        if (upload_vec(m, tm, p + ".norm2.weight", kDModel, &d.ln2_g) || upload_vec(m, tm, p + ".norm2.bias", kDModel, &d.ln2_b) ||
            upload_vec(m, tm, p + ".norm3.weight", kDModel, &d.ln3_g) || upload_vec(m, tm, p + ".norm3.bias", kDModel, &d.ln3_b))
            return 1;
        // decoder.layers.N.norm1.* exists in the checkpoint but transformer.py:185-201 never uses it.
    }
    {
        const std::string last = "transformer.encoder.layers." + std::to_string(kEncLayers - 1) + ".norm2";
        const cotr_tensor* g = tm.get(last + ".weight", {kDModel});
        const cotr_tensor* be = tm.get(last + ".bias", {kDModel});
        if (!g || !be) return 1;
        std::vector<float> cb;
        if (make_linear_ln(m, kv_w, nullptr, kKvN, kDModel, g->data, be->data, &m->kv_all, &cb)) return 1;
        std::vector<float> kv_b_tc = kv_b;
        for (int i = 0; i < kKvN; ++i) kv_b_tc[i] += cb[i];
        jobs.push_back({kv_wm, kv_b_tc, kKvN, &m->add_kv_tc});
    }
    jobs.push_back({kv_wm, kv_b, kKvN, &m->add_kv});
    if (make_linear(m, qp_w, &qp_b, kQpCols, kDModel, &m->qpos_all)) return 1;
    if (upload_vec(m, tm, "transformer.decoder.norm.weight", kDModel, &m->dec_norm_g) ||
        upload_vec(m, tm, "transformer.decoder.norm.bias", kDModel, &m->dec_norm_b))
        return 1;
    if (linear_from("corr_embed.layers.0", kDModel, kDModel, &m->head[0])) return 1;
    if (linear_from("corr_embed.layers.1", kDModel, kDModel, &m->head[1])) return 1;
    if (linear_from("corr_embed.layers.2", 2, kDModel, &m->head[2])) return 1;

    // add matrices: pos [512,256] x Wmasked^T + bias  (fp32 SIMT GEMM on the split16 pos table, fp32 result)
    TmpSplit pos16;
    if (pos16.from_f32(m->pos, (size_t)kTokens * kDModel)) return 1;
    for (PosBiasJob& j : jobs) {
        DevAllocs tmp;
        float *wd = nullptr, *bd = nullptr;
        if (tmp.upload((void**)&wd, j.w_masked.data(), j.w_masked.size() * sizeof(float)) ||
            tmp.upload((void**)&bd, j.bias.data(), j.bias.size() * sizeof(float)))
            return 1;
        if (dev_alloc(m, (void**)j.dst, (size_t)kTokens * j.N * sizeof(float))) return 1;
        GemmParams p = gemm_base(kTokens, j.N, kDModel, cs(pos16.t), kDModel, wd, nullptr, 1.f, kNoSplit, j.N);
        p.bias = bd;
        if (launch_gemm_simt_raw(p, *j.dst, 0)) return 1;
        COTR_CHECK_CUDA(cudaDeviceSynchronize());
    }
    if (!m->enc[0].add_qkv_tc) m->enc[0].add_qkv_tc = m->enc[0].add_qkv;     // layer 0 reads the un-normalised input projection
    return 0;
}

}  // namespace
}  // namespace cotr

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
using namespace cotr;

extern "C" {

const char* cotr_last_error(void) { return g_error; }
const char* cotr_version(void) { return "cotr_b200 0.3 (sm_90a)"; }

int cotr_create(int device, const cotr_tensor* tensors, int n_tensors, cotr_model** out) {
    COTR_CHECK(out != nullptr && tensors != nullptr && n_tensors > 0, "cotr_create: bad arguments");
    *out = nullptr;
    int n_dev = 0;
    COTR_CHECK_CUDA(cudaGetDeviceCount(&n_dev));
    COTR_CHECK(device >= 0 && device < n_dev, "cotr_create: CUDA device %d not available (%d visible)", device, n_dev);
    COTR_CHECK_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    COTR_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
    COTR_CHECK(prop.major == 9 && prop.minor == 0, "cotr_create: this library is built for sm_90a only; device %d is sm_%d%d", device, prop.major, prop.minor);
    TensorMap tm;
    for (int i = 0; i < n_tensors; ++i) {
        COTR_CHECK(tensors[i].name != nullptr, "cotr_create: tensor %d has no name", i);
        tm.m[tensors[i].name] = &tensors[i];
    }
    cotr_model* m = new cotr_model();
    m->device = device;
    g_error[0] = 0;
    if (build_model(m, tm) || cotr_context_create(m, 1, &m->own_ctx) ||
        cudaStreamCreateWithFlags(&m->host_stream, cudaStreamNonBlocking) != cudaSuccess) {
        if (g_error[0] == 0) set_error("cotr_create: stream creation failed");
        cotr_destroy(m);
        return 1;
    }
    *out = m;
    return 0;
}

void cotr_destroy(cotr_model* m) {
    if (!m) return;
    cudaSetDevice(m->device);
    cudaDeviceSynchronize();
    if (m->own_ctx) cotr_context_destroy(m->own_ctx);
    for (void* p : m->allocs) cudaFree(p);
    Workspace& w = m->ws;
    ws_release(encode_ws_bufs(w, 0));
    ws_release(decode_ws_bufs(w, 0));
    ws_release(match_ws_bufs(w, 0));
    ws_release(refine_ws_bufs(w, RefineCaps()));
    for (float** b : {&w.img_stage, &w.q_stage, &w.pred_stage}) ws_free_f32(b);
    if (m->host_stream) cudaStreamDestroy(m->host_stream);
    for (auto& kv : m->graphs) cudaGraphExecDestroy(kv.second);
    preprocessor_destroy(m->pre);
    flow_merger_destroy(m->merger);
    resizer_destroy(m->resizer);
    for (cudaEvent_t e : m->prof_events) cudaEventDestroy(e);
    if (m->order_event) cudaEventDestroy(m->order_event);
    delete m;
}

int cotr_context_create(cotr_model* m, int max_pairs, cotr_context** out) {
    COTR_CHECK(m && out && max_pairs >= 1, "cotr_context_create: bad arguments");
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    cotr_context* c = new cotr_context();
    c->model = m;
    c->max_pairs = max_pairs;
    const size_t img_bytes = (size_t)max_pairs * kDecLayers * kHeads * kAttnHeadImgBytes;
    if (ws_alloc(&c->k, (size_t)max_pairs * kTokens * kKCols) || ws_alloc(&c->vt, (size_t)max_pairs * kDecLayers * kVtLayer) ||
        cudaMalloc((void**)&c->img, img_bytes) != cudaSuccess || cudaMemset(c->img, 0, img_bytes) != cudaSuccess) {
        set_error("cotr_context_create: out of device memory for %d pairs", max_pairs);
        cotr_context_destroy(c);
        return 1;
    }
    *out = c;
    return 0;
}

void cotr_context_destroy(cotr_context* c) {
    if (!c) return;
    ws_free(&c->k);
    ws_free(&c->vt);
    if (c->img) cudaFree(c->img);
    delete c;
}

int cotr_encode_context(cotr_model* m, const float* img_dev, int B, cotr_context* ctx, void* cuda_stream) {
    COTR_CHECK(m && img_dev, "cotr_encode_context: null argument");
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    CallOrder order(m, (cudaStream_t)cuda_stream);
    m->launches = 0;
    return encode_impl(m, img_dev, B, ctx, (cudaStream_t)cuda_stream);
}

int cotr_decode(cotr_model* m, const cotr_context* ctx, const float* queries_dev, int B, int Q, float* pred_dev, void* cuda_stream) {
    COTR_CHECK(m && (Q == 0 || (queries_dev && pred_dev)), "cotr_decode: null argument");
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    CallOrder order(m, (cudaStream_t)cuda_stream);
    m->launches = 0;
    return decode_impl(m, ctx, queries_dev, B, Q, pred_dev, (cudaStream_t)cuda_stream);
}

int cotr_decode_ragged(cotr_model* m, const cotr_context* ctx, const float* queries_dev, const int64_t* offsets_host, int B,
                       float* pred_dev, void* cuda_stream) {
    const char* fn = "cotr_decode_ragged";
    COTR_CHECK(m != nullptr, "%s: null model", fn);
    m->launches = 0;
    if (check_decode_context(m, fn, B, ctx)) return 1;
    COTR_CHECK(offsets_host != nullptr, "%s: null offsets_host", fn);
    COTR_CHECK(offsets_host[0] == 0, "%s: offsets_host[0] = %lld, must be 0", fn, (long long)offsets_host[0]);
    for (int p = 0; p < B; ++p)
        COTR_CHECK(offsets_host[p + 1] >= offsets_host[p], "%s: offsets_host decreases at pair %d (%lld -> %lld)", fn, p,
                   (long long)offsets_host[p], (long long)offsets_host[p + 1]);
    const int64_t R = offsets_host[B];
    COTR_CHECK(R <= INT32_MAX, "%s: %lld query rows in one call (at most %d)", fn, (long long)R, INT32_MAX);
    if (R == 0) return 0;
    COTR_CHECK(queries_dev && pred_dev, "%s: null queries_dev or pred_dev for %lld rows", fn, (long long)R);
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    CallOrder order(m, (cudaStream_t)cuda_stream);
    return decode_ragged_impl(m, ctx, queries_dev, offsets_host, B, pred_dev, (cudaStream_t)cuda_stream);
}

namespace {
int check_layer_mask(const char* fn, int layer_mask, const float* attn_dev, int n_layers) {
    COTR_CHECK((layer_mask & ~((1 << n_layers) - 1)) == 0, "%s: layer_mask 0x%x selects layers outside 0..%d", fn, (unsigned)layer_mask, n_layers - 1);
    COTR_CHECK(layer_mask == 0 || attn_dev != nullptr, "%s: null attn_dev for layer_mask 0x%x", fn, (unsigned)layer_mask);
    return 0;
}
}  // namespace

int cotr_encode_context_attention(cotr_model* m, const float* img_dev, int B, cotr_context* ctx, int layer_mask, float* attn_dev,
                                  void* cuda_stream) {
    COTR_CHECK(m && img_dev, "cotr_encode_context_attention: null argument");
    if (check_layer_mask("cotr_encode_context_attention", layer_mask, attn_dev, kEncLayers)) return 1;
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    CallOrder order(m, (cudaStream_t)cuda_stream);
    m->launches = 0;
    return encode_impl(m, img_dev, B, ctx, (cudaStream_t)cuda_stream, attn_maps(layer_mask, attn_dev, B, kTokens));
}

int cotr_encode_images(cotr_model* m, const float* img_dev, int N, void* feat_dev, void* cuda_stream) {
    COTR_CHECK(m && img_dev && feat_dev, "cotr_encode_images: null argument");
    COTR_CHECK(N >= 1, "cotr_encode_images: N must be >= 1 (got %d)", N);
    COTR_CHECK(((uintptr_t)img_dev & 3) == 0, "cotr_encode_images: img_dev is not 4-byte aligned");
    COTR_CHECK(((uintptr_t)feat_dev & 15) == 0, "cotr_encode_images: feat_dev is not 16-byte aligned");
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    CallOrder order(m, (cudaStream_t)cuda_stream);
    m->launches = 0;
    return encode_images_impl(m, img_dev, N, feat_dev, (cudaStream_t)cuda_stream);
}

int cotr_encode_context_pairs(cotr_model* m, const void* feat_dev, int n_images, const int32_t* pairs_host, int B,
                              cotr_context* ctx, int layer_mask, float* attn_dev, void* cuda_stream) {
    const char* fn = "cotr_encode_context_pairs";
    COTR_CHECK(m && feat_dev && pairs_host, "%s: null argument", fn);
    COTR_CHECK(((uintptr_t)feat_dev & 15) == 0, "%s: feat_dev is not 16-byte aligned", fn);
    COTR_CHECK(((uintptr_t)attn_dev & 3) == 0, "%s: attn_dev is not 4-byte aligned", fn);
    COTR_CHECK(n_images >= 1, "%s: n_images must be >= 1 (got %d)", fn, n_images);
    if (check_context(m, fn, B, ctx)) return 1;
    for (int i = 0; i < 2 * B; ++i)
        COTR_CHECK(pairs_host[i] >= 0 && pairs_host[i] < n_images, "%s: pairs[%d][%d] = %d is outside [0, %d)", fn, i / 2, i % 2,
                   (int)pairs_host[i], n_images);
    if (check_layer_mask(fn, layer_mask, attn_dev, kEncLayers)) return 1;
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    CallOrder order(m, (cudaStream_t)cuda_stream);
    m->launches = 0;
    return encode_pairs_impl(m, feat_dev, n_images, pairs_host, B, ctx, (cudaStream_t)cuda_stream,
                             attn_maps(layer_mask, attn_dev, B, kTokens));
}

int cotr_decode_attention(cotr_model* m, const cotr_context* ctx, const float* queries_dev, int B, int Q, int layer_mask,
                          float* attn_dev, float* pred_dev, void* cuda_stream) {
    COTR_CHECK(m && (Q == 0 || (queries_dev && pred_dev)), "cotr_decode_attention: null argument");
    if (check_layer_mask("cotr_decode_attention", layer_mask, attn_dev, kDecLayers)) return 1;
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    CallOrder order(m, (cudaStream_t)cuda_stream);
    m->launches = 0;
    return decode_impl(m, ctx, queries_dev, B, Q, pred_dev, (cudaStream_t)cuda_stream, attn_maps(layer_mask, attn_dev, B, Q));
}

namespace {

int ensure_stage(cotr_model* m, int B, int Q) {
    Workspace& w = m->ws;
    const size_t img_elems = (size_t)B * 3 * COTR_CANVAS_H * COTR_CANVAS_W;
    const size_t q_elems = (size_t)B * Q * 2;
    if (img_elems > w.img_stage_elems) {
        COTR_CHECK_CUDA(cudaDeviceSynchronize());
        drop_graphs(m);
        ws_free_f32(&w.img_stage);
        w.img_stage_elems = 0;
        if (ws_alloc_f32(&w.img_stage, img_elems)) return 1;
        w.img_stage_elems = img_elems;
    }
    if (q_elems > w.q_stage_elems) {
        COTR_CHECK_CUDA(cudaDeviceSynchronize());
        drop_graphs(m);
        ws_free_f32(&w.q_stage); ws_free_f32(&w.pred_stage);
        w.q_stage_elems = 0;
        if (ws_alloc_f32(&w.q_stage, q_elems ? q_elems : 2) || ws_alloc_f32(&w.pred_stage, q_elems ? q_elems : 2)) return 1;
        w.q_stage_elems = q_elems;
    }
    return 0;
}

int forward_eager(cotr_model* m, const float* img, const float* queries, int B, int Q, float* pred, cudaStream_t s) {
    if (m->own_ctx->max_pairs < B) {
        COTR_CHECK_CUDA(cudaDeviceSynchronize());
        drop_graphs(m);
        cotr_context_destroy(m->own_ctx);
        m->own_ctx = nullptr;
        if (cotr_context_create(m, B, &m->own_ctx)) return 1;
    }
    m->launches = 0;
    if (encode_impl(m, img, B, m->own_ctx, s)) return 1;
    return decode_impl(m, m->own_ctx, queries, B, Q, pred, s);
}

// Forward on the staging buffers (img_stage, q_stage -> pred_stage): graph replay when a graph exists for the shape.
int forward_staged(cotr_model* m, int B, int Q, cudaStream_t s) {
    Workspace& w = m->ws;
    const bool graphable = m->graph_mode && !m->prof_on;
    const long long key = ((long long)B << 32) | (unsigned)Q;
    if (graphable) {
        auto it = m->graphs.find(key);
        if (it != m->graphs.end()) {
            COTR_CHECK_CUDA(cudaGraphLaunch(it->second, s));
            m->launches = m->graph_launches[key];
            return 0;
        }
        if (m->shapes_seen.count(key) && m->graphs.size() < 256) {
            // second call with this shape: workspace, contexts and kernel attributes are in place -> capture
            cudaGraph_t graph = nullptr;
            // the legacy default stream (what torch hands over by default) cannot be captured: record on ours,
            // the resulting graph is launched on the caller's stream either way
            cudaStream_t cs = (s == nullptr || s == cudaStreamLegacy || s == cudaStreamPerThread) ? m->host_stream : s;
            COTR_CHECK_CUDA(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
            const int rc = forward_eager(m, w.img_stage, w.q_stage, B, Q, w.pred_stage, cs);
            const cudaError_t e = cudaStreamEndCapture(cs, &graph);
            if (rc || e != cudaSuccess || graph == nullptr) {
                if (graph) cudaGraphDestroy(graph);
                if (!rc) set_error("cotr_forward: stream capture failed: %s", cudaGetErrorString(e));
                return 1;
            }
            cudaGraphExec_t exec = nullptr;
            const cudaError_t ei = cudaGraphInstantiate(&exec, graph, 0);
            cudaGraphDestroy(graph);
            COTR_CHECK(ei == cudaSuccess, "cotr_forward: cudaGraphInstantiate failed: %s", cudaGetErrorString(ei));
            m->graphs[key] = exec;
            m->graph_launches[key] = m->launches;
            COTR_CHECK_CUDA(cudaGraphLaunch(exec, s));
            return 0;
        }
        m->shapes_seen.insert(key);
    }
    return forward_eager(m, w.img_stage, w.q_stage, B, Q, w.pred_stage, s);
}

// get_patch_centered_at's two crop sides of one level into sizes[0] ("from") and sizes[1] ("to"), each checked to be at
// least 2 and to fit its image; `where` opens the error message.
int refine_crop_sides(const char* where, int level, double zoom, int h_from, int w_from, double s_from, int h_to, int w_to, double s_to,
                      int* sizes) {
    for (int side = 0; side < 2; ++side) {
        const int h = side ? h_to : h_from, w = side ? w_to : w_from;
        sizes[side] = refine_crop_size(h, w, (side ? s_to : s_from) * zoom);
        COTR_CHECK(sizes[side] >= 2 && sizes[side] <= h && sizes[side] <= w, "%s: level %d: %s crop side %d in a %d x %d image", where,
                   level, side ? "to" : "from", sizes[side], h, w);
    }
    return 0;
}

// The crop template of level `level` of L from one image to another: everything of a RefineLevel but its entries (task0,
// count, chunk), with the Pillow coefficient tables of both crop sides (uploaded once per side length).
int refine_level_template(cotr_model* m, const uint8_t* img_from, int h_from, int w_from, const uint8_t* img_to, int h_to, int w_to,
                          int fs, int ts, int level, int L, double rel, RefineLevel* lv) {
    if (!m->pre) m->pre = preprocessor_create();
    *lv = RefineLevel();
    lv->level = level; lv->levels = L;
    lv->h_from = h_from; lv->w_from = w_from; lv->h_to = h_to; lv->w_to = w_to;
    lv->thr = refine_threshold(rel, h_to, w_to);
    lv->from.img = img_from; lv->from.img_w = w_from;
    lv->to.img = img_to; lv->to.img_w = w_to;
    return preprocess_coeffs(m->pre, fs, &lv->from) || preprocess_coeffs(m->pre, ts, &lv->to);
}

// One level of a zoom-in walk (refine.cu's entries, squads and tables), enqueued without a wait: the pilots' crops, rects
// and queries, then, when `step`, their canvases, the forward at (n_squads, longest) and every member's step, with the
// good count going to *good_count.  Adds its launches to m->launches.
int refine_level(cotr_model* m, const RefineLevel& lv, const int32_t* ids, const int32_t* squad, const int32_t* rank, int n_squads,
                 int longest, bool step, const double* loc_from, double* history, int32_t* rects, int32_t* good, int32_t* good_count,
                 cudaStream_t s) {
    Workspace& w = m->ws;
    Run r{m, s};
    {
        LaunchScope scope(r, K_REFINE_GEOMETRY, lv.count, lv.level, 0);
        if (launch_refine_geometry(lv, ids, squad, rank, n_squads, longest, loc_from, history, w.refine_sides, rects, w.refine_q,
                                   w.refine_counts, s)) return 1;
    }
    if (!step) return 0;
    {
        LaunchScope scope(r, K_RESIZE_H, 2 * n_squads, 0, 0);
        if (launch_resize_h(w.refine_sides, 2 * n_squads, std::max(lv.from.size, lv.to.size), w.refine_tmp, s)) return 1;
    }
    {
        LaunchScope scope(r, K_RESIZE_V, 2 * n_squads, 0, 0);
        if (launch_resize_v(w.refine_sides, 2 * n_squads, w.refine_tmp, w.refine_canvas, s)) return 1;
    }
    const int launches = m->launches;     // forward_eager counts its own launches from 0
    if (forward_eager(m, w.refine_canvas, w.refine_q, n_squads, longest, w.refine_pred, s)) return 1;
    m->launches += launches;
    LaunchScope scope(r, K_REFINE_STEP, lv.count, lv.level, 0);
    return launch_refine_step(lv, ids, squad, rank, longest, w.refine_pred, rects, history, good, good_count, w.refine_counts, s);
}

// The zoom-in walk of cotr_refine, arguments checked.  sizes: n_groups x L x 2 crop sides.  The host loop's batches
// fall on the chunks: its first `batch` open tasks are the first chunk not yet finished, and after one step each of them
// is open again one level deeper, so a chunk walks all L levels before the next one starts.  Its good count, and so the
// max_corrs stop, changes only after a chunk's last level.  Waves only decide how often the host looks at the counts.
int refine_walk_impl(cotr_model* m, const uint8_t* const* images, const int32_t* hw, const cotr_refine_group* groups, int n_groups,
                     const std::vector<int>& sizes, int L, int batch, int wave, int64_t max_good, double rel,
                     const double* loc_from, const double* loc_to, double* history, int32_t* rects, int32_t* good,
                     int64_t* walked, int32_t* status, cudaStream_t s) {
    struct Chunk { int group, first, count; };
    std::vector<Chunk> chunks;
    size_t tmp = 256;
    for (int g = 0; g < n_groups; ++g) {
        const cotr_refine_group& G = groups[g];
        for (int f = G.first; f < G.first + G.count; f += batch) chunks.push_back({g, f, std::min(batch, G.first + G.count - f)});
        const size_t rows = (size_t)std::min(batch, G.count);
        for (int l = 0; l < L; ++l) tmp = std::max(tmp, rows * (sizes[(g * L + l) * 2] + sizes[(g * L + l) * 2 + 1]) * 256 * 3);
    }
    const int64_t n = groups[n_groups - 1].first + (int64_t)groups[n_groups - 1].count;
    const int64_t n_chunks = (int64_t)chunks.size();
    status[0] = status[1] = status[2] = 0;
    *walked = 0;
    if (n == 0 || max_good <= 0) { m->launches = 0; return 0; }

    // the per-level crop templates
    std::vector<RefineLevel> levels((size_t)n_groups * L);
    for (int g = 0; g < n_groups; ++g) {
        const cotr_refine_group& G = groups[g];
        const int a = G.image_from, b = G.image_to;
        for (int l = 0; l < L; ++l)
            if (refine_level_template(m, images[a], hw[2 * a], hw[2 * a + 1], images[b], hw[2 * b], hw[2 * b + 1], sizes[(g * L + l) * 2],
                                      sizes[(g * L + l) * 2 + 1], l, L, rel, &levels[(size_t)g * L + l])) return 1;
    }
    // squads of one: chunk task i is entry i, squad i, rank 0
    const int64_t rows = std::min<int64_t>(batch, n);
    RefineCaps need;
    need.squads = need.rows = need.ids = rows; need.tmp = tmp; need.chunks = n_chunks;
    if (ensure_refine_ws(m, need)) return 1;
    Workspace& w = m->ws;
    int32_t* chunk_good = reinterpret_cast<int32_t*>(w.refine_counts + 1);
    COTR_CHECK_CUDA(cudaMemsetAsync(w.refine_counts, 0xFF, sizeof(unsigned long long), s));
    COTR_CHECK_CUDA(cudaMemsetAsync(chunk_good, 0, (size_t)n_chunks * sizeof(int32_t), s));
    // history row 0 = the first guesses
    COTR_CHECK_CUDA(cudaMemcpy2DAsync(history, (size_t)(L + 1) * 2 * sizeof(double), loc_to, 2 * sizeof(double), 2 * sizeof(double),
                                      (size_t)n, cudaMemcpyDeviceToDevice, s));

    m->launches = 0;
    const bool look_each_wave = max_good < n;
    std::vector<int32_t> counts;
    int64_t good_so_far = 0;
    for (int64_t w0 = 0; w0 < n_chunks; w0 += wave) {
        const int64_t w1 = std::min<int64_t>(n_chunks, w0 + wave);
        for (int64_t c = w0; c < w1; ++c) {
            const Chunk& ch = chunks[c];
            for (int l = 0; l < L; ++l) {
                RefineLevel lv = levels[(size_t)ch.group * L + l];
                lv.task0 = ch.first; lv.count = ch.count; lv.chunk = (int)c;
                if (refine_level(m, lv, w.refine_iota, w.refine_iota, w.refine_zeros, ch.count, 1, true, loc_from, history, rects, good,
                                 chunk_good + c, s)) return 1;
            }
        }
        const bool last = w1 == n_chunks;
        if (!look_each_wave && !last) continue;
        // one small copy: the status word, then (when the stop may fall in this wave) the wave's good counts
        const int64_t n_read = look_each_wave ? w1 - w0 : 0;
        counts.assign(2 + (size_t)n_read, 0);
        COTR_CHECK_CUDA(cudaMemcpyAsync(counts.data(), w.refine_counts, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
        if (n_read) COTR_CHECK_CUDA(cudaMemcpyAsync(counts.data() + 2, chunk_good + w0, (size_t)n_read * sizeof(int32_t),
                                                    cudaMemcpyDeviceToHost, s));
        COTR_CHECK_CUDA(cudaStreamSynchronize(s));
        unsigned long long key;
        memcpy(&key, counts.data(), sizeof(key));
        int64_t stop = -1;              // the chunk in which the good count reached max_good
        for (int64_t c = w0; c < w1 && look_each_wave; ++c) {
            good_so_far += counts[2 + (c - w0)];
            if (good_so_far >= max_good) { stop = c; break; }
        }
        if (key != ~0ull) {
            const int64_t bad_chunk = (int64_t)(key >> 5);
            if (stop < 0 || bad_chunk <= stop) {      // the host loop meets it before it stops
                status[0] = (int32_t)(key & 3);
                status[1] = (int32_t)bad_chunk;
                status[2] = (int32_t)((key >> 2) & 7);
                *walked = chunks[bad_chunk].first;
                return 0;
            }
        }
        if (stop >= 0) {
            *walked = chunks[stop].first + (int64_t)chunks[stop].count;
            return 0;
        }
    }
    *walked = n;
    return 0;
}

// One grouped batch of cotr_refine_grouped, arguments checked; fs / ts are the level's two crop sides.  The candidates'
// end points and pilot boxes, and the squads, are made on the device; one small copy brings back the squad table, the
// candidates' crop failures and, while the max_corrs stop can fall, the good count.  Then the batch either ends there
// (a pilot whose crop raises in Python), or only writes its rects (the max_corrs stop: the squads are submitted, not
// stepped), or enqueues its geometry, canvases, forward and step without another wait.
int refine_grouped_impl(cotr_model* m, const uint8_t* img_from, int h_from, int w_from, const uint8_t* img_to, int h_to, int w_to,
                        int fs, int ts, int level, int L, const int32_t* ids_host, int n_ids, int n_tasks, int batch_size,
                        int max_load, int64_t max_good, double rel, const double* loc_from, double* history, int32_t* rects,
                        int32_t* good, int32_t* squad_host, int32_t* result, cudaStream_t s) {
    for (int k = 0; k < 5; ++k) result[k] = 0;
    m->launches = 0;
    if (n_ids == 0) return 0;
    RefineLevel lv;
    if (refine_level_template(m, img_from, h_from, w_from, img_to, h_to, w_to, fs, ts, level, L, rel, &lv)) return 1;
    lv.count = n_ids;
    // every buffer at its largest for this batch before the first launch: growing one later would drop the squad table
    RefineCaps need;
    need.squads = std::min(batch_size, n_ids);
    need.rows = need.squads * std::min<int64_t>((int64_t)max_load + 1, n_ids);
    need.ids = n_ids;
    need.tmp = (size_t)need.squads * (fs + ts) * 256 * 3;
    if (ensure_refine_ws(m, need)) return 1;
    if (m->grouped_ids.upload(ids_host, (size_t)n_ids, s)) return 1;
    Workspace& w = m->ws;
    const int32_t* ids = m->grouped_ids.dev;
    int32_t* n_squads_dev = w.grouped_tab;
    int32_t* squad = w.grouped_tab + 1;
    int32_t* fail = squad + n_ids;
    int32_t* rank = fail + n_ids;

    Run r{m, s};
    {
        LaunchScope scope(r, K_GROUPED_CANDIDATES, n_ids, level, 0);
        if (launch_grouped_candidates(lv, ids, loc_from, history, w.grouped_pts, w.grouped_box, fail, s)) return 1;
    }
    {
        LaunchScope scope(r, K_GROUP_TASKS, n_ids, level, 0);
        if (group_tasks_launch(w.grouped_pts, w.grouped_box, n_ids, batch_size, max_load, squad, rank, n_squads_dev, s)) return 1;
    }
    std::vector<int32_t> tab(1 + 2 * (size_t)n_ids);
    int32_t good_count = 0;
    const bool read_good = max_good > 0 && max_good <= n_tasks;     // otherwise the count cannot decide the stop
    COTR_CHECK_CUDA(cudaMemcpyAsync(tab.data(), w.grouped_tab, tab.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    if (read_good) COTR_CHECK_CUDA(cudaMemcpyAsync(&good_count, good + n_tasks, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    COTR_CHECK_CUDA(cudaStreamSynchronize(s));
    const int n_squads = tab[0];
    std::vector<int> members((size_t)n_squads, 0);
    int num_steps = 0, status = 0;
    for (int i = 0; i < n_ids; ++i) {
        const int sq = tab[1 + i];
        squad_host[i] = sq;
        if (sq < 0) continue;
        // a squad's pilot precedes its members in list order, and pilots come in squad order: the first failing pilot
        // met here is the one at which the host loop raises
        if (members[sq] == 0 && status == 0) status = tab[1 + n_ids + i];
        ++members[sq];
        ++num_steps;
    }
    const int longest = n_squads ? *std::max_element(members.begin(), members.end()) : 0;
    result[0] = n_squads; result[1] = longest; result[2] = num_steps; result[4] = status;
    if (status != 0 || n_squads == 0) return 0;
    const bool step = !(max_good <= 0 || (read_good && good_count >= max_good));
    COTR_CHECK_CUDA(cudaMemsetAsync(w.refine_q, 0, (size_t)n_squads * longest * 2 * sizeof(float), s));    // padding rows
    if (refine_level(m, lv, ids, squad, rank, n_squads, longest, step, loc_from, history, rects, good, good + n_tasks, s)) return 1;
    result[3] = step;
    return 0;
}

}  // namespace

int cotr_forward(cotr_model* m, const float* img_dev, const float* queries_dev, int B, int Q, float* pred_dev, void* cuda_stream) {
    COTR_CHECK(m && img_dev && (Q == 0 || (queries_dev && pred_dev)), "cotr_forward: null argument");
    COTR_CHECK(B >= 1 && Q >= 0, "cotr_forward: B must be >= 1 and Q >= 0");
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    cudaStream_t s = (cudaStream_t)cuda_stream;
    CallOrder order(m, s);
    const bool graphable = m->graph_mode && !m->prof_on && Q > 0;
    if (!graphable) return forward_eager(m, img_dev, queries_dev, B, Q, pred_dev, s);
    // graph replay needs fixed addresses: go through the staging buffers (two small device-to-device copies in, one out)
    if (ensure_stage(m, B, Q)) return 1;
    Workspace& w = m->ws;
    const size_t img_bytes = (size_t)B * 3 * COTR_CANVAS_H * COTR_CANVAS_W * sizeof(float), q_bytes = (size_t)B * Q * 2 * sizeof(float);
    COTR_CHECK_CUDA(cudaMemcpyAsync(w.img_stage, img_dev, img_bytes, cudaMemcpyDeviceToDevice, s));
    COTR_CHECK_CUDA(cudaMemcpyAsync(w.q_stage, queries_dev, q_bytes, cudaMemcpyDeviceToDevice, s));
    if (forward_staged(m, B, Q, s)) return 1;
    COTR_CHECK_CUDA(cudaMemcpyAsync(pred_dev, w.pred_stage, q_bytes, cudaMemcpyDeviceToDevice, s));
    return 0;
}

int cotr_forward_host(cotr_model* m, const float* img_host, const float* queries_host, int B, int Q, float* pred_host) {
    COTR_CHECK(m && img_host && (Q == 0 || (queries_host && pred_host)), "cotr_forward_host: null argument");
    COTR_CHECK(B >= 1 && Q >= 0, "cotr_forward_host: B must be >= 1 and Q >= 0");
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    if (ensure_stage(m, B, Q)) return 1;
    Workspace& w = m->ws;
    const size_t img_bytes = (size_t)B * 3 * COTR_CANVAS_H * COTR_CANVAS_W * sizeof(float), q_bytes = (size_t)B * Q * 2 * sizeof(float);
    cudaStream_t s = m->host_stream;
    CallOrder order(m, s);
    COTR_CHECK_CUDA(cudaMemcpyAsync(w.img_stage, img_host, img_bytes, cudaMemcpyHostToDevice, s));
    if (q_bytes) COTR_CHECK_CUDA(cudaMemcpyAsync(w.q_stage, queries_host, q_bytes, cudaMemcpyHostToDevice, s));
    if (Q > 0) {
        if (forward_staged(m, B, Q, s)) return 1;
        COTR_CHECK_CUDA(cudaMemcpyAsync(pred_host, w.pred_stage, q_bytes, cudaMemcpyDeviceToHost, s));
    }
    COTR_CHECK_CUDA(cudaStreamSynchronize(s));
    return 0;
}

int cotr_preprocess(cotr_model* m, const uint8_t* img_from_dev, int h_from, int w_from, const uint8_t* img_to_dev, int h_to,
                    int w_to, const int32_t* rects_host, int n, float* canvas_dev, void* cuda_stream) {
    COTR_CHECK(m != nullptr, "cotr_preprocess: null model");
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    if (!m->pre) m->pre = preprocessor_create();
    CallOrder order(m, (cudaStream_t)cuda_stream);
    return preprocess_launch(m->pre, img_from_dev, h_from, w_from, img_to_dev, h_to, w_to, rects_host, n, canvas_dev,
                             (cudaStream_t)cuda_stream);
}

int cotr_refine(cotr_model* m, const uint8_t* const* images_host, const int32_t* hw_host, int n_images,
                const cotr_refine_group* groups_host, int n_groups, const double* zoom_host, int n_zoom, int batch, int wave,
                int64_t max_good, double rel_threshold, const double* loc_from_dev, const double* loc_to_dev,
                double* history_dev, int32_t* rects_dev, int32_t* good_dev, int64_t* walked_host, int32_t* status_host,
                void* cuda_stream) {
    const char* fn = "cotr_refine";
    COTR_CHECK(m != nullptr, "%s: null model", fn);
    COTR_CHECK(walked_host && status_host, "%s: null walked_host or status_host", fn);
    COTR_CHECK(images_host && hw_host && groups_host && zoom_host, "%s: null images_host, hw_host, groups_host or zoom_host", fn);
    COTR_CHECK(n_images >= 1 && n_groups >= 1, "%s: n_images (%d) and n_groups (%d) must be >= 1", fn, n_images, n_groups);
    COTR_CHECK(n_zoom >= 1 && n_zoom <= 7, "%s: %d zoom levels (1 .. 7: conclude() sums the history sequentially)", fn, n_zoom);
    COTR_CHECK(batch >= 1 && wave >= 1, "%s: batch (%d) and wave (%d) must be >= 1", fn, batch, wave);
    for (int i = 0; i < n_images; ++i) {
        COTR_CHECK(images_host[i] != nullptr, "%s: image %d is null", fn, i);
        COTR_CHECK(hw_host[2 * i] >= 2 && hw_host[2 * i + 1] >= 2, "%s: image %d is %d x %d", fn, i, hw_host[2 * i], hw_host[2 * i + 1]);
    }
    int64_t n = 0;
    std::vector<int> sizes((size_t)n_groups * n_zoom * 2);
    for (int g = 0; g < n_groups; ++g) {
        const cotr_refine_group& G = groups_host[g];
        COTR_CHECK(G.image_from >= 0 && G.image_from < n_images && G.image_to >= 0 && G.image_to < n_images,
                   "%s: group %d images (%d, %d) outside [0, %d)", fn, g, G.image_from, G.image_to, n_images);
        COTR_CHECK(G.count >= 1 && G.first == n, "%s: group %d (first %d, count %d): groups must be non-empty and consecutive from task 0",
                   fn, g, G.first, G.count);
        n += G.count;
        COTR_CHECK(n <= INT32_MAX, "%s: more than %d tasks", fn, INT32_MAX);
        char where[48];
        snprintf(where, sizeof(where), "%s: group %d", fn, g);
        const int a = G.image_from, b = G.image_to;
        for (int l = 0; l < n_zoom; ++l)
            if (refine_crop_sides(where, l, zoom_host[l], hw_host[2 * a], hw_host[2 * a + 1], G.s_from, hw_host[2 * b], hw_host[2 * b + 1],
                                  G.s_to, &sizes[((size_t)g * n_zoom + l) * 2])) return 1;
    }
    COTR_CHECK(loc_from_dev && loc_to_dev && history_dev && rects_dev && good_dev, "%s: null device buffer", fn);
    COTR_CHECK(((uintptr_t)loc_from_dev & 7) == 0 && ((uintptr_t)loc_to_dev & 7) == 0 && ((uintptr_t)history_dev & 7) == 0,
               "%s: loc_from_dev, loc_to_dev or history_dev is not 8-byte aligned", fn);
    COTR_CHECK(((uintptr_t)rects_dev & 3) == 0 && ((uintptr_t)good_dev & 3) == 0, "%s: rects_dev or good_dev is not 4-byte aligned", fn);
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    cudaStream_t s = (cudaStream_t)cuda_stream;
    CallOrder order(m, s);
    return refine_walk_impl(m, images_host, hw_host, groups_host, n_groups, sizes, n_zoom, batch, wave, max_good, rel_threshold,
                            loc_from_dev, loc_to_dev, history_dev, rects_dev, good_dev, walked_host, status_host, s);
}

int cotr_refine_grouped(cotr_model* m, const uint8_t* img_from_dev, int h_from, int w_from, const uint8_t* img_to_dev, int h_to,
                        int w_to, double s_from, double s_to, const double* zoom_host, int n_zoom, int level, const int32_t* ids_host,
                        int n_ids, int n_tasks, int batch_size, int max_load, int64_t max_good, double rel_threshold,
                        const double* loc_from_dev, double* history_dev, int32_t* rects_dev, int32_t* good_dev, int32_t* squad_host,
                        int32_t* result_host, void* cuda_stream) {
    const char* fn = "cotr_refine_grouped";
    COTR_CHECK(m != nullptr, "%s: null model", fn);
    COTR_CHECK(result_host && zoom_host, "%s: null result_host or zoom_host", fn);
    COTR_CHECK(img_from_dev && img_to_dev, "%s: null image", fn);
    COTR_CHECK(h_from >= 2 && w_from >= 2 && h_to >= 2 && w_to >= 2, "%s: images %d x %d and %d x %d", fn, h_from, w_from, h_to, w_to);
    COTR_CHECK(n_zoom >= 1 && n_zoom <= 7, "%s: %d zoom levels (1 .. 7: conclude() sums the history sequentially)", fn, n_zoom);
    COTR_CHECK(level >= 0 && level < n_zoom, "%s: level %d of %d", fn, level, n_zoom);
    COTR_CHECK(batch_size >= 1 && max_load >= 0, "%s: batch_size (%d) must be >= 1 and max_load (%d) >= 0", fn, batch_size, max_load);
    COTR_CHECK(n_tasks >= 1 && n_ids >= 0 && n_ids <= n_tasks, "%s: %d candidates of %d tasks", fn, n_ids, n_tasks);
    COTR_CHECK(n_ids == 0 || (ids_host && squad_host), "%s: null ids_host or squad_host", fn);
    std::vector<char> seen((size_t)n_tasks, 0);
    for (int i = 0; i < n_ids; ++i) {
        const int32_t t = ids_host[i];
        COTR_CHECK(t >= 0 && t < n_tasks && !seen[t], "%s: candidate %d is task %d (outside [0, %d) or repeated)", fn, i, t, n_tasks);
        seen[t] = 1;
    }
    int sizes[2];
    if (refine_crop_sides(fn, level, zoom_host[level], h_from, w_from, s_from, h_to, w_to, s_to, sizes)) return 1;
    COTR_CHECK(loc_from_dev && history_dev && rects_dev && good_dev, "%s: null device buffer", fn);
    COTR_CHECK(((uintptr_t)loc_from_dev & 7) == 0 && ((uintptr_t)history_dev & 7) == 0, "%s: loc_from_dev or history_dev is not 8-byte aligned", fn);
    COTR_CHECK(((uintptr_t)rects_dev & 3) == 0 && ((uintptr_t)good_dev & 3) == 0, "%s: rects_dev or good_dev is not 4-byte aligned", fn);
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    cudaStream_t s = (cudaStream_t)cuda_stream;
    CallOrder order(m, s);
    return refine_grouped_impl(m, img_from_dev, h_from, w_from, img_to_dev, h_to, w_to, sizes[0], sizes[1], level, n_zoom, ids_host, n_ids,
                               n_tasks, batch_size, max_load, max_good, rel_threshold, loc_from_dev, history_dev, rects_dev, good_dev,
                               squad_host, result_host, s);
}

int cotr_test_pilot_boxes(int device, const double* pts_host, int n, const int32_t* geom_host, double* box_host, int32_t* fail_host) {
    const char* fn = "cotr_test_pilot_boxes";
    COTR_CHECK(n >= 1 && pts_host && geom_host && box_host && fail_host, "%s: bad arguments", fn);
    const int32_t* g = geom_host;
    COTR_CHECK(g[4] >= 2 && g[4] <= g[0] && g[4] <= g[1] && g[5] >= 2 && g[5] <= g[2] && g[5] <= g[3], "%s: bad geometry", fn);
    COTR_CHECK_CUDA(cudaSetDevice(device));
    // the launch reads candidate i as task i at level 0 of a one-level walk: loc_from (n,2), history (n,2,2) row 0
    std::vector<double> lf((size_t)n * 2), hist((size_t)n * 4, 0.0);
    std::vector<int32_t> ids((size_t)n);
    for (int i = 0; i < n; ++i) {
        lf[2 * i] = pts_host[4 * i]; lf[2 * i + 1] = pts_host[4 * i + 1];
        hist[4 * i] = pts_host[4 * i + 2]; hist[4 * i + 1] = pts_host[4 * i + 3];
        ids[i] = i;
    }
    DevAllocs d;
    void *lf_dev, *hist_dev, *ids_dev, *pts_dev, *box_dev, *fail_dev;
    if (d.upload(&lf_dev, lf.data(), lf.size() * sizeof(double)) || d.upload(&hist_dev, hist.data(), hist.size() * sizeof(double)) ||
        d.upload(&ids_dev, ids.data(), ids.size() * sizeof(int32_t)) || d.alloc(&pts_dev, (size_t)n * 4 * sizeof(double)) ||
        d.alloc(&box_dev, (size_t)n * 8 * sizeof(double)) || d.alloc(&fail_dev, (size_t)n * sizeof(int32_t)))
        return 1;
    RefineLevel lv = RefineLevel();
    lv.count = n; lv.level = 0; lv.levels = 1;
    lv.h_from = g[0]; lv.w_from = g[1]; lv.h_to = g[2]; lv.w_to = g[3];
    lv.from.size = g[4]; lv.to.size = g[5];
    if (launch_grouped_candidates(lv, (const int32_t*)ids_dev, (const double*)lf_dev, (const double*)hist_dev, (double*)pts_dev,
                                  (double*)box_dev, (int32_t*)fail_dev, 0)) return 1;
    COTR_CHECK_CUDA(cudaMemcpy(box_host, box_dev, (size_t)n * 8 * sizeof(double), cudaMemcpyDeviceToHost));
    COTR_CHECK_CUDA(cudaMemcpy(fail_host, fail_dev, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return 0;
}

int cotr_dense_postprocess(cotr_model* m, const float* pred_dev, int n, float* out_dev, void* cuda_stream) {
    COTR_CHECK(m != nullptr, "cotr_dense_postprocess: null model");
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    return dense_post_launch(pred_dev, out_dev, n, (cudaStream_t)cuda_stream);
}

int cotr_flow_tile_merge(cotr_model* m, const float* tile_dev, int pitch_floats, const double* affine_host, int px, int py, int pw, int ph,
                         int ow, int oh, float* flow_dev, float* conf_dev, int first, void* cuda_stream) {
    COTR_CHECK(m != nullptr, "cotr_flow_tile_merge: null model");
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    if (!m->merger) m->merger = flow_merger_create();
    CallOrder order(m, (cudaStream_t)cuda_stream);
    return flow_tile_merge_launch(m->merger, tile_dev, pitch_floats, affine_host, px, py, pw, ph, ow, oh, flow_dev, conf_dev, first,
                                  (cudaStream_t)cuda_stream);
}

// cotr_resize_image and cotr_resize_maps: every argument checked, then at most two passes (or one copy) on the stream.
static int resize_impl(cotr_model* m, const char* fn, int u8, const void* src, int h, int w, int c, void* dst, int out_h, int out_w,
                       void* cuda_stream) {
    COTR_CHECK(m != nullptr, "%s: null model", fn);
    COTR_CHECK(src && dst, "%s: null src_dev or dst_dev", fn);
    COTR_CHECK(h >= 1 && w >= 1 && out_h >= 1 && out_w >= 1 && h <= 65536 && w <= 65536 && out_h <= 65536 && out_w <= 65536,
               "%s: sizes %d x %d -> %d x %d must lie in 1 .. 65536", fn, h, w, out_h, out_w);
    COTR_CHECK(c >= 1 && c <= 3, "%s: %d channels (1 .. 3)", fn, c);
    const size_t elem = u8 ? 1 : sizeof(float);
    COTR_CHECK(u8 || (((uintptr_t)src & 3) == 0 && ((uintptr_t)dst & 3) == 0), "%s: src_dev or dst_dev is not 4-byte aligned", fn);
    const uintptr_t s0 = (uintptr_t)src, s1 = s0 + (size_t)h * w * c * elem, d0 = (uintptr_t)dst, d1 = d0 + (size_t)out_h * out_w * c * elem;
    COTR_CHECK(d1 <= s0 || s1 <= d0, "%s: src_dev and dst_dev overlap", fn);
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    if (!m->resizer) m->resizer = resizer_create();
    cudaStream_t s = (cudaStream_t)cuda_stream;
    ResizePlan p;
    if (resize_plan(m->resizer, u8, h, w, c, out_h, out_w, &p)) return 1;
    CallOrder order(m, s);
    const Run r{m, s};
    const int kernel = u8 ? K_RESIZE_IMAGE : K_RESIZE_MAPS;
    if (!p.need_h && !p.need_v) {
        COTR_CHECK_CUDA(cudaMemcpyAsync(dst, src, (size_t)h * w * c * elem, cudaMemcpyDeviceToDevice, s));
        return 0;
    }
    if (p.need_h) {
        LaunchScope ls(r, kernel, h, out_w, 0);
        if (resize_pass(p, 0, src, p.need_v ? p.tmp : dst, s)) return 1;
    }
    if (p.need_v) {
        LaunchScope ls(r, kernel, out_h, out_w, 1);
        if (resize_pass(p, 1, p.need_h ? p.tmp : src, dst, s)) return 1;
    }
    return 0;
}

int cotr_resize_image(cotr_model* m, const uint8_t* src_dev, int h, int w, uint8_t* dst_dev, int out_h, int out_w, void* cuda_stream) {
    return resize_impl(m, "cotr_resize_image", 1, src_dev, h, w, 3, dst_dev, out_h, out_w, cuda_stream);
}

int cotr_resize_maps(cotr_model* m, const float* src_dev, int h, int w, int c, float* dst_dev, int out_h, int out_w, void* cuda_stream) {
    return resize_impl(m, "cotr_resize_maps", 0, src_dev, h, w, c, dst_dev, out_h, out_w, cuda_stream);
}

int cotr_group_tasks(int device, const double* pts_dev, const double* box_dev, int n, int batch_size, int max_load, int32_t* squad_dev,
                     int32_t* rank_dev, int32_t* n_squads_dev, void* cuda_stream) {
    COTR_CHECK_CUDA(cudaSetDevice(device));
    return group_tasks_launch(pts_dev, box_dev, n, batch_size, max_load, squad_dev, rank_dev, n_squads_dev, (cudaStream_t)cuda_stream);
}

int cotr_mutual_nearest(int device, const double* kpts_dev, const int64_t* kpt_offsets_host, int n_images, const int32_t* pairs_host,
                        int B, const double* corr_dev, int32_t* nearest_dev, int32_t* match_dev, int32_t* count_dev, void* cuda_stream) {
    const char* fn = "cotr_mutual_nearest";
    MatchPlan plan;
    if (plan_match(fn, kpt_offsets_host, n_images, pairs_host, B, nullptr, &plan)) return 1;
    if (check_match_outputs(fn, plan.rows, kpts_dev, corr_dev, nearest_dev, match_dev, count_dev)) return 1;
    COTR_CHECK_CUDA(cudaSetDevice(device));
    cudaStream_t s = (cudaStream_t)cuda_stream;
    // No model, so no persistent staging: the tables live in stream-ordered memory for the duration of the call, copied
    // from pageable host memory (the runtime may wait for the stream to stage that copy; see the header).
    const size_t bytes = plan.tab.size() * sizeof(int4);
    int4* tab = nullptr;
    COTR_CHECK_CUDA(cudaMallocAsync((void**)&tab, bytes, s));
    int rc = 0;
    const cudaError_t e = cudaMemcpyAsync(tab, plan.tab.data(), bytes, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) { set_error("%s: table upload failed: %s", fn, cudaGetErrorString(e)); rc = 1; }
    if (!rc) rc = launch_nearest(reinterpret_cast<const MatchTile*>(tab), plan.n_tiles, kpts_dev, corr_dev, nearest_dev, s);
    if (!rc) rc = launch_mutual(tab + 3 * (size_t)plan.n_tiles, B, nearest_dev, match_dev, count_dev, s);
    cudaFreeAsync(tab, s);
    return rc;
}

int cotr_match_keypoints(cotr_model* m, const void* feat_dev, int n_images, const int32_t* sizes_host, const double* kpts_dev,
                         const int64_t* kpt_offsets_host, const int32_t* pairs_host, int B, cotr_context* ctx, double* corr_dev,
                         int32_t* nearest_dev, int32_t* match_dev, int32_t* count_dev, void* cuda_stream) {
    const char* fn = "cotr_match_keypoints";
    COTR_CHECK(m != nullptr, "%s: null model", fn);
    m->launches = 0;
    COTR_CHECK(feat_dev && sizes_host, "%s: null feat_dev or sizes_host", fn);
    COTR_CHECK(((uintptr_t)feat_dev & 15) == 0, "%s: feat_dev is not 16-byte aligned", fn);
    COTR_CHECK(ctx && ctx->model == m, "%s: context does not belong to this model", fn);
    MatchPlan plan;
    if (plan_match(fn, kpt_offsets_host, n_images, pairs_host, B, sizes_host, &plan)) return 1;
    COTR_CHECK(2 * (int64_t)B <= ctx->max_pairs, "%s: B = %d pairs need %d contexts, the context holds at most %d", fn, B,
               2 * B, ctx->max_pairs);
    if (check_match_outputs(fn, plan.rows, kpts_dev, corr_dev, nearest_dev, match_dev, count_dev)) return 1;
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    cudaStream_t s = (cudaStream_t)cuda_stream;
    CallOrder order(m, s);
    // 1. the contexts [a_p | b_p], [b_p | a_p]
    std::vector<int32_t> ctx_pairs(4 * (size_t)B);
    for (int p = 0; p < B; ++p) {
        ctx_pairs[4 * p] = ctx_pairs[4 * p + 3] = pairs_host[2 * p];
        ctx_pairs[4 * p + 1] = ctx_pairs[4 * p + 2] = pairs_host[2 * p + 1];
    }
    if (encode_pairs_impl(m, feat_dev, n_images, ctx_pairs.data(), 2 * B, ctx, s, AttnMaps())) return 1;
    if (ensure_match_ws(m, plan.rows)) return 1;
    if (m->match_tab.upload(plan.tab.data(), plan.tab.size(), s)) return 1;
    const MatchTile* tiles = reinterpret_cast<const MatchTile*>(m->match_tab.dev);
    const int4* pair_tab = m->match_tab.dev + 3 * (size_t)plan.n_tiles;
    Workspace& w = m->ws;
    Run r{m, s};
    const int R = (int)plan.rows;
    if (R > 0) {
        // 2. - 4. keypoints -> canvas queries -> ragged decode -> pixels of the right image
        {
            LaunchScope scope(r, K_MATCH_QUERIES, R, 2, 0);
            if (launch_match_queries(tiles, plan.n_tiles, kpts_dev, w.match_q, s)) return 1;
        }
        if (decode_ragged_impl(m, ctx, w.match_q, plan.ctx_off.data(), 2 * B, w.match_pred, s)) return 1;
        {
            LaunchScope scope(r, K_MATCH_PIXELS, R, 2, 0);
            if (launch_match_pixels(tiles, plan.n_tiles, w.match_pred, corr_dev, s)) return 1;
        }
        // 5. cotr_mutual_nearest on the same layout
        LaunchScope scope(r, K_NEAREST, R, 2, 0);
        if (launch_nearest(tiles, plan.n_tiles, kpts_dev, corr_dev, nearest_dev, s)) return 1;
    }
    LaunchScope scope(r, K_MUTUAL, B, 0, 0);
    return launch_mutual(pair_tab, B, nearest_dev, match_dev, count_dev, s);
}

int cotr_rasterize_triangles(int device, const float* tris_dev, int n_tri, int H, int W, float* out_dev, void* cuda_stream) {
    COTR_CHECK_CUDA(cudaSetDevice(device));
    return rasterize_triangles_launch(tris_dev, n_tri, H, W, out_dev, (cudaStream_t)cuda_stream);
}

int cotr_set_graph_mode(cotr_model* m, int enabled) {
    COTR_CHECK(m != nullptr, "cotr_set_graph_mode: null model");
    m->graph_mode = enabled != 0;
    return 0;
}

size_t cotr_workspace_bytes(int B, int Q) {
    if (B < 1 || Q < 0) return 0;
    const long long total = (long long)B * Q;
    const int rows = (int)(total < kDecodeChunkRows ? total : kDecodeChunkRows);
    Workspace w;
    return ws_bytes(encode_ws_bufs(w, B)) + ws_bytes(decode_ws_bufs(w, rows));
}

int cotr_last_launch_count(const cotr_model* m) { return m ? m->launches : -1; }

int cotr_profile_begin(cotr_model* m, int max_records) {
    COTR_CHECK(m && max_records > 0, "cotr_profile_begin: bad arguments");
    m->prof_records.clear();
    m->prof_records.reserve(max_records);
    m->prof_max = max_records;
    m->prof_on = true;
    return 0;
}

int cotr_profile_end(cotr_model* m, cotr_launch_record* out, int max_records) {
    COTR_CHECK(m && out, "cotr_profile_end: bad arguments");
    m->prof_on = false;
    COTR_CHECK_CUDA(cudaSetDevice(m->device));
    COTR_CHECK_CUDA(cudaDeviceSynchronize());
    int n = (int)m->prof_records.size();
    if (n > max_records) n = max_records;
    for (int i = 0; i < n; ++i) {
        float ms = 0.f;
        COTR_CHECK_CUDA(cudaEventElapsedTime(&ms, m->prof_events[2 * i], m->prof_events[2 * i + 1]));
        m->prof_records[i].ms = ms;
        out[i] = m->prof_records[i];
    }
    return -n - 1;     // see header: success is encoded as -(count + 1)
}

int64_t cotr_debug_read(cotr_model* m, const char* name, float* out_host, int64_t max_elems) {
    if (!m || !name || !out_host) return -1;
    cudaSetDevice(m->device);
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    CSplit16 src{nullptr, nullptr};
    const float* src_f32 = nullptr;
    int64_t n = 0;
    const std::string s(name);
    if (s == "feat") { src = cs(m->last_feat); n = (int64_t)m->last_pairs * 2 * 16 * 16 * 1024; }
    else if (s == "src") { src = cs(m->ws.src); n = (int64_t)m->last_pairs * kTokens * kDModel; }
    else if (s == "mem") { src = cs(m->last_mem); n = (int64_t)m->last_pairs * kTokens * kDModel; }
    TmpSplit mem_ln;
    if (s == "mem" && m->last_mem_pre_ln && src.hi && n > 0) {
        // tensor-core path: the encoder output exists only before its last (deferred) LayerNorm - apply it here
        const EncLayer& e = m->enc[kEncLayers - 1];
        if (ws_alloc(&mem_ln.t, (size_t)n) || launch_layernorm(src, e.ln2_g, e.ln2_b, mem_ln.t, (int)(n / kDModel), 0) ||
            cudaDeviceSynchronize() != cudaSuccess)
            return -1;
        src = cs(mem_ln.t);
    }
    else if (s == "hs") { src = cs(m->ws.hs); n = (int64_t)m->last_rows * kDModel; }
    else if (s == "pos") { src_f32 = m->pos; n = (int64_t)kTokens * kDModel; }
    // bring-up: raw workspace buffers of the last forward (tokens = pairs * 512, rows = the decoder rows of the last chunk)
    else if (s == "ws.xa") { src = cs(m->ws.xa); n = (int64_t)m->last_pairs * kTokens * kDModel; }
    else if (s == "ws.xb") { src = cs(m->ws.xb); n = (int64_t)m->last_pairs * kTokens * kDModel; }
    else if (s == "ws.ao") { src = cs(m->ws.ao); n = (int64_t)m->last_pairs * kTokens * kDModel; }
    else if (s == "ws.qk") { src = cs(m->ws.qk); n = (int64_t)m->last_pairs * kTokens * 2 * kDModel; }
    else if (s == "ws.ffh") { src = cs(m->ws.ffh); n = (int64_t)m->last_pairs * kTokens * kFF; }
    else if (s == "ws.t") { src = cs(m->ws.t); n = (int64_t)m->last_rows * kDModel; }
    else if (s == "ws.t2") { src = cs(m->ws.t2); n = (int64_t)m->last_rows * kDModel; }
    else if (s == "ws.dao") { src = cs(m->ws.dao); n = (int64_t)m->last_rows * kDModel; }
    else if (s == "ws.st_a") { src_f32 = reinterpret_cast<const float*>(m->ws.enc_st_a); n = (int64_t)m->last_pairs * kTokens * 32; }
    else if (s == "ws.st_b") { src_f32 = reinterpret_cast<const float*>(m->ws.enc_st_b); n = (int64_t)m->last_pairs * kTokens * 32; }
    if ((!src.hi && !src_f32) || n <= 0 || n > max_elems) return -1;
    float* tmp = nullptr;
    if (!src_f32) {
        if (cudaMalloc((void**)&tmp, n * sizeof(float)) != cudaSuccess) return -1;
        if (launch_split16_to_f32(src, tmp, (size_t)n, 0) || cudaDeviceSynchronize() != cudaSuccess) { cudaFree(tmp); return -1; }
        src_f32 = tmp;
    }
    const cudaError_t e = cudaMemcpy(out_host, src_f32, n * sizeof(float), cudaMemcpyDeviceToHost);
    if (tmp) cudaFree(tmp);
    return e == cudaSuccess ? n : -1;
}

int cotr_set_gemm_path(cotr_model* m, int path) {
    COTR_CHECK(m && (path == 0 || path == 1), "cotr_set_gemm_path: path must be 0 (tensor cores) or 1 (fp32 SIMT)");
    if (m->gemm_path != path) {          // captured graphs embed the kernels of the old path
        cudaSetDevice(m->device);
        cudaDeviceSynchronize();
        drop_graphs(m);
        m->shapes_seen.clear();
    }
    m->gemm_path = path;
    return 0;
}

void cotr_debug_set_variant(int variant) { g_tc_variant = variant; g_use_pdl = (variant & 256) ? 0 : 1; }

// ---- kernel-level test hooks: fp32 device tensors in / out, converted to split16 around the kernel under test -------
namespace {
// tensor-core image of a host [N,K] weight, as the model uploads it; returns acc_scale in *scale
int upload_tc_weight(DevAllocs& mem, const float* w_host, int N, int K, void** wtc, float* scale) {
    std::vector<uint8_t> img(tc_weight_bytes(N, K));
    *scale = tc_pack_weight(w_host, N, K, img.data());
    return mem.upload(wtc, img.data(), img.size());
}

std::vector<float> identity(int n) {
    std::vector<float> eye((size_t)n * n, 0.f);
    for (int i = 0; i < n; ++i) eye[(size_t)i * n + i] = 1.f;
    return eye;
}

// Writes the keys and values (kv: [rows][512] = [K | V]) of every pair into slot `slot` of the `slots` attention
// operand images per pair at img, by the same epilogue store as the model's projections: a tensor-core GEMM with the
// identity as its weight.
int write_operand_images(DevAllocs& mem, CSplit16 kv, int rows, int slot, int slots, unsigned char* img) {
    const int n = 2 * kDModel;
    const std::vector<float> eye = identity(n);
    void* wtc = nullptr;
    float scale = 1.f;
    if (upload_tc_weight(mem, eye.data(), n, n, &wtc, &scale)) return 1;
    GemmParams p = gemm_base(rows, n, n, kv, n, nullptr, wtc, scale, kNoSplit, n);
    p.remap = 1; p.blk_map[0] = -1000 - slot; p.blk_map[1] = -(slot + 1); p.n_vt = slots; p.kv_img = img;
    return launch_gemm_tc(p, 0);
}
}  // namespace

int cotr_test_gemm(cotr_test_gemm_desc* d, const float* A_dev, const float* w_host, const float* bias_dev,
                   const float* addmat_dev, const float* residual_dev, const float* ln_gamma_dev,
                   const float* ln_beta_dev, float* out_dev, float* part_out_dev, const int32_t* pairs_host, float* vt_dev,
                   unsigned char* img_dev) {
    COTR_CHECK(d && A_dev && w_host && out_dev, "cotr_test_gemm: null argument");
    COTR_CHECK(d->path == 0 || d->path == 1, "cotr_test_gemm: path %d (0 tensor cores, 1 fp32 SIMT)", d->path);
    COTR_CHECK(d->M >= 1 && d->N >= 1 && d->K >= 1, "cotr_test_gemm: empty problem %d x %d x %d", d->M, d->N, d->K);
    const bool f32_out = (d->N & 15) != 0;
    const int out_rows = d->out_rows > 0 ? d->out_rows : d->M;
    COTR_CHECK(out_rows >= d->M, "cotr_test_gemm: out has %d rows, the launch writes %d", out_rows, d->M);
    COTR_CHECK((d->redirect || d->ldc >= d->N) && (f32_out || d->ldc % 8 == 0),
               "cotr_test_gemm: ldc %d (>= N = %d without a redirect, a multiple of 8)", d->ldc, d->N);
    if (d->a_mode == A_ROWMAJOR || d->a_mode == A_TOKENS)
        COTR_CHECK(d->lda >= d->K, "cotr_test_gemm: lda %d < K %d", d->lda, d->K);
    if (d->a_mode == A_ROWMAJOR)
        COTR_CHECK(d->a_elems >= (int64_t)d->M * d->lda, "cotr_test_gemm: A holds %lld elements, %d rows of lda %d need more",
                   (long long)d->a_elems, d->M, d->lda);
    if (d->a_mode == A_CONV_NHWC)
        COTR_CHECK(d->OH > 0 && d->OW > 0 && d->M % (d->OH * d->OW) == 0 &&
                   d->a_elems >= (int64_t)(d->M / (d->OH * d->OW)) * d->H * d->W * d->C,
                   "cotr_test_gemm: A holds %lld elements, too few for %d x %d x %d images", (long long)d->a_elems, d->H, d->W, d->C);
    std::vector<int> pair_tab;
    if (d->a_mode == A_TOKENS) {
        // pair p = images (pairs_host[2p], pairs_host[2p+1]) of the (n_images,16,16,lda) features in A
        COTR_CHECK(d->M % kTokens == 0 && d->n_pairs == d->M / kTokens && pairs_host != nullptr,
                   "cotr_test_gemm: the token gather needs M = 512 x n_pairs and a pair table (M %d, n_pairs %d)", d->M, d->n_pairs);
        COTR_CHECK(d->n_images >= 1 && d->a_elems >= (int64_t)d->n_images * 256 * d->lda,
                   "cotr_test_gemm: A holds %lld elements, too few for %d images of 256 x %d", (long long)d->a_elems, d->n_images, d->lda);
        pair_tab.assign(pairs_host, pairs_host + 2 * (size_t)d->n_pairs);
        for (size_t i = 0; i < pair_tab.size(); ++i)
            COTR_CHECK(pair_tab[i] >= 0 && pair_tab[i] < d->n_images, "cotr_test_gemm: pair %d reads image %d of %d",
                       (int)(i / 2), pair_tab[i], d->n_images);
    }
    const int res_rows = d->res_rows > 0 ? d->res_rows : d->M;
    if (residual_dev)
        COTR_CHECK(res_rows >= d->M && d->res_col0 >= 0 && d->res_col0 % 16 == 0 && (int64_t)d->res_col0 + d->N <= d->ldr,
                   "cotr_test_gemm: residual columns %d .. %d of ldr %d (res_col0 a multiple of 16), %d rows for M = %d",
                   d->res_col0, d->res_col0 + d->N - 1, d->ldr, res_rows, d->M);
    COTR_CHECK(d->redirect >= 0 && d->redirect <= 2, "cotr_test_gemm: redirect %d (0 none, 1 transposed values, 2 operand images)", d->redirect);
    if (d->redirect) {
        COTR_CHECK(!f32_out && d->N % kDModel == 0 && d->N / kDModel <= 12, "cotr_test_gemm: block redirect needs N a multiple of 256 up to 3072 (N %d)", d->N);
        COTR_CHECK(d->n_vt >= 1 && d->vt_pairs >= (d->M + kTokens - 1) / kTokens, "cotr_test_gemm: %d slots of %d pairs for M = %d",
                   d->n_vt, d->vt_pairs, d->M);
        COTR_CHECK(d->redirect == 1 ? vt_dev != nullptr : (img_dev != nullptr && d->path == 0),
                   "cotr_test_gemm: redirect %d needs %s", d->redirect, d->redirect == 1 ? "vt" : "the image buffer and path 0");
        for (int b = 0; b < d->N / kDModel; ++b) {
            const int m = d->blk_map[b];
            const bool ok = m >= 0 ? (m % 8 == 0 && (int64_t)m + kDModel <= d->ldc)
                                   : ((m >= -d->n_vt) || (d->redirect == 2 && m <= -1000 && m > -1000 - d->n_vt));
            COTR_CHECK(ok, "cotr_test_gemm: blk_map[%d] = %d (ldc %d, %d slots)", b, m, d->ldc, d->n_vt);
        }
    } else {
        COTR_CHECK(vt_dev == nullptr && img_dev == nullptr, "cotr_test_gemm: vt / images without a redirect");
    }
    COTR_CHECK(d->force_bn == 0 || d->path == 0, "cotr_test_gemm: a forced plan needs path 0");
    COTR_CHECK(d->force_ksplit == 0 || d->path == 0, "cotr_test_gemm: a forced plan needs path 0");

    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.M = d->M; p.N = d->N; p.K = d->K;
    p.a_mode = d->a_mode; p.lda = d->lda;
    p.H = d->H; p.W = d->W; p.C = d->C; p.OH = d->OH; p.OW = d->OW;
    p.KH = d->KH; p.KW = d->KW; p.stride = d->stride; p.pad = d->pad;
    p.bias = bias_dev; p.addmat = addmat_dev; p.add_period = d->add_period > 0 ? d->add_period : 1; p.ld_add = d->ld_add;
    p.ldr = d->ldr; p.relu = d->relu;
    const bool dln = d->a_ln != 0 || d->res_ln != 0;
    COTR_CHECK(!dln || (d->path == 0 && ln_gamma_dev && ln_beta_dev), "cotr_test_gemm: deferred LayerNorm needs path 0 and gamma / beta");
    const bool out_ln = !dln && ln_gamma_dev != nullptr;
    COTR_CHECK(!out_ln || (d->N == kDModel && d->ldc == kDModel && !d->redirect), "cotr_test_gemm: the LayerNorm epilogue needs N = ldc = 256");
    if (!dln) { p.ln_gamma = ln_gamma_dev; p.ln_beta = ln_beta_dev; }
    p.ldc = d->ldc;
    DevAllocs mem;
    TmpSplit a16, res16, out16, vt16;
    int K = d->K;
    std::vector<float> w_stem;
    if (d->a_mode == A_STEM_NHWC4) {
        // the stem as the model runs it: A_dev is the fp32 (B,3,256,512) canvas, w_host [N][7][7][3]; the hook builds the
        // bordered NHWC4 operand and the matching weight order (K = 224)
        COTR_CHECK(d->K == 147 && d->OH == 128 && d->OW == 128 && d->M % (128 * 128) == 0, "cotr_test_gemm: the stem mode expects K = 147, 128 x 128 outputs per image");
        const int n_img = d->M / (128 * 128);
        if (a16.empty((size_t)n_img * kStemCanvasElems)) return 1;
        COTR_CHECK_CUDA(cudaMemset(a16.t.hi, 0, (size_t)n_img * kStemCanvasElems * 2 * sizeof(__half)));
        if (launch_stem_canvas(A_dev, true, a16.t, n_img, 0)) return 1;
        p.a = cs(a16.t);
        w_stem = stem_weight_order(std::vector<float>(w_host, w_host + (size_t)d->N * 147), d->N);
        w_host = w_stem.data();
        K = kStemK; p.K = K; p.KW = 8; p.C = 4;
    } else {
        COTR_CHECK(d->a_elems > 0, "cotr_test_gemm: a_elems missing");
        if (a16.from_f32(A_dev, (size_t)d->a_elems)) return 1;      // the whole buffer: NaN in its padding reaches the kernel
        p.a = cs(a16.t);
    }
    if (d->a_mode == A_TOKENS) {
        int* pair_id = nullptr;
        if (mem.upload((void**)&pair_id, pair_tab.data(), pair_tab.size() * sizeof(int))) return 1;
        p.a_pairs = pair_id;
    }
    if (residual_dev) {
        if (res16.from_f32(residual_dev, (size_t)res_rows * d->ldr)) return 1;
        p.res = offset(cs(res16.t), (size_t)d->res_col0);
    }
    // the output buffers are converted in, so everything the launch does not write comes back as it was passed
    const size_t out_elems = (size_t)out_rows * d->ldc;
    const size_t vt_elems = d->redirect == 1 ? (size_t)d->vt_pairs * d->n_vt * kVtLayer : 0;
    if (f32_out) p.out_f32 = out_dev;
    else { if (out16.from_f32(out_dev, out_elems)) return 1; p.out = out16.t; }
    if (d->redirect) {
        p.remap = 1;
        memcpy(p.blk_map, d->blk_map, sizeof(p.blk_map));
        p.n_vt = d->n_vt;
        if (d->redirect == 1) { if (vt16.from_f32(vt_dev, vt_elems)) return 1; p.vt = vt16.t; }
        else p.kv_img = img_dev;
    }
    float* wd = nullptr;
    if (mem.upload((void**)&wd, w_host, (size_t)d->N * K * sizeof(float))) return 1;
    p.Wt = wd;
    // deferred LayerNorm of A: the packed weights carry gamma, column sums and beta W^T + bias go to the epilogue
    LnFold fold;
    if (d->a_ln) {
        COTR_CHECK(d->K == 256 && d->a_mode == A_ROWMAJOR, "cotr_test_gemm: a_ln needs K = 256, row-major A");
        std::vector<float> g(d->K), be(d->K), bias_h(d->N, 0.f);
        COTR_CHECK_CUDA(cudaMemcpy(g.data(), ln_gamma_dev, d->K * sizeof(float), cudaMemcpyDeviceToHost));
        COTR_CHECK_CUDA(cudaMemcpy(be.data(), ln_beta_dev, d->K * sizeof(float), cudaMemcpyDeviceToHost));
        if (bias_dev) COTR_CHECK_CUDA(cudaMemcpy(bias_h.data(), bias_dev, d->N * sizeof(float), cudaMemcpyDeviceToHost));
        fold = fold_ln(w_host, bias_h.data(), d->N, d->K, g.data(), be.data());
        float *cs_dev = nullptr, *cb_dev = nullptr;
        float2* stats_dev = nullptr;
        if (mem.upload((void**)&cs_dev, fold.cs.data(), d->N * sizeof(float)) ||
            mem.upload((void**)&cb_dev, fold.b.data(), d->N * sizeof(float)) ||
            mem.alloc((void**)&stats_dev, (size_t)d->M * 16 * sizeof(float2)))
            return 1;
        p.a_ln_cs = cs_dev; p.bias = cb_dev;
        w_host = fold.w.data();
        COTR_CHECK(d->lda == kDModel, "cotr_test_gemm: a_ln needs lda = 256");
        if (launch_ln_partials(p.a, stats_dev, d->M, 0)) return 1;
        p.a_ln_part = stats_dev;
    }
    if (d->res_ln) {
        COTR_CHECK(residual_dev && d->ldr == 256 && d->N == 256 && d->res_col0 == 0, "cotr_test_gemm: res_ln needs a [M,256] residual");
        float2* res_stats_dev = nullptr;
        if (mem.alloc((void**)&res_stats_dev, (size_t)d->M * 16 * sizeof(float2))) return 1;
        if (launch_ln_partials(p.res, res_stats_dev, d->M, 0)) return 1;
        p.res_ln_part = res_stats_dev; p.res_ln_gamma = ln_gamma_dev; p.res_ln_beta = ln_beta_dev;
    }
    if (d->emit_part) {
        COTR_CHECK(d->path == 0 && part_out_dev != nullptr && d->N == 256 && d->ldc == 256, "cotr_test_gemm: emit_part needs path 0, N = ldc = 256 and an output buffer");
        p.ln_part_out = reinterpret_cast<float2*>(part_out_dev);
    }
    void* wtc = nullptr;
    if (upload_tc_weight(mem, w_host, d->N, K, &wtc, &p.acc_scale)) return 1;
    p.Wtc = wtc;
    d->plan_bn = d->plan_loader = d->plan_dln = d->plan_ksplit = d->plan_grid_x = d->plan_grid_y = d->plan_ln_defused = 0;
    int rc;
    if (d->path == 0) {
        // the LayerNorm epilogue as run_gemm launches it: fused into the 256-wide tile, or (few rows, or a narrower
        // tile forced) a narrow-tile GEMM followed by the in-place LayerNorm kernel
        const bool defuse = out_ln && (d->force_bn ? d->force_bn != 256 : ln_defused(d->M));
        if (defuse) { p.ln_gamma = nullptr; p.ln_beta = nullptr; }
        GemmPlan plan{};
        rc = launch_gemm_tc_forced(p, d->force_bn, d->force_ksplit, &plan, 0);
        if (!rc && defuse) rc = launch_layernorm(cs(p.out), ln_gamma_dev, ln_beta_dev, p.out, p.M, 0);
        if (!rc) {
            d->plan_bn = plan.bn; d->plan_loader = plan.loader; d->plan_dln = plan.dln; d->plan_ksplit = plan.ksplit;
            d->plan_grid_x = plan.grid_x; d->plan_grid_y = plan.grid_y; d->plan_ln_defused = defuse;
        }
    } else {
        const float* g = p.ln_gamma; const float* b = p.ln_beta;
        p.ln_gamma = nullptr; p.ln_beta = nullptr;
        if (g) {
            float* scratch = nullptr;
            rc = mem.alloc((void**)&scratch, (size_t)d->M * d->N * sizeof(float));
            if (!rc) rc = launch_gemm_simt_raw(p, scratch, 0);
            if (!rc) rc = launch_layernorm_f32(scratch, g, b, p.out, p.M, 0);
        } else {
            rc = launch_gemm_simt(p, 0);
        }
    }
    if (!rc && !f32_out) rc = launch_split16_to_f32(cs(out16.t), out_dev, out_elems, 0);
    if (!rc && d->redirect == 1) rc = launch_split16_to_f32(cs(vt16.t), vt_dev, vt_elems, 0);
    cudaError_t e = cudaDeviceSynchronize();
    if (rc) return rc;
    COTR_CHECK(e == cudaSuccess, "cotr_test_gemm: kernel failed: %s", cudaGetErrorString(e));
    return 0;
}

// The attention launch as the model makes it (see cotr_test_attention_desc).  K / V reach the kernel in the layout of
// the chosen schedule, produced by the same epilogue stores as in the model: V transposed by the fp32 SIMT identity
// GEMM (operands 0), or K and V of the slot as the operand images of one tensor-core identity GEMM over [K | V]
// (operands 1), the other slots' images left 0xFF (fp16 NaN).  `out` is converted in before the launch, so every row
// the launch does not own comes back as it was passed.  With `maps` the maps kernel of the path follows, over the
// AttnParams the attention launch read (as run_attention_weights launches it); it writes fp32 rows straight into maps.
int cotr_test_attention(const cotr_test_attention_desc* d, const float* q_dev, const float* k_dev, const float* v_dev,
                        float* out_dev, const int32_t* tiles_host, float* maps_dev) {
    COTR_CHECK(d && q_dev && k_dev && v_dev && out_dev, "cotr_test_attention: null argument");
    COTR_CHECK(d->path == 0 || d->path == 1, "cotr_test_attention: path %d (0 tensor cores, 1 fp32 SIMT)", d->path);
    COTR_CHECK(d->operands == 0 || d->operands == 1, "cotr_test_attention: operands %d (0 row-major, 1 images)", d->operands);
    COTR_CHECK(d->slots >= 1 && d->slot >= 0 && d->slot < d->slots, "cotr_test_attention: slot %d of %d", d->slot, d->slots);
    COTR_CHECK(d->ctx_pairs >= 1 && d->pair0 >= 0, "cotr_test_attention: pair0 %d of %d pairs", d->pair0, d->ctx_pairs);
    COTR_CHECK(d->q_rows >= 1, "cotr_test_attention: q has %d rows", d->q_rows);
    COTR_CHECK(d->ldq > 0 && d->ldq % 8 == 0, "cotr_test_attention: ldq %d is not a positive multiple of 8", d->ldq);
    COTR_CHECK(d->q_col0 >= 0 && d->q_col0 % 8 == 0 && (int64_t)d->q_col0 + kDModel <= d->ldq,
               "cotr_test_attention: q columns %d .. %d do not fit ldq %d (q_col0 must be a multiple of 8)", d->q_col0,
               d->q_col0 + kDModel - 1, d->ldq);
    COTR_CHECK(d->key_split >= 0 && d->key_split <= 2 && (d->path == 0 || d->key_split == 0),
               "cotr_test_attention: key split %d (0 = launch rule, 1 or 2 on path 0)", d->key_split);
    COTR_CHECK(d->n_tiles >= 0, "cotr_test_attention: n_tiles %d", d->n_tiles);
    std::vector<int4> tiles((size_t)d->n_tiles);
    if (d->n_tiles > 0) {
        COTR_CHECK(tiles_host, "cotr_test_attention: n_tiles %d without a tile table", d->n_tiles);
        const int cap = d->path == 0 ? kAttnTcTileRows : kAttnSimtTileRows;
        for (int i = 0; i < d->n_tiles; ++i) {
            const int pair = tiles_host[3 * i], row0 = tiles_host[3 * i + 1], rows = tiles_host[3 * i + 2];
            COTR_CHECK(rows >= 1 && rows <= cap, "cotr_test_attention: tile %d has %d rows (1 .. %d on path %d)", i, rows, cap, d->path);
            COTR_CHECK(row0 >= 0 && (int64_t)row0 + rows <= d->q_rows, "cotr_test_attention: rows %d .. %d of tile %d fall outside q (%d rows)",
                       row0, row0 + rows - 1, i, d->q_rows);
            COTR_CHECK(pair >= 0 && (int64_t)d->pair0 + pair < d->ctx_pairs, "cotr_test_attention: tile %d reads pair %d + %d of %d",
                       i, d->pair0, pair, d->ctx_pairs);
            tiles[i] = make_int4(pair, row0, rows, 0);
        }
    } else {
        COTR_CHECK(d->nq >= 1 && d->npairs >= 1, "cotr_test_attention: nq %d, npairs %d", d->nq, d->npairs);
        COTR_CHECK((int64_t)d->pair0 + d->npairs <= d->ctx_pairs, "cotr_test_attention: pairs %d .. %d of %d", d->pair0,
                   d->pair0 + d->npairs - 1, d->ctx_pairs);
        COTR_CHECK((int64_t)d->nq * d->npairs <= d->q_rows, "cotr_test_attention: %d x %d rows, q has %d", d->npairs, d->nq, d->q_rows);
    }
    if (maps_dev) {
        COTR_CHECK(d->n_tiles == 0, "cotr_test_attention: maps of a tile-table launch (the model asks maps of uniform launches only)");
        COTR_CHECK(d->path != 0 || d->operands == 1, "cotr_test_attention: tensor-core maps read the keys as operand images (operands 1)");
        COTR_CHECK(d->path != 1 || d->operands == 0, "cotr_test_attention: fp32 SIMT maps read row-major keys (operands 0)");
        COTR_CHECK(d->maps_row0 >= 0 && (int64_t)d->maps_row0 + (int64_t)d->npairs * d->nq <= d->maps_rows,
                   "cotr_test_attention: map rows %d .. %lld do not fit the %d rows of maps", d->maps_row0,
                   (long long)d->maps_row0 + (int64_t)d->npairs * d->nq - 1, d->maps_rows);
    }

    DevAllocs mem;
    TmpSplit q16, o16, k16, v16, vt16, kv16;
    const size_t kv_rows = (size_t)d->ctx_pairs * kTokens, kv_ld = (size_t)d->slots * kDModel;
    if (q16.from_f32(q_dev, (size_t)d->q_rows * d->ldq) || o16.from_f32(out_dev, (size_t)d->q_rows * kDModel)) return 1;
    AttnParams a{};
    a.q = offset(cs(q16.t), (size_t)d->q_col0); a.ldq = d->ldq;
    a.out = o16.t; a.ldo = kDModel;
    a.nq = d->nq; a.npairs = d->npairs; a.pair0 = d->pair0;
    if (d->operands == 1) {
        float* kv = nullptr;
        unsigned char* img = nullptr;
        const size_t img_bytes = (size_t)d->ctx_pairs * d->slots * kHeads * kAttnHeadImgBytes;
        if (mem.alloc((void**)&kv, kv_rows * 2 * kDModel * sizeof(float)) || mem.alloc((void**)&img, img_bytes)) return 1;
        COTR_CHECK_CUDA(cudaMemcpy2D(kv, 2 * kDModel * sizeof(float), k_dev + (size_t)d->slot * kDModel, kv_ld * sizeof(float),
                                     kDModel * sizeof(float), kv_rows, cudaMemcpyDeviceToDevice));
        COTR_CHECK_CUDA(cudaMemcpy2D(kv + kDModel, 2 * kDModel * sizeof(float), v_dev + (size_t)d->slot * kDModel, kv_ld * sizeof(float),
                                     kDModel * sizeof(float), kv_rows, cudaMemcpyDeviceToDevice));
        COTR_CHECK_CUDA(cudaMemset(img, 0xFF, img_bytes));
        if (kv16.from_f32(kv, kv_rows * 2 * kDModel) ||
            write_operand_images(mem, cs(kv16.t), (int)kv_rows, d->slot, d->slots, img)) return 1;
        a.kv_img = img + (size_t)d->slot * kHeads * kAttnHeadImgBytes;
        a.img_pair_stride = (size_t)d->slots * kHeads * kAttnHeadImgBytes;
    } else {
        float* wd = nullptr;
        const std::vector<float> eye = identity(kDModel);
        if (k16.from_f32(k_dev, kv_rows * kv_ld) || v16.from_f32(v_dev, kv_rows * kv_ld) || vt16.empty(kv_rows * kv_ld) ||
            mem.upload((void**)&wd, eye.data(), eye.size() * sizeof(float))) return 1;
        COTR_CHECK_CUDA(cudaMemset(vt16.t.hi, 0xFF, (size_t)(vt16.t.lo - vt16.t.hi) * 2 * sizeof(__half)));
        GemmParams p;     // transpose V of the slot with an identity "GEMM" stored through the transposed-block epilogue
        memset(&p, 0, sizeof(p));
        p.M = (int)kv_rows; p.N = kDModel; p.K = kDModel;
        p.a = offset(cs(v16.t), (size_t)d->slot * kDModel); p.a_mode = A_ROWMAJOR; p.lda = (int)kv_ld;
        p.Wt = wd; p.acc_scale = 1.f; p.add_period = 1;
        p.remap = 1; p.blk_map[0] = -(d->slot + 1); p.vt = vt16.t; p.n_vt = d->slots; p.ldc = kDModel;
        if (launch_gemm_simt(p, 0)) return 1;
        a.k = offset(cs(k16.t), (size_t)d->slot * kDModel); a.ldk = (int)kv_ld;
        a.vt = offset(cs(vt16.t), (size_t)d->slot * kVtLayer); a.vt_pair_stride = (size_t)d->slots * kVtLayer;
    }
    if (d->n_tiles > 0) {
        int4* tab = nullptr;
        if (mem.upload((void**)&tab, tiles.data(), tiles.size() * sizeof(int4))) return 1;
        a.tiles = tab; a.n_tiles = d->n_tiles;
    }
    int rc;
    if (d->path == 1) rc = launch_attention_simt(a, 0);
    else rc = d->key_split ? launch_attention_tc_split(a, d->key_split, 0) : launch_attention_tc(a, 0);
    if (!rc && maps_dev) {
        const AttnWeightsParams w = attention_weights_params(a, maps_dev + (size_t)d->maps_row0 * kTokens, (size_t)d->nq * kTokens);
        rc = d->path == 0 ? launch_attention_weights_tc(w, 0) : launch_attention_weights_simt(w, 0);
    }
    if (!rc) rc = launch_split16_to_f32(cs(o16.t), out_dev, (size_t)d->q_rows * kDModel, 0);
    const cudaError_t e = cudaDeviceSynchronize();
    if (rc) return rc;
    COTR_CHECK(e == cudaSuccess, "cotr_test_attention: kernel failed: %s", cudaGetErrorString(e));
    return 0;
}

// The fused feed-forward launch on its own; `out` (or x, in place) is converted in before the launch, so the rows >= M
// come back as they were passed.
int cotr_test_mlp(const cotr_test_mlp_desc* d, const float* x_dev, const float* w1_host, const float* b1_dev,
                  const float* w2_host, const float* b2_dev, const float* g_dev, const float* be_dev,
                  const float* g2_dev, const float* be2_dev, float* out_dev) {
    COTR_CHECK(d && x_dev && w1_host && b1_dev && w2_host && b2_dev && g_dev && be_dev && out_dev, "cotr_test_mlp: null argument");
    COTR_CHECK((g2_dev == nullptr) == (be2_dev == nullptr), "cotr_test_mlp: g2 and be2 go together");
    COTR_CHECK(d->M >= 1 && d->rows >= d->M, "cotr_test_mlp: M %d of %d rows", d->M, d->rows);
    COTR_CHECK(d->split == 0 || d->split == 4 || d->split == 8, "cotr_test_mlp: split %d (0 = launch rule, 4 or 8)", d->split);
    const size_t n = (size_t)d->rows * kDModel;
    DevAllocs mem;
    TmpSplit x16, o16;
    if (x16.from_f32(x_dev, n) || (!d->in_place && o16.from_f32(out_dev, n))) return 1;
    MlpParams p;
    memset(&p, 0, sizeof(p));
    void *w1 = nullptr, *w2 = nullptr;
    if (upload_tc_weight(mem, w1_host, kFF, kDModel, &w1, &p.w1_scale) || upload_tc_weight(mem, w2_host, kDModel, kFF, &w2, &p.w2_scale)) return 1;
    p.M = d->M; p.x = cs(x16.t); p.out = d->in_place ? x16.t : o16.t;
    p.w1 = w1; p.b1 = b1_dev; p.w2 = w2; p.b2 = b2_dev;
    p.g = g_dev; p.be = be_dev; p.g2 = g2_dev; p.be2 = be2_dev;
    int rc = d->split ? launch_mlp_tc_split(p, d->split, 0) : launch_mlp_tc(p, 0);
    if (!rc) rc = launch_split16_to_f32(cs(p.out), out_dev, n, 0);
    const cudaError_t e = cudaDeviceSynchronize();
    if (rc) return rc;
    COTR_CHECK(e == cudaSuccess, "cotr_test_mlp: kernel failed: %s", cudaGetErrorString(e));
    return 0;
}

int cotr_test_rowwise(int op, int rows, const float* in_dev, const float* g1_dev, const float* b1_dev,
                      const float* g2_dev, const float* b2_dev, float* out_dev) {
    COTR_CHECK(in_dev && out_dev && rows >= 1, "cotr_test_rowwise: null argument or %d rows", rows);
    COTR_CHECK(op >= 0 && op <= 3, "cotr_test_rowwise: op %d (0 LayerNorm, 1 fp32 LayerNorm, 2 two LayerNorms, 3 query encoding)", op);
    COTR_CHECK(op == 3 || (g1_dev && b1_dev), "cotr_test_rowwise: op %d needs g1 / b1", op);
    COTR_CHECK(op != 2 || (g2_dev && b2_dev), "cotr_test_rowwise: op 2 needs g2 / b2");
    const size_t n = (size_t)rows * kDModel;
    TmpSplit x16, o16;
    if (o16.empty(n) || ((op == 0 || op == 2) && x16.from_f32(in_dev, n))) return 1;
    int rc;
    switch (op) {
        case 0: rc = launch_layernorm(cs(x16.t), g1_dev, b1_dev, o16.t, rows, 0); break;
        case 1: rc = launch_layernorm_f32(in_dev, g1_dev, b1_dev, o16.t, rows, 0); break;
        case 2: rc = launch_layernorm_twice(cs(x16.t), g1_dev, b1_dev, g2_dev, b2_dev, o16.t, rows, 0); break;
        default: rc = launch_query_encode(in_dev, o16.t, rows, 0); break;
    }
    if (!rc) rc = launch_split16_to_f32(cs(o16.t), out_dev, n, 0);
    const cudaError_t e = cudaDeviceSynchronize();
    if (rc) return rc;
    COTR_CHECK(e == cudaSuccess, "cotr_test_rowwise: kernel failed: %s", cudaGetErrorString(e));
    return 0;
}

}  // extern "C"
