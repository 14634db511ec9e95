// extern "C" surface of libytk_b200.so (declared in include/yomitoku_b200.h).
#include "../../include/yomitoku_b200.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <tuple>
#include <vector>

#include "crop_ops.h"
#include "dbnet_engine.h"
#include "dbnet_ops.h"
#include "dbpost_ops.h"
#include "gemm_tc.h"
#include "parseq_engine.h"
#include "resample_ops.h"
#include "rtdetr_engine.h"

// Binds the calling host thread to a device for the duration of an API call and puts the previous device back (host
// threads start on device 0, and a handle on cuda:1 must not leave "the current device" changed for the caller - PyTorch
// allocates `device="cuda"` tensors on it).
struct DevGuard {
    int prev = -1, dev = -1;
    explicit DevGuard(int d) : dev(d) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
    }
    ~DevGuard() {
        if (prev >= 0 && prev != dev) cudaSetDevice(prev);
    }
    DevGuard(const DevGuard&) = delete;
    DevGuard& operator=(const DevGuard&) = delete;
};

struct ytk_parseq {
    ytk::ParseqModel model;
    ytk::ParseqEngine engine;
    std::mutex mu;
    int device = 0;  // the device current at create(); every later call binds the calling thread to it
};

struct ytk_dbnet {
    ytk::DbnetModel model;
    // launch plans + activation buffers per input shape (n, Hn, Wn); least recently used ones are dropped beyond
    // max_engines (YTK_DBNET_MAX_ENGINES, default 6) so that a stream of differently sized pages cannot exhaust HBM
    std::map<std::tuple<int, int, int>, std::unique_ptr<ytk::DbnetEngine>> engines;
    std::map<std::tuple<int, int, int>, unsigned long long> last_use;
    unsigned long long tick = 0;
    int max_engines = 6;
    std::mutex mu;
    int device = 0;
    int shortest = 1280, limit = 1600;
    void* stage = nullptr;  // device staging for host inputs
    size_t stage_bytes = 0;
    // The staging buffer and an engine's input / activation / probability buffers are shared by all calls on this
    // handle.  A call that leaves its output on the device returns while its kernels are still queued, so every call
    // first makes its stream wait for the previous call's last operation (recorded here), whatever stream that was on.
    cudaEvent_t last_done = nullptr;
};

static void order_after_previous(ytk_dbnet* h, cudaStream_t st) {
    if (h->last_done) cudaStreamWaitEvent(st, h->last_done, 0);
}
static void mark_done(ytk_dbnet* h, cudaStream_t st) {
    if (!h->last_done) cudaEventCreateWithFlags(&h->last_done, cudaEventDisableTiming);
    if (h->last_done) cudaEventRecord(h->last_done, st);
}

static ytk::DbnetEngine* get_engine(ytk_dbnet* h, int n, int Hn, int Wn) {
    auto key = std::make_tuple(n, Hn, Wn);
    h->last_use[key] = ++h->tick;
    auto it = h->engines.find(key);
    if (it != h->engines.end()) return it->second.get();
    while ((int)h->engines.size() >= h->max_engines && !h->engines.empty()) {
        auto victim = h->engines.begin();
        for (auto e = h->engines.begin(); e != h->engines.end(); ++e)
            if (h->last_use[e->first] < h->last_use[victim->first]) victim = e;
        cudaDeviceSynchronize();  // its last run may still be in flight on some stream
        h->last_use.erase(victim->first);
        h->engines.erase(victim);
    }
    auto e = std::make_unique<ytk::DbnetEngine>();
    if (e->build(h->model, n, Hn, Wn)) return nullptr;
    ytk::DbnetEngine* p = e.get();
    h->engines[key] = std::move(e);
    return p;
}

static int ensure_stage(ytk_dbnet* h, size_t bytes) {
    if (h->stage_bytes >= bytes) return 0;
    if (h->last_done) cudaEventSynchronize(h->last_done);  // the previous call may still be reading the old buffer
    if (h->stage) cudaFree(h->stage);
    h->stage = nullptr;
    h->stage_bytes = 0;
    if (cudaMalloc(&h->stage, bytes) != cudaSuccess) {
        ytk::set_error("cudaMalloc(%zu) for input staging failed", bytes);
        return 1;
    }
    h->stage_bytes = bytes;
    return 0;
}

static int finish_forward(ytk_dbnet* h, ytk::DbnetEngine* e, float* prob_out, int out_on_device, cudaStream_t st) {
    if (e->run(st)) return YTK_ERR;
    const size_t bytes = (size_t)e->N * e->Hn * e->Wn * sizeof(float);
    cudaError_t err = cudaMemcpyAsync(prob_out, e->prob, bytes,
                                      out_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st);
    mark_done(h, st);
    if (err == cudaSuccess && !out_on_device) err = cudaStreamSynchronize(st);
    if (err != cudaSuccess) {
        ytk::set_error("DBNet output copy failed: %s", cudaGetErrorString(err));
        return YTK_ERR;
    }
    return YTK_OK;
}

extern "C" {

const char* ytk_last_error(void) { return ytk::last_error(); }
int ytk_version(void) { return 1; }
long long ytk_launch_count(void) { return ytk::launch_count(); }
void ytk_gemm_profile_begin(void) { ytk::gemm_profile_begin(); }
int ytk_gemm_profile_end(double* flops, double* ms, long long* launches) {
    return ytk::gemm_profile_end(flops, ms, launches) ? YTK_ERR : YTK_OK;
}

int ytk_op_conv2d_f16(const void* in, int N, int H, int W, int Cin, long long in_ld, const void* w, const float* bias,
                       int kh, int kw, int stride, int pad, int dil, int Cout, const void* resid, int resid_f32,
                       long long ldr, void* out, int out_f32, long long ldc, int act, int mode, void* cuda_stream) {
    ytk::ConvGeom g{N, H, W, Cin, in_ld, kh, kw, stride, pad, dil, Cout};
    ytk::Epilogue e;
    e.bias = bias;
    e.resid = resid;
    e.resid_f32 = resid_f32;
    e.ldr = ldr;
    e.out = out;
    e.out_f32 = out_f32;
    e.ldc = ldc;
    e.act = act;
    e.mode = mode;
    ytk::GemmPlan plan;
    if (ytk::conv_plan_create(&plan, in, g, w, e)) return YTK_ERR;
    return ytk::gemm_plan_launch(&plan, static_cast<cudaStream_t>(cuda_stream)) ? YTK_ERR : YTK_OK;
}

int ytk_op_linear_f16(const void* A, long long lda, int M, int K, const void* W, int N, const float* bias,
                       const void* resid, int resid_f32, long long ldr, void* out, int out_f32, long long ldc, int act,
                       void* cuda_stream) {
    ytk::Epilogue e;
    e.bias = bias;
    e.resid = resid;
    e.resid_f32 = resid_f32;
    e.ldr = ldr;
    e.out = out;
    e.out_f32 = out_f32;
    e.ldc = ldc;
    e.act = act;
    ytk::GemmPlan plan;
    if (ytk::gemm_plan_create(&plan, A, lda, M, K, W, N, e)) return YTK_ERR;
    return ytk::gemm_plan_launch(&plan, static_cast<cudaStream_t>(cuda_stream)) ? YTK_ERR : YTK_OK;
}

static_assert(sizeof(ytk_attn_seq) == sizeof(ytk::SeqDesc), "ytk_attn_seq and ytk::SeqDesc must have one layout");

int ytk_op_attention_f16(const void* Q, long long ldq, long long q_rows, const void* K, const void* V, long long ldkv,
                         long long kv_rows, void* O, long long ldo, const ytk_attn_seq* seqs_dev, int nseq, int max_q_len,
                         int heads, int head_dim, int masked, int impl, void* cuda_stream) {
    return ytk::launch_flash_attention(Q, ldq, q_rows, K, V, ldkv, kv_rows, O, ldo,
                                       reinterpret_cast<const ytk::SeqDesc*>(seqs_dev), nseq, max_q_len, heads, head_dim,
                                       masked, static_cast<cudaStream_t>(cuda_stream), impl)
               ? YTK_ERR
               : YTK_OK;
}

int ytk_op_topk_f32(const float* scores_dev, int n, int L, int K, int* out_idx_dev, void* cuda_stream) {
    if (!scores_dev || !out_idx_dev) {
        ytk::set_error("ytk_op_topk_f32: null argument");
        return YTK_ERR;
    }
    return ytk::launch_rt_topk(scores_dev, n, L, K, out_idx_dev, static_cast<cudaStream_t>(cuda_stream)) ? YTK_ERR
                                                                                                         : YTK_OK;
}

static bool misaligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0; }

int ytk_op_deform_attn_f16(const float* ow, long long ldo, const float* ref, const void* value, long long ldv, int voff,
                           const int* level_h, const int* level_w, const int* level_points, int n_levels, int n_img, int K,
                           int heads, int head_dim, float offset_scale, void* out, long long ldout, void* cuda_stream) {
    if (!ow || !ref || !value || !out || !level_h || !level_w || !level_points) {
        ytk::set_error("ytk_op_deform_attn_f16: null argument");
        return YTK_ERR;
    }
    if (n_levels < 1 || n_levels > ytk::RtLevels::kMax) {
        ytk::set_error("ytk_op_deform_attn_f16: %d levels unsupported (1..%d)", n_levels, ytk::RtLevels::kMax);
        return YTK_ERR;
    }
    if (n_img < 1 || K < 1 || heads < 1 || head_dim < 1 || voff < 0) {
        ytk::set_error("ytk_op_deform_attn_f16: non-positive size (n_img %d, K %d, heads %d, head_dim %d, voff %d)", n_img,
                       K, heads, head_dim, voff);
        return YTK_ERR;
    }
    ytk::RtLevels lv;
    lv.n = n_levels;
    lv.off[0] = 0;
    int P = 0;
    for (int l = 0; l < n_levels; ++l) {
        if (level_h[l] < 1 || level_w[l] < 1 || level_points[l] < 1) {
            ytk::set_error("ytk_op_deform_attn_f16: level %d is %dx%d with %d points", l, level_h[l], level_w[l],
                           level_points[l]);
            return YTK_ERR;
        }
        lv.h[l] = level_h[l];
        lv.w[l] = level_w[l];
        lv.points[l] = level_points[l];
        lv.off[l + 1] = lv.off[l] + level_h[l] * level_w[l];
        P += level_points[l];
    }
    lv.total = lv.off[n_levels];
    if (ldo < 3LL * heads * P || ldv < (long long)voff + (long long)heads * head_dim || ldout < (long long)heads * head_dim ||
        misaligned(ref, 16)) {
        ytk::set_error("ytk_op_deform_attn_f16: pitches too small (ldo %lld, ldv %lld with voff %d, ldout %lld) or ref not "
                       "16-byte aligned", ldo, ldv, voff, ldout);
        return YTK_ERR;
    }
    return ytk::launch_rt_deform_attn(ow, ldo, ref, value, ldv, voff, lv, n_img, K, heads, head_dim, offset_scale, out,
                                      ldout, static_cast<cudaStream_t>(cuda_stream))
               ? YTK_ERR
               : YTK_OK;
}

int ytk_op_layernorm_f32(float* x, int M, int D, int d_real, const float* gamma, const float* beta, float eps,
                         void* out_f16, float* out_f32, const float* addvec, int period, const int* add_row0_dev,
                         int add_row0, int writeback, void* cuda_stream) {
    if (!x || !gamma || !beta) {
        ytk::set_error("ytk_op_layernorm_f32: null argument");
        return YTK_ERR;
    }
    // the first table row comes from *add_row0_dev when that is given: add_row0 is read only without it
    if (M < 1 || (addvec && (period < 1 || (!add_row0_dev && add_row0 < 0)))) {
        ytk::set_error("ytk_op_layernorm_f32: %d rows, addvec period %d / first row %d unsupported", M, period, add_row0);
        return YTK_ERR;
    }
    if (misaligned(x, 16) || misaligned(gamma, 16) || misaligned(beta, 16) || misaligned(out_f32, 16) ||
        misaligned(addvec, 16) || misaligned(out_f16, 8)) {
        ytk::set_error("ytk_op_layernorm_f32: fp32 pointers must be 16-byte and out_f16 8-byte aligned");
        return YTK_ERR;
    }
    return ytk::launch_layernorm(x, M, D, d_real, gamma, beta, eps, out_f16, out_f32, addvec, period, add_row0_dev,
                                 add_row0, writeback, static_cast<cudaStream_t>(cuda_stream))
               ? YTK_ERR
               : YTK_OK;
}

int ytk_op_single_query_attn_f16(int mode, const void* q, const void* kv, int B, int S, int D, int heads,
                                 const int* step_dev, const ytk_crop* crops, void* out, void* cuda_stream) {
    constexpr int kMaxTokens = ytk::kMaxMem;   // keys per (row, head) the kernel's shared-memory score row holds
    if (mode != 0 && mode != 1) {
        ytk::set_error("ytk_op_single_query_attn_f16: mode %d unknown (0 = self, 1 = cross)", mode);
        return YTK_ERR;
    }
    if (!q || !kv || !out || (mode == 0 && !step_dev) || (mode == 1 && !crops)) {
        ytk::set_error("ytk_op_single_query_attn_f16: null argument");
        return YTK_ERR;
    }
    const int hd = heads > 0 ? D / heads : 0;
    if (B < 1 || heads < 1 || D % heads != 0 || (hd != 32 && hd != 48 && hd != 64 && hd != 96)) {
        ytk::set_error("ytk_op_single_query_attn_f16: B %d, D %d, %d heads unsupported (head dim 32/48/64/96)", B, D,
                       heads);
        return YTK_ERR;
    }
    if (mode == 0 && (S < 1 || S > kMaxTokens)) {
        ytk::set_error("ytk_op_single_query_attn_f16: S %d unsupported (1..%d)", S, kMaxTokens);
        return YTK_ERR;
    }
    if (misaligned(q, 16) || misaligned(kv, 16) || misaligned(out, 16)) {
        ytk::set_error("ytk_op_single_query_attn_f16: q, kv and out must be 16-byte aligned");
        return YTK_ERR;
    }
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    if (mode == 0) return ytk::launch_dec_self_attn(q, kv, B, S, D, heads, step_dev, out, st) ? YTK_ERR : YTK_OK;
    std::vector<ytk::CropDesc> descs(B);
    for (int i = 0; i < B; ++i) {
        const ytk_crop& c = crops[i];
        if (c.ntok < 1 || c.ntok > kMaxTokens || c.tok_off < 0) {
            ytk::set_error("ytk_op_single_query_attn_f16: crop %d has %d tokens from row %d (1..%d tokens)", i, c.ntok,
                           c.tok_off, kMaxTokens);
            return YTK_ERR;
        }
        descs[i] = ytk::CropDesc{c.pix_off, c.w, c.wp, c.tok_off, c.ntok, c.group};
    }
    const size_t bytes = descs.size() * sizeof(ytk::CropDesc);
    void* descs_dev = nullptr;
    if (cudaMallocAsync(&descs_dev, bytes, st) != cudaSuccess) {
        cudaGetLastError();
        ytk::set_error("ytk_op_single_query_attn_f16: cudaMallocAsync(%zu) failed", bytes);
        return YTK_ERR;
    }
    // pageable source: the call returns after the records are staged, so `descs` may go out of scope
    int rc = cudaMemcpyAsync(descs_dev, descs.data(), bytes, cudaMemcpyHostToDevice, st) != cudaSuccess;
    if (rc) ytk::set_error("ytk_op_single_query_attn_f16: record upload failed");
    if (!rc) rc = ytk::launch_dec_cross_attn(q, kv, reinterpret_cast<const ytk::CropDesc*>(descs_dev), B, D, heads, out, st);
    cudaFreeAsync(descs_dev, st);
    return rc ? YTK_ERR : YTK_OK;
}

// ---- the recognizer's decoding tail (parseq_ops.cu, gemm_tc.cu EPI_ROWMAX), each entry called as the engine calls it
int ytk_op_linear_rowmax_f16(const void* A, long long lda, int M, int K, const void* W, int N, const float* bias,
                             int argmax_only, void* partials, long long partials_capacity, int* npart_out,
                             int* block_n_out, void* cuda_stream) {
    if (!A || !W || !partials) {
        ytk::set_error("ytk_op_linear_rowmax_f16: null argument");
        return YTK_ERR;
    }
    if (M < 1 || N < 1 || K < 64 || K % 64 != 0 || lda < K || lda % 8 != 0) {
        ytk::set_error("ytk_op_linear_rowmax_f16: M %d, K %d, N %d, lda %lld unsupported (K a multiple of 64, lda >= K "
                       "and a multiple of 8)", M, K, N, lda);
        return YTK_ERR;
    }
    if (misaligned(A, 16) || misaligned(W, 16) || misaligned(bias, 16) || misaligned(partials, 16)) {
        ytk::set_error("ytk_op_linear_rowmax_f16: A, W, bias and partials must be 16-byte aligned");
        return YTK_ERR;
    }
    // the widest N tile (256) gives the fewest partials: a capacity below that is too small whatever the plan picks
    const long long least = (long long)M * 2 * ((N + 255) / 256);
    if (partials_capacity < least) {
        ytk::set_error("ytk_op_linear_rowmax_f16: partials_capacity %lld float4s < %lld (M %d x at least %lld partials)",
                       partials_capacity, least, M, least / M);
        return YTK_ERR;
    }
    ytk::Epilogue e;
    e.bias = bias;
    e.out = partials;
    e.out_f32 = 1;
    e.mode = ytk::EPI_ROWMAX;
    e.act = argmax_only ? ytk::ACT_RELU : ytk::ACT_NONE;   // ACT_RELU: the sum-free mode of the AR loop
    ytk::GemmPlan plan;
    if (ytk::gemm_plan_create(&plan, A, lda, M, K, W, N, e)) return YTK_ERR;
    const long long npart = plan.args.ldc;                // 2 * tiles_n float4s per row
    if (partials_capacity < (long long)M * npart) {
        ytk::set_error("ytk_op_linear_rowmax_f16: partials_capacity %lld float4s < %lld (M %d x %lld partials at "
                       "block_n %d)", partials_capacity, (long long)M * npart, M, npart, plan.block_n);
        return YTK_ERR;
    }
    if (npart_out) *npart_out = (int)npart;
    if (block_n_out) *block_n_out = plan.block_n;
    return ytk::gemm_plan_launch(&plan, static_cast<cudaStream_t>(cuda_stream)) ? YTK_ERR : YTK_OK;
}

// rows / positions / output indices shared by the two softmax-statistics entries
static bool bad_stat_rows(const char* who, int C, int rows, int S, long long g_stride, long long g_off, int eos_id) {
    if (C < 1 || rows < 1 || S < 1 || g_stride < 0 || g_off < 0 || eos_id < 0) {
        ytk::set_error("%s: C %d, %d rows, S %d, g_stride %lld, g_off %lld, eos_id %d unsupported", who, C, rows, S,
                       g_stride, g_off, eos_id);
        return true;
    }
    return false;
}

int ytk_op_softmax_max_f32(const float* logits, long long ldl, int C, int rows, int S, long long g_stride,
                           long long g_off, const int* rep_cut, int eos_id, int* ids, float* probs, void* cuda_stream) {
    if (!logits || !ids || !probs) {
        ytk::set_error("ytk_op_softmax_max_f32: null argument");
        return YTK_ERR;
    }
    if (bad_stat_rows("ytk_op_softmax_max_f32", C, rows, S, g_stride, g_off, eos_id)) return YTK_ERR;
    // the kernel reads rows as float4: 16-byte aligned rows of at least C floats
    if (ldl < C || ldl % 4 != 0 || misaligned(logits, 16)) {
        ytk::set_error("ytk_op_softmax_max_f32: ldl %lld for C %d (ldl >= C, a multiple of 4) or logits not 16-byte "
                       "aligned", ldl, C);
        return YTK_ERR;
    }
    return ytk::launch_softmax_max(logits, ldl, C, rows, S, g_stride, g_off, rep_cut, eos_id, ids, probs,
                                   static_cast<cudaStream_t>(cuda_stream))
               ? YTK_ERR
               : YTK_OK;
}

int ytk_op_rowmax_finalize_f32(const void* partials, long long ldp, int npart, int C, int rows, int S,
                               long long g_stride, long long g_off, const int* rep_cut, int eos_id, int* ids,
                               float* probs, void* cuda_stream) {
    if (!partials || !ids || !probs) {
        ytk::set_error("ytk_op_rowmax_finalize_f32: null argument");
        return YTK_ERR;
    }
    if (bad_stat_rows("ytk_op_rowmax_finalize_f32", C, rows, S, g_stride, g_off, eos_id)) return YTK_ERR;
    if (npart < 1 || npart > ldp || misaligned(partials, 16)) {
        ytk::set_error("ytk_op_rowmax_finalize_f32: npart %d, ldp %lld (1 <= npart <= ldp) or partials not 16-byte "
                       "aligned", npart, ldp);
        return YTK_ERR;
    }
    return ytk::launch_rowmax_finalize(static_cast<const float*>(partials), ldp, npart, C, rows, S, g_stride, g_off,
                                       rep_cut, eos_id, ids, probs, static_cast<cudaStream_t>(cuda_stream))
               ? YTK_ERR
               : YTK_OK;
}

static_assert(sizeof(ytk_ar_state) == sizeof(ytk::ArState), "ytk_ar_state and ytk::ArState must have one layout");
static_assert(offsetof(ytk_ar_state, ticket) == offsetof(ytk::ArState, ticket) &&
                  offsetof(ytk_ar_state, group_len) == offsetof(ytk::ArState, group_len),
              "ytk_ar_state and ytk::ArState must have one layout");

// content embedding + LN_c arguments shared by ar_control and refine_embed
static bool bad_embed(const char* who, const float* embed, const float* pos_q, int D, int d_real, const float* g_c,
                      const float* b_c, const void* cin) {
    if (!embed || !pos_q || !g_c || !b_c || !cin) {
        ytk::set_error("%s: null argument", who);
        return true;
    }
    if (D < 1 || D > 1024 || d_real < 1 || d_real > D) {   // 256 threads x 4 features per row
        ytk::set_error("%s: D %d / d_real %d unsupported (1 <= d_real <= D <= 1024)", who, D, d_real);
        return true;
    }
    return false;
}

int ytk_op_ar_control(const float* logits, long long ldl, int C, int npart, int B, int S, const int* row_group, int g0,
                      int ngroups, const ytk_ar_state* state, int eos_id, int rep_on, int rep_period_max,
                      int rep_min_run_p1, int rep_min_repeats, const float* embed, const float* pos_q, int D,
                      int d_real, const float* g_c, const float* b_c, void* cin, void* cuda_stream) {
    const char* who = "ytk_op_ar_control";
    if (!logits || !row_group || !state || !state->tgt || !state->raw || !state->rep_cut || !state->rep_done ||
        !state->has_eos || !state->group_len || !state->n_active || !state->step || !state->open_rows ||
        !state->ticket) {
        ytk::set_error("%s: null argument", who);
        return YTK_ERR;
    }
    if (bad_embed(who, embed, pos_q, D, d_real, g_c, b_c, cin)) return YTK_ERR;
    if (B < 1 || S < 1 || C < 1 || npart < 0) {
        ytk::set_error("%s: B %d, S %d, C %d, npart %d unsupported", who, B, S, C, npart);
        return YTK_ERR;
    }
    // npart > 0: rows of ldl float4 partials; npart == 0: rows of ldl fp32 logits read as float4
    if ((npart > 0 ? ldl < npart : (ldl < C || ldl % 4 != 0)) || misaligned(logits, 16)) {
        ytk::set_error("%s: ldl %lld too small for C %d / npart %d (or not a multiple of 4), or logits not 16-byte "
                       "aligned", who, ldl, C, npart);
        return YTK_ERR;
    }
    if (eos_id < 0 || eos_id >= C) {
        ytk::set_error("%s: eos_id %d outside [0, %d)", who, eos_id, C);
        return YTK_ERR;
    }
    if (ngroups < 1 || g0 < 0) {
        ytk::set_error("%s: %d groups from g0 %d unsupported", who, ngroups, g0);
        return YTK_ERR;
    }
    if (rep_on && (rep_period_max < 1 || rep_min_run_p1 < 1 || rep_min_repeats < 1)) {
        ytk::set_error("%s: repetition stop with period_max %d, min_run_p1 %d, min_repeats %d unsupported", who,
                       rep_period_max, rep_min_run_p1, rep_min_repeats);
        return YTK_ERR;
    }
    ytk::ArState a;
    a.tgt = state->tgt;
    a.raw = state->raw;
    a.rep_cut = state->rep_cut;
    a.rep_done = state->rep_done;
    a.has_eos = state->has_eos;
    a.group_len = state->group_len;
    a.n_active = state->n_active;
    a.step = state->step;
    a.open_rows = state->open_rows;
    a.ticket = state->ticket;
    return ytk::launch_ar_control(logits, ldl, C, npart, B, S, row_group, g0, ngroups, a, eos_id, rep_on, rep_period_max,
                                  rep_min_run_p1, rep_min_repeats, embed, pos_q, D, d_real, g_c, b_c, cin,
                                  static_cast<cudaStream_t>(cuda_stream))
               ? YTK_ERR
               : YTK_OK;
}

int ytk_op_refine_embed(const int* raw, const int* row_group, const int* group_len, int B, int S, int bos_id,
                        int eos_id, const float* embed, const float* pos_q, int D, int d_real, const float* g_c,
                        const float* b_c, void* cin, int* klen, int* kpad, void* cuda_stream) {
    const char* who = "ytk_op_refine_embed";
    if (!raw || !row_group || !group_len || !klen || !kpad) {
        ytk::set_error("%s: null argument", who);
        return YTK_ERR;
    }
    if (bad_embed(who, embed, pos_q, D, d_real, g_c, b_c, cin)) return YTK_ERR;
    if (B < 1 || B > 65535 || S < 1 || bos_id < 0 || eos_id < 0) {   // grid (S, B)
        ytk::set_error("%s: B %d, S %d, bos_id %d, eos_id %d unsupported (1 <= B <= 65535)", who, B, S, bos_id,
                       eos_id);
        return YTK_ERR;
    }
    return ytk::launch_refine_embed(raw, row_group, group_len, B, S, bos_id, eos_id, embed, pos_q, D, d_real, g_c, b_c,
                                    cin, klen, kpad, static_cast<cudaStream_t>(cuda_stream))
               ? YTK_ERR
               : YTK_OK;
}

int ytk_op_apply_rep_cut(const int* rep_cut, int B, int S, int C, int eos_id, int* ids, float* probs,
                         void* cuda_stream) {
    if (!rep_cut || !ids || !probs) {
        ytk::set_error("ytk_op_apply_rep_cut: null argument");
        return YTK_ERR;
    }
    if (B < 1 || S < 1 || C < 1 || eos_id < 0) {
        ytk::set_error("ytk_op_apply_rep_cut: B %d, S %d, C %d, eos_id %d unsupported", B, S, C, eos_id);
        return YTK_ERR;
    }
    return ytk::launch_apply_rep_cut(rep_cut, B, S, C, eos_id, ids, probs, static_cast<cudaStream_t>(cuda_stream))
               ? YTK_ERR
               : YTK_OK;
}

// Allocates `bytes` on the stream and, if `host` is given, uploads it.  The copy is from pageable memory: the call
// returns after the data is staged, so `host` may go out of scope.  The caller frees the buffer with cudaFreeAsync.
static void* stream_buffer(const void* host, size_t bytes, cudaStream_t st, const char* who) {
    void* d = nullptr;
    if (cudaMallocAsync(&d, bytes, st) != cudaSuccess) {
        cudaGetLastError();
        ytk::set_error("%s: cudaMallocAsync(%zu) failed", who, bytes);
        return nullptr;
    }
    if (host && cudaMemcpyAsync(d, host, bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) {
        cudaGetLastError();
        cudaFreeAsync(d, st);
        ytk::set_error("%s: upload of %zu bytes failed", who, bytes);
        return nullptr;
    }
    return d;
}

// A page table: n records {page_off, H, W, rectangle} of pages back to back in `pages_bytes` bytes (ytk_page).  Records
// come from the caller: a page beyond the buffer, an empty page or a rectangle outside its page is an error, and so is
// a rectangle other than the whole page where the entry reads whole pages.
static int check_page_table(const ytk_page* t, int n, long long pages_bytes, bool whole, const char* who) {
    if (!t || n < 1 || n > 65535 || pages_bytes < 1) {
        ytk::set_error("%s: %d page records for %lld page bytes (1..65535 records, a non-empty buffer)", who, n,
                       pages_bytes);
        return 1;
    }
    for (int i = 0; i < n; ++i) {
        const ytk_page& p = t[i];
        const bool ok = p.page_off >= 0 && p.H >= 1 && p.W >= 1 && p.page_off <= pages_bytes &&
                        (long long)p.H * p.W <= (pages_bytes - p.page_off) / 3 && p.x0 >= 0 && p.x0 < p.x1 &&
                        p.x1 <= p.W && p.y0 >= 0 && p.y0 < p.y1 && p.y1 <= p.H;
        if (!ok) {
            ytk::set_error("%s: page %d (at %lld, %dx%d, rectangle x %d..%d y %d..%d) is empty, has a rectangle outside "
                           "it, or overruns the %lld page bytes", who, i, p.page_off, p.H, p.W, p.x0, p.x1, p.y0, p.y1,
                           pages_bytes);
            return 1;
        }
        if (whole && (p.x0 != 0 || p.y0 != 0 || p.x1 != p.W || p.y1 != p.H)) {
            ytk::set_error("%s: page %d (%dx%d) has the rectangle x %d..%d y %d..%d; the detector reads whole pages", who,
                           i, p.H, p.W, p.x0, p.x1, p.y0, p.y1);
            return 1;
        }
    }
    return 0;
}

static_assert(sizeof(ytk_page) == sizeof(ytk::RtSrc), "ytk_page and ytk::RtSrc must have one layout");

// The two pre-processing entries: `up` = 0 takes the shapes OpenCV decimates with its area tables (no axis grows),
// `up` = 1 the shapes it up-scales bilinearly (some axis grows).  One launcher serves both and picks by the same rule.
static int op_dbnet_preprocess(const char* who, int up, const uint8_t* src_dev, int n, int H0, int W0, int Hn, int Wn,
                               void* canvas_dev, void* cuda_stream) {
    if (!src_dev || !canvas_dev) {
        ytk::set_error("%s: null argument", who);
        return YTK_ERR;
    }
    if (n < 1 || H0 < 1 || W0 < 1 || Hn < 1 || Wn < 1) {
        ytk::set_error("%s: non-positive size (n %d, page %dx%d, input %dx%d)", who, n, H0, W0, Hn, Wn);
        return YTK_ERR;
    }
    const bool grows = Hn > H0 || Wn > W0;
    if (grows && !up) {
        ytk::set_error("%s: %dx%d -> %dx%d is an upscale; INTER_AREA decimation only (ytk_op_dbnet_preprocess_up_u8 "
                       "takes it)", who, H0, W0, Hn, Wn);
        return YTK_ERR;
    }
    if (!grows && up) {
        ytk::set_error("%s: %dx%d -> %dx%d grows no axis; INTER_AREA decimation is ytk_op_dbnet_preprocess_u8", who, H0,
                       W0, Hn, Wn);
        return YTK_ERR;
    }
    if (misaligned(canvas_dev, 16)) {
        ytk::set_error("%s: canvas_dev must be 16-byte aligned", who);
        return YTK_ERR;
    }
    return ytk::launch_preprocess(src_dev, n, H0, W0, Hn, Wn, canvas_dev, static_cast<cudaStream_t>(cuda_stream))
               ? YTK_ERR
               : YTK_OK;
}

int ytk_op_dbnet_preprocess_u8(const uint8_t* src_dev, int n, int H0, int W0, int Hn, int Wn, void* canvas_dev,
                               void* cuda_stream) {
    return op_dbnet_preprocess("ytk_op_dbnet_preprocess_u8", 0, src_dev, n, H0, W0, Hn, Wn, canvas_dev, cuda_stream);
}

int ytk_op_dbnet_preprocess_up_u8(const uint8_t* src_dev, int n, int H0, int W0, int Hn, int Wn, void* canvas_dev,
                                  void* cuda_stream) {
    return op_dbnet_preprocess("ytk_op_dbnet_preprocess_up_u8", 1, src_dev, n, H0, W0, Hn, Wn, canvas_dev, cuda_stream);
}

int ytk_op_dbnet_preprocess_table_u8(const uint8_t* pages_dev, long long pages_bytes, const ytk_page* table, int n,
                                     int Hn, int Wn, void* canvas_dev, void* cuda_stream) {
    const char* who = "ytk_op_dbnet_preprocess_table_u8";
    if (!pages_dev || !canvas_dev) {
        ytk::set_error("%s: null argument", who);
        return YTK_ERR;
    }
    if (Hn < 1 || Wn < 1) {
        ytk::set_error("%s: non-positive input size %dx%d", who, Hn, Wn);
        return YTK_ERR;
    }
    if (check_page_table(table, n, pages_bytes, true, who)) return YTK_ERR;
    if (misaligned(canvas_dev, 16)) {
        ytk::set_error("%s: canvas_dev must be 16-byte aligned", who);
        return YTK_ERR;
    }
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    void* d = stream_buffer(table, (size_t)n * sizeof(ytk_page), st, who);
    if (!d) return YTK_ERR;
    const int rc = ytk::launch_preprocess_table(pages_dev, static_cast<const ytk::RtSrc*>(d), n, Hn, Wn, canvas_dev, st);
    cudaFreeAsync(d, st);
    return rc ? YTK_ERR : YTK_OK;
}

int ytk_op_dbnet_stem_f16(const void* canvas_dev, int n, int Hn, int Wn, const float* w_host, const float* bias_host,
                          void* out_dev, void* cuda_stream) {
    if (!canvas_dev || !w_host || !bias_host || !out_dev) {
        ytk::set_error("ytk_op_dbnet_stem_f16: null argument");
        return YTK_ERR;
    }
    if (n < 1 || Hn < 32 || Wn < 32 || Hn % 32 || Wn % 32) {
        ytk::set_error("ytk_op_dbnet_stem_f16: n %d, input %dx%d unsupported (multiples of 32)", n, Hn, Wn);
        return YTK_ERR;
    }
    if (misaligned(canvas_dev, 16) || misaligned(out_dev, 16)) {
        ytk::set_error("ytk_op_dbnet_stem_f16: canvas_dev and out_dev must be 16-byte aligned");
        return YTK_ERR;
    }
    // one buffer: packed weights [64][7][64] 16-bit, then the bias [64] fp32
    std::vector<uint16_t> wp;
    ytk::pack_stem_weights(w_host, nullptr, &wp);
    const size_t wbytes = wp.size() * 2;
    std::vector<uint8_t> blob(wbytes + 64 * 4);
    memcpy(blob.data(), wp.data(), wbytes);
    memcpy(blob.data() + wbytes, bias_host, 64 * 4);
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    uint8_t* d = static_cast<uint8_t*>(stream_buffer(blob.data(), blob.size(), st, "ytk_op_dbnet_stem_f16"));
    if (!d) return YTK_ERR;
    ytk::Epilogue e;
    e.bias = reinterpret_cast<const float*>(d + wbytes);
    e.out = out_dev;
    e.ldc = 64;
    e.act = ytk::ACT_RELU;
    ytk::GemmPlan plan;
    int rc = ytk::stem_plan_create(&plan, canvas_dev, n, Hn, Wn, d, e);
    if (!rc) rc = ytk::gemm_plan_launch(&plan, st);
    cudaFreeAsync(d, st);
    return rc ? YTK_ERR : YTK_OK;
}

int ytk_op_maxpool3x3s2_f16(const void* in, int n, int H, int W, int C, void* out, void* cuda_stream) {
    if (!in || !out) {
        ytk::set_error("ytk_op_maxpool3x3s2_f16: null argument");
        return YTK_ERR;
    }
    if (n < 1 || H < 1 || W < 1 || C < 8 || C % 8) {
        ytk::set_error("ytk_op_maxpool3x3s2_f16: n %d, %dx%d, C %d unsupported (C a positive multiple of 8)", n, H, W, C);
        return YTK_ERR;
    }
    if (misaligned(in, 16) || misaligned(out, 16)) {
        ytk::set_error("ytk_op_maxpool3x3s2_f16: in and out must be 16-byte aligned");
        return YTK_ERR;
    }
    return ytk::launch_maxpool(in, out, n, H, W, C, static_cast<cudaStream_t>(cuda_stream)) ? YTK_ERR : YTK_OK;
}

int ytk_op_upsample_bilinear_f16(const void* src, int n, int Hs, int Ws, int C, void* dst, int Hd, int Wd, long long ldd,
                                 int coff, int accumulate, void* cuda_stream) {
    if (!src || !dst) {
        ytk::set_error("ytk_op_upsample_bilinear_f16: null argument");
        return YTK_ERR;
    }
    if (n < 1 || Hs < 1 || Ws < 1 || Hd < 1 || Wd < 1 || C < 8 || C % 8) {
        ytk::set_error("ytk_op_upsample_bilinear_f16: n %d, %dx%d -> %dx%d, C %d unsupported (C a positive multiple of 8)",
                       n, Hs, Ws, Hd, Wd, C);
        return YTK_ERR;
    }
    if (coff < 0 || coff % 8 || ldd % 8 || (long long)coff + C > ldd) {
        ytk::set_error("ytk_op_upsample_bilinear_f16: channels [%d, %d) do not fit a pitch of %lld (coff and ldd multiples "
                       "of 8)", coff, coff + C, ldd);
        return YTK_ERR;
    }
    if (misaligned(src, 16) || misaligned(dst, 16)) {
        ytk::set_error("ytk_op_upsample_bilinear_f16: src and dst must be 16-byte aligned");
        return YTK_ERR;
    }
    return ytk::launch_upsample(src, n, Hs, Ws, C, dst, Hd, Wd, ldd, coff, accumulate,
                                static_cast<cudaStream_t>(cuda_stream))
               ? YTK_ERR
               : YTK_OK;
}

int ytk_op_asf_f16(const void* a, void* fuse, int n, int H, int W, const float* w1_dev, const float* w2_dev,
                   const float* sp3_host, float sp1, const float* att_host, float* gvec_out, float* m_out,
                   void* cuda_stream) {
    if (!a || !fuse || !w1_dev || !w2_dev || !sp3_host || !att_host) {
        ytk::set_error("ytk_op_asf_f16: null argument");
        return YTK_ERR;
    }
    // the pooling grid is (chunks, n): n is bounded by gridDim.y
    if (n < 1 || n > 65535 || H < 1 || W < 1 || (long long)H * W > INT_MAX) {
        ytk::set_error("ytk_op_asf_f16: n %d, %dx%d unsupported (1 <= n <= 65535)", n, H, W);
        return YTK_ERR;
    }
    if (misaligned(a, 16) || misaligned(fuse, 16)) {
        ytk::set_error("ytk_op_asf_f16: a and fuse must be 16-byte aligned");
        return YTK_ERR;
    }
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    // fp32 scratch on the stream: gsum partials, gmean, and the outputs the caller does not want
    const size_t n_gsum = (size_t)n * ytk::kAsfPoolChunks * 64, n_gvec = gvec_out ? 0 : (size_t)n * 64,
                 n_m = m_out ? 0 : (size_t)n * H * W;
    float* d = static_cast<float*>(stream_buffer(nullptr, (n_gsum + n + n_gvec + n_m) * 4, st, "ytk_op_asf_f16"));
    if (!d) return YTK_ERR;
    float* gsum = d;
    float* gmean = gsum + n_gsum;
    float* gvec = gvec_out ? gvec_out : gmean + n;
    float* m = m_out ? m_out : gmean + n + n_gvec;
    const int rc = ytk::launch_asf(a, fuse, n, H, W, w1_dev, w2_dev, sp3_host, sp1, att_host, gsum, gvec, gmean, m, st);
    cudaFreeAsync(d, st);
    return rc ? YTK_ERR : YTK_OK;
}

int ytk_op_dbnet_head_f32(const void* x_dev, int n, int H, int W, const float* w1_host, const float* b1_host,
                          const float* w2_host, float b2, float* prob_dev, void* cuda_stream) {
    if (!x_dev || !w1_host || !b1_host || !w2_host || !prob_dev) {
        ytk::set_error("ytk_op_dbnet_head_f32: null argument");
        return YTK_ERR;
    }
    if (n < 1 || H < 1 || W < 1) {
        ytk::set_error("ytk_op_dbnet_head_f32: non-positive size (n %d, %dx%d)", n, H, W);
        return YTK_ERR;
    }
    if (misaligned(x_dev, 16) || misaligned(prob_dev, 8)) {
        ytk::set_error("ytk_op_dbnet_head_f32: x_dev must be 16-byte and prob_dev 8-byte aligned");
        return YTK_ERR;
    }
    // one buffer: GEMM rows [256][64] 16-bit, bias [256] fp32, final conv weights [4][64] fp32
    std::vector<uint16_t> wp;
    std::vector<float> bias, fin;
    ytk::pack_convt_head(w1_host, b1_host, nullptr, nullptr, w2_host, &wp, &bias, &fin);
    const size_t wbytes = wp.size() * 2, bbytes = bias.size() * 4;
    std::vector<uint8_t> blob(wbytes + bbytes + fin.size() * 4);
    memcpy(blob.data(), wp.data(), wbytes);
    memcpy(blob.data() + wbytes, bias.data(), bbytes);
    memcpy(blob.data() + wbytes + bbytes, fin.data(), fin.size() * 4);
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    uint8_t* d = static_cast<uint8_t*>(stream_buffer(blob.data(), blob.size(), st, "ytk_op_dbnet_head_f32"));
    if (!d) return YTK_ERR;
    ytk::ConvGeom g{n, H, W, 64, 64, 1, 1, 1, 0, 1, 256};
    ytk::Epilogue e;
    e.bias = reinterpret_cast<const float*>(d + wbytes);
    e.out = prob_dev;
    e.out_f32 = 1;
    e.ldc = 4;
    e.mode = ytk::EPI_CONVT_FINAL;
    e.fin_w = reinterpret_cast<const float*>(d + wbytes + bbytes);
    e.fin_b = b2;
    ytk::GemmPlan plan;
    int rc = ytk::conv_plan_create(&plan, x_dev, g, d, e);
    if (!rc) rc = ytk::gemm_plan_launch(&plan, st);
    cudaFreeAsync(d, st);
    return rc ? YTK_ERR : YTK_OK;
}

static_assert(sizeof(ytk_db_run) == sizeof(ytk::DbRun), "ytk_db_run and ytk::DbRun must have one layout");

int ytk_dbnet_post_front(const float* prob_dev, int n_pages, int H, int W, float thresh, void* scratch_dev,
                         long long scratch_bytes, ytk_db_run* runs_dev, int max_runs_per_page, int32_t* meta_dev,
                         void* cuda_stream) {
    if (!prob_dev || !scratch_dev || !runs_dev || !meta_dev || n_pages <= 0 || H <= 0 || W <= 0 || max_runs_per_page <= 0 ||
        (long long)H * W >= 0x7fffffffLL) {
        ytk::set_error("ytk_dbnet_post_front: bad arguments");
        return YTK_ERR;
    }
    if (scratch_bytes < ytk::dbpost_scratch_bytes(n_pages, H, W)) {
        ytk::set_error("ytk_dbnet_post_front: scratch_dev holds %lld bytes, need %lld", scratch_bytes,
                       ytk::dbpost_scratch_bytes(n_pages, H, W));
        return YTK_ERR;
    }
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, prob_dev) != cudaSuccess || attr.type != cudaMemoryTypeDevice) {
        cudaGetLastError();
        ytk::set_error("ytk_dbnet_post_front: prob_dev is not a device pointer");
        return YTK_ERR;
    }
    DevGuard dev_guard(attr.device);
    if (ytk::launch_dbpost_front(prob_dev, n_pages, H, W, thresh, reinterpret_cast<int*>(scratch_dev),
                                 reinterpret_cast<ytk::DbRun*>(runs_dev), max_runs_per_page, meta_dev,
                                 static_cast<cudaStream_t>(cuda_stream))) {
        ytk::set_error("ytk_dbnet_post_front: kernel launch failed");
        return YTK_ERR;
    }
    return YTK_OK;
}

int ytk_dbnet_create(const ytk_tensor* tensors, int n_tensors, int shortest_size, int limit_size, ytk_dbnet** out) {
    if (!tensors || !out) {
        ytk::set_error("ytk_dbnet_create: null argument");
        return YTK_ERR;
    }
    ytk::WeightSet ws;
    for (int i = 0; i < n_tensors; ++i) {
        ytk::TensorView v;
        v.data = tensors[i].data;
        v.ndim = tensors[i].ndim;
        for (int d = 0; d < 4; ++d) v.shape[d] = d < v.ndim ? tensors[i].shape[d] : 1;
        ws.map[tensors[i].name] = v;
    }
    auto h = std::make_unique<ytk_dbnet>();
    cudaGetDevice(&h->device);
    h->shortest = shortest_size;
    h->limit = limit_size;
    if (const char* me = getenv("YTK_DBNET_MAX_ENGINES")) h->max_engines = std::max(1, atoi(me));
    if (h->model.load(ws)) return YTK_ERR;
    *out = h.release();
    return YTK_OK;
}

void ytk_dbnet_destroy(ytk_dbnet* h) {
    if (!h) return;
    DevGuard dev_guard(h->device);
    if (h->last_done) {
        cudaEventSynchronize(h->last_done);
        cudaEventDestroy(h->last_done);
    }
    if (h->stage) cudaFree(h->stage);
    delete h;
}

int ytk_dbnet_device(const ytk_dbnet* h) { return h ? h->device : -1; }
int ytk_parseq_device(const ytk_parseq* h) { return h ? h->device : -1; }

int ytk_dbnet_input_size(const ytk_dbnet* h, int H0, int W0, int* Hn, int* Wn) {
    ytk::dbnet_input_size(H0, W0, h->shortest, h->limit, Hn, Wn);
    return YTK_OK;
}

int ytk_dbnet_forward_u8(ytk_dbnet* h, const uint8_t* pages, int pages_on_device, int n_pages, int H0, int W0,
                         float* prob_out, int out_on_device, void* cuda_stream) {
    std::lock_guard<std::mutex> lk(h->mu);
    DevGuard dev_guard(h->device);  // host threads start on device 0: the handle's device is the one that counts
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    int Hn, Wn;
    ytk::dbnet_input_size(H0, W0, h->shortest, h->limit, &Hn, &Wn);
    ytk::DbnetEngine* e = get_engine(h, n_pages, Hn, Wn);
    if (!e) return YTK_ERR;
    order_after_previous(h, st);
    const uint8_t* src = pages;
    if (!pages_on_device) {
        const size_t bytes = (size_t)n_pages * H0 * W0 * 3;
        if (ensure_stage(h, bytes)) return YTK_ERR;
        if (cudaMemcpyAsync(h->stage, pages, bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) {
            ytk::set_error("H2D copy of pages failed");
            return YTK_ERR;
        }
        src = reinterpret_cast<const uint8_t*>(h->stage);
    }
    if (ytk::launch_preprocess(src, n_pages, H0, W0, Hn, Wn, e->input, st)) {
        ytk::set_error("preprocess launch failed");
        return YTK_ERR;
    }
    return finish_forward(h, e, prob_out, out_on_device, st);
}

int ytk_dbnet_forward_table_u8(ytk_dbnet* h, const uint8_t* pages, int pages_on_device, long long pages_bytes,
                               const ytk_page* table, int n_pages, float* prob_out, int out_on_device,
                               void* cuda_stream) {
    const char* who = "ytk_dbnet_forward_table_u8";
    if (!h || !pages || !prob_out) {
        ytk::set_error("%s: null argument", who);
        return YTK_ERR;
    }
    if (check_page_table(table, n_pages, pages_bytes, true, who)) return YTK_ERR;
    // one engine per call: every page must map to the same network input
    int Hn, Wn;
    ytk::dbnet_input_size(table[0].H, table[0].W, h->shortest, h->limit, &Hn, &Wn);
    for (int i = 1; i < n_pages; ++i) {
        int hn, wn;
        ytk::dbnet_input_size(table[i].H, table[i].W, h->shortest, h->limit, &hn, &wn);
        if (hn != Hn || wn != Wn) {
            ytk::set_error("%s: page 0 (%dx%d) maps to the input %dx%d but page %d (%dx%d) to %dx%d; one call takes pages "
                           "of one input size", who, table[0].H, table[0].W, Hn, Wn, i, table[i].H, table[i].W, hn, wn);
            return YTK_ERR;
        }
    }
    std::lock_guard<std::mutex> lk(h->mu);
    DevGuard dev_guard(h->device);  // host threads start on device 0: the handle's device is the one that counts
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    ytk::DbnetEngine* e = get_engine(h, n_pages, Hn, Wn);
    if (!e) return YTK_ERR;
    // the staging buffer holds [host pages (16-byte aligned) |] the page table
    const size_t page_bytes = pages_on_device ? 0 : (size_t)(pages_bytes + 15) / 16 * 16;
    const size_t table_bytes = (size_t)n_pages * sizeof(ytk_page);
    if (ensure_stage(h, page_bytes + table_bytes)) return YTK_ERR;
    order_after_previous(h, st);
    const uint8_t* src = pages;
    uint8_t* stage = reinterpret_cast<uint8_t*>(h->stage);
    if (!pages_on_device) {
        if (cudaMemcpyAsync(stage, pages, (size_t)pages_bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) {
            ytk::set_error("%s: H2D copy of pages failed", who);
            return YTK_ERR;
        }
        src = stage;
    }
    // pageable records: the call returns after they are staged, so the caller may reuse them at once
    if (cudaMemcpyAsync(stage + page_bytes, table, table_bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) {
        ytk::set_error("%s: page table upload failed", who);
        return YTK_ERR;
    }
    if (ytk::launch_preprocess_table(src, reinterpret_cast<const ytk::RtSrc*>(stage + page_bytes), n_pages, Hn, Wn,
                                     e->input, st)) {
        ytk::set_error("%s: preprocess launch failed", who);
        return YTK_ERR;
    }
    return finish_forward(h, e, prob_out, out_on_device, st);
}

int ytk_dbnet_forward_f32(ytk_dbnet* h, const float* x, int x_on_device, int n, int H, int W, float* prob_out,
                          int out_on_device, void* cuda_stream) {
    std::lock_guard<std::mutex> lk(h->mu);
    DevGuard dev_guard(h->device);  // host threads start on device 0: the handle's device is the one that counts
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    ytk::DbnetEngine* e = get_engine(h, n, H, W);
    if (!e) return YTK_ERR;
    order_after_previous(h, st);
    const float* src = x;
    if (!x_on_device) {
        const size_t bytes = (size_t)n * 3 * H * W * 4;
        if (ensure_stage(h, bytes)) return YTK_ERR;
        if (cudaMemcpyAsync(h->stage, x, bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) {
            ytk::set_error("H2D copy of input tensor failed");
            return YTK_ERR;
        }
        src = reinterpret_cast<const float*>(h->stage);
    }
    if (ytk::launch_pack_nchw_f32(src, n, H, W, e->input, st)) {
        ytk::set_error("input pack launch failed");
        return YTK_ERR;
    }
    return finish_forward(h, e, prob_out, out_on_device, st);
}

double ytk_dbnet_flops(ytk_dbnet* h, int n_pages, int Hn, int Wn) {
    std::lock_guard<std::mutex> lk(h->mu);
    DevGuard dev_guard(h->device);  // host threads start on device 0: the handle's device is the one that counts
    ytk::DbnetEngine* e = get_engine(h, n_pages, Hn, Wn);
    return e ? e->flops : -1.0;
}

int ytk_dbnet_debug_tensor(ytk_dbnet* h, int n_pages, int Hn, int Wn, const char* name, float* host_out,
                           long long capacity, int* shape4) {
    std::lock_guard<std::mutex> lk(h->mu);
    DevGuard dev_guard(h->device);  // host threads start on device 0: the handle's device is the one that counts
    ytk::DbnetEngine* e = get_engine(h, n_pages, Hn, Wn);
    if (!e) return YTK_ERR;
    auto it = e->dbg.find(name);
    if (it == e->dbg.end() || !it->second.p) {
        ytk::set_error("no debug tensor named '%s'", name);
        return YTK_ERR;
    }
    const ytk::DebugTensor& t = it->second;
    const long long n = (long long)t.n * t.h * t.w * t.c;
    shape4[0] = t.n; shape4[1] = t.h; shape4[2] = t.w; shape4[3] = t.c;
    if (n > capacity) {
        ytk::set_error("debug tensor '%s' needs %lld floats, capacity %lld", name, n, capacity);
        return YTK_ERR;
    }
    cudaDeviceSynchronize();
    if (t.f32) {
        if (cudaMemcpy(host_out, t.p, n * 4, cudaMemcpyDeviceToHost) != cudaSuccess) return YTK_ERR;
    } else {
        float* tmp = nullptr;
        if (cudaMalloc(&tmp, n * 4) != cudaSuccess) return YTK_ERR;
        ytk::launch_op_to_f32(t.p, tmp, n, 0);
        cudaError_t err = cudaMemcpy(host_out, tmp, n * 4, cudaMemcpyDeviceToHost);
        cudaFree(tmp);
        if (err != cudaSuccess) return YTK_ERR;
    }
    return YTK_OK;
}

static_assert(sizeof(ytk_crop_geom) == sizeof(ytk::CropGeom), "ytk_crop_geom and ytk::CropGeom must have one layout");

int ytk_extract_crops_u8(const uint8_t* pages_dev, int n_pages, int H0, int W0, const ytk_crop_geom* geoms, int n_crops,
                         uint8_t* scratch_dev, long long scratch_bytes, uint8_t* canvases_dev, long long canvases_bytes,
                         void* cuda_stream) {
    if (n_crops == 0) return YTK_OK;
    if (!pages_dev || !geoms || !scratch_dev || !canvases_dev || n_pages <= 0 || H0 <= 0 || W0 <= 0 || n_crops < 0) {
        ytk::set_error("ytk_extract_crops_u8: null or empty argument");
        return YTK_ERR;
    }
    long long roi_end = 0;
    for (int i = 0; i < n_crops; ++i) {
        const ytk_crop_geom& g = geoms[i];
        const long long sw = (g.rot & 1) ? g.h : g.w, sh = (g.rot & 1) ? g.w : g.h;
        const bool ok = g.page >= 0 && g.page < n_pages && g.x0 >= 0 && g.y0 >= 0 && g.rw >= 1 && g.rh >= 1 &&
                        (long long)g.x0 + g.rw <= W0 && (long long)g.y0 + g.rh <= H0 && g.w >= 1 && g.h >= 1 &&
                        g.rot >= 0 && g.rot <= 3 && g.cw >= 1 && g.ch >= 1 && g.cw <= sw && g.ch <= sh &&
                        g.cw <= g.canvas_w && g.ch <= g.canvas_h && g.roi_off >= 0 &&
                        g.roi_off + (long long)g.w * g.h * 3 <= scratch_bytes && g.pix_off >= 0 &&
                        g.pix_off + (long long)g.canvas_w * g.canvas_h * 3 <= canvases_bytes;
        if (!ok) {
            ytk::set_error("ytk_extract_crops_u8: inconsistent crop record %d (page %d, roi %d,%d %dx%d, out %dx%d rot %d, "
                           "content %dx%d, canvas %dx%d)", i, g.page, g.x0, g.y0, g.rw, g.rh, g.w, g.h, g.rot, g.cw,
                           g.ch, g.canvas_w, g.canvas_h);
            return YTK_ERR;
        }
        roi_end = std::max(roi_end, g.roi_off + (long long)g.w * g.h * 3);
    }
    // the records are staged in the caller's scratch buffer, 16-byte aligned after the ROIs: no allocation here
    const long long rec_off = (roi_end + 15) / 16 * 16;
    const long long rec_bytes = (long long)n_crops * (long long)sizeof(ytk::CropGeom);
    if (rec_off + rec_bytes > scratch_bytes) {
        ytk::set_error("ytk_extract_crops_u8: scratch_dev holds %lld bytes, need %lld (ROIs) + %lld (records)", scratch_bytes,
                       rec_off, rec_bytes);
        return YTK_ERR;
    }
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, pages_dev) != cudaSuccess || attr.type != cudaMemoryTypeDevice) {
        cudaGetLastError();
        ytk::set_error("ytk_extract_crops_u8: pages_dev is not a device pointer");
        return YTK_ERR;
    }
    DevGuard dev_guard(attr.device);  // host threads start on device 0: the device that owns the pages is the one that counts
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    ytk::CropGeom* dev = reinterpret_cast<ytk::CropGeom*>(scratch_dev + rec_off);
    cudaError_t err = cudaMemcpyAsync(dev, geoms, (size_t)rec_bytes, cudaMemcpyHostToDevice, st);
    if (err != cudaSuccess) {
        ytk::set_error("ytk_extract_crops_u8: record upload failed: %s", cudaGetErrorString(err));
        return YTK_ERR;
    }
    if (ytk::launch_extract_crops(pages_dev, H0, W0, dev, n_crops, scratch_dev, canvases_dev, st)) {
        ytk::set_error("ytk_extract_crops_u8: kernel launch failed");
        return YTK_ERR;
    }
    return YTK_OK;
}

int ytk_extract_crops_table_u8(const uint8_t* pages_dev, long long pages_bytes, const ytk_page* table, int n_pages,
                               const ytk_crop_geom* geoms, int n_crops, uint8_t* scratch_dev, long long scratch_bytes,
                               uint8_t* canvases_dev, long long canvases_bytes, void* cuda_stream) {
    const char* who = "ytk_extract_crops_table_u8";
    if (n_crops == 0) return YTK_OK;
    if (!pages_dev || !geoms || !scratch_dev || !canvases_dev || n_crops < 0) {
        ytk::set_error("%s: null or empty argument", who);
        return YTK_ERR;
    }
    if (check_page_table(table, n_pages, pages_bytes, false, who)) return YTK_ERR;
    long long roi_end = 0;
    for (int i = 0; i < n_crops; ++i) {
        const ytk_crop_geom& g = geoms[i];
        const long long sw = (g.rot & 1) ? g.h : g.w, sh = (g.rot & 1) ? g.w : g.h;
        // the ROI lies inside the crop's own page
        const bool in_page = g.page >= 0 && g.page < n_pages && (long long)g.x0 + g.rw <= table[g.page].W &&
                             (long long)g.y0 + g.rh <= table[g.page].H;
        const bool ok = in_page && g.x0 >= 0 && g.y0 >= 0 && g.rw >= 1 && g.rh >= 1 && g.w >= 1 && g.h >= 1 &&
                        g.rot >= 0 && g.rot <= 3 && g.cw >= 1 && g.ch >= 1 && g.cw <= sw && g.ch <= sh &&
                        g.cw <= g.canvas_w && g.ch <= g.canvas_h && g.roi_off >= 0 &&
                        g.roi_off + (long long)g.w * g.h * 3 <= scratch_bytes && g.pix_off >= 0 &&
                        g.pix_off + (long long)g.canvas_w * g.canvas_h * 3 <= canvases_bytes;
        if (!ok) {
            ytk::set_error("%s: inconsistent crop record %d (page %d of %d, roi %d,%d %dx%d, out %dx%d rot %d, content "
                           "%dx%d, canvas %dx%d)", who, i, g.page, n_pages, g.x0, g.y0, g.rw, g.rh, g.w, g.h, g.rot, g.cw,
                           g.ch, g.canvas_w, g.canvas_h);
            return YTK_ERR;
        }
        roi_end = std::max(roi_end, g.roi_off + (long long)g.w * g.h * 3);
    }
    // records and page table are staged in the caller's scratch buffer, 16-byte aligned after the ROIs, with ONE copy
    const long long rec_off = (roi_end + 15) / 16 * 16;
    const long long rec_bytes = (long long)n_crops * (long long)sizeof(ytk::CropGeom);
    const long long tab_bytes = (long long)n_pages * (long long)sizeof(ytk_page);
    if (rec_off + rec_bytes + tab_bytes > scratch_bytes) {
        ytk::set_error("%s: scratch_dev holds %lld bytes, need %lld (ROIs) + %lld (records) + %lld (page table)", who,
                       scratch_bytes, rec_off, rec_bytes, tab_bytes);
        return YTK_ERR;
    }
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, pages_dev) != cudaSuccess || attr.type != cudaMemoryTypeDevice) {
        cudaGetLastError();
        ytk::set_error("%s: pages_dev is not a device pointer", who);
        return YTK_ERR;
    }
    DevGuard dev_guard(attr.device);
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    std::vector<uint8_t> blob((size_t)(rec_bytes + tab_bytes));
    memcpy(blob.data(), geoms, (size_t)rec_bytes);
    memcpy(blob.data() + rec_bytes, table, (size_t)tab_bytes);
    cudaError_t err = cudaMemcpyAsync(scratch_dev + rec_off, blob.data(), blob.size(), cudaMemcpyHostToDevice, st);
    if (err != cudaSuccess) {
        ytk::set_error("%s: record upload failed: %s", who, cudaGetErrorString(err));
        return YTK_ERR;
    }
    const ytk::CropGeom* dev = reinterpret_cast<const ytk::CropGeom*>(scratch_dev + rec_off);
    const ytk::RtSrc* tab = reinterpret_cast<const ytk::RtSrc*>(scratch_dev + rec_off + rec_bytes);
    if (ytk::launch_extract_crops_table(pages_dev, tab, dev, n_crops, scratch_dev, canvases_dev, st)) {
        ytk::set_error("%s: kernel launch failed", who);
        return YTK_ERR;
    }
    return YTK_OK;
}

int ytk_halve_pages_u8(const uint8_t* src_dev, int n_pages, int H, int W, uint8_t* dst_dev, int dH, int dW,
                       void* cuda_stream) {
    // cv2.resize(..., fx=0.5, fy=0.5): dsize = (cvRound(W * 0.5), cvRound(H * 0.5)), round half to even
    const int eh = (int)nearbyint(H * 0.5), ew = (int)nearbyint(W * 0.5);
    if (!src_dev || !dst_dev || n_pages <= 0 || H <= 0 || W <= 0 || dH != eh || dW != ew || dH < 1 || dW < 1) {
        ytk::set_error("ytk_halve_pages_u8: bad arguments (%d pages %dx%d -> %dx%d, expected %dx%d)", n_pages, H, W, dH, dW,
                       eh, ew);
        return YTK_ERR;
    }
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, src_dev) != cudaSuccess || attr.type != cudaMemoryTypeDevice) {
        cudaGetLastError();
        ytk::set_error("ytk_halve_pages_u8: src_dev is not a device pointer");
        return YTK_ERR;
    }
    DevGuard dev_guard(attr.device);
    if (ytk::launch_halve_pages(src_dev, n_pages, H, W, dst_dev, dH, dW, static_cast<cudaStream_t>(cuda_stream))) {
        ytk::set_error("ytk_halve_pages_u8: kernel launch failed");
        return YTK_ERR;
    }
    return YTK_OK;
}

int ytk_halve_pages_table_u8(const uint8_t* src_dev, long long src_bytes, const ytk_page* src_table, int n_pages,
                             uint8_t* dst_dev, long long dst_bytes, const ytk_page* dst_table, uint8_t* scratch_dev,
                             long long scratch_bytes, void* cuda_stream) {
    const char* who = "ytk_halve_pages_table_u8";
    if (!src_dev || !dst_dev || !scratch_dev) {
        ytk::set_error("%s: null argument", who);
        return YTK_ERR;
    }
    if (check_page_table(src_table, n_pages, src_bytes, true, who) ||
        check_page_table(dst_table, n_pages, dst_bytes, true, who))
        return YTK_ERR;
    long long max_pixels = 0;
    for (int i = 0; i < n_pages; ++i) {
        const int eh = (int)nearbyint(src_table[i].H * 0.5), ew = (int)nearbyint(src_table[i].W * 0.5);
        if (dst_table[i].H != eh || dst_table[i].W != ew) {
            ytk::set_error("%s: page %d %dx%d -> %dx%d, expected %dx%d", who, i, src_table[i].H, src_table[i].W,
                           dst_table[i].H, dst_table[i].W, eh, ew);
            return YTK_ERR;
        }
        max_pixels = std::max(max_pixels, (long long)eh * ew);
    }
    const long long tab_bytes = (long long)n_pages * (long long)sizeof(ytk_page);
    if (scratch_bytes < 2 * tab_bytes) {
        ytk::set_error("%s: scratch_dev holds %lld bytes, need %lld (two page tables)", who, scratch_bytes, 2 * tab_bytes);
        return YTK_ERR;
    }
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, src_dev) != cudaSuccess || attr.type != cudaMemoryTypeDevice) {
        cudaGetLastError();
        ytk::set_error("%s: src_dev is not a device pointer", who);
        return YTK_ERR;
    }
    DevGuard dev_guard(attr.device);
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    std::vector<uint8_t> blob((size_t)(2 * tab_bytes));
    memcpy(blob.data(), src_table, (size_t)tab_bytes);
    memcpy(blob.data() + tab_bytes, dst_table, (size_t)tab_bytes);
    cudaError_t err = cudaMemcpyAsync(scratch_dev, blob.data(), blob.size(), cudaMemcpyHostToDevice, st);
    if (err != cudaSuccess) {
        ytk::set_error("%s: page table upload failed: %s", who, cudaGetErrorString(err));
        return YTK_ERR;
    }
    const ytk::RtSrc* tabs = reinterpret_cast<const ytk::RtSrc*>(scratch_dev);
    if (ytk::launch_halve_pages_table(src_dev, tabs, n_pages, dst_dev, tabs + n_pages, max_pixels, st)) {
        ytk::set_error("%s: kernel launch failed", who);
        return YTK_ERR;
    }
    return YTK_OK;
}

int ytk_parseq_create(const ytk_tensor* tensors, int n_tensors, const ytk_parseq_cfg* cfg, ytk_parseq** out) {
    if (!tensors || !cfg || !out) {
        ytk::set_error("ytk_parseq_create: null argument");
        return YTK_ERR;
    }
    ytk::WeightSet ws;
    for (int i = 0; i < n_tensors; ++i) {
        ytk::TensorView v;
        v.data = tensors[i].data;
        v.ndim = tensors[i].ndim;
        for (int d = 0; d < 4; ++d) v.shape[d] = d < v.ndim ? tensors[i].shape[d] : 1;
        ws.map[tensors[i].name] = v;
    }
    ytk::ParseqCfg c{cfg->embed_dim, cfg->enc_heads, cfg->enc_depth, cfg->patch_h, cfg->patch_w, cfg->img_h,
                     cfg->img_w, cfg->num_tokens, cfg->max_label_length, cfg->dec_heads, cfg->mlp_ratio,
                     cfg->dec_mlp_ratio, cfg->refine_iters, cfg->repetition_stop, cfg->rep_period_max,
                     cfg->rep_min_run_p1, cfg->rep_min_repeats, cfg->decode_ar};
    auto h = std::make_unique<ytk_parseq>();
    cudaGetDevice(&h->device);
    if (h->model.load(ws, c)) return YTK_ERR;
    h->engine.m = &h->model;
    *out = h.release();
    return YTK_OK;
}

void ytk_parseq_destroy(ytk_parseq* h) { delete h; }

void ytk_parseq_set_refine_iters(ytk_parseq* h, int refine_iters) {
    std::lock_guard<std::mutex> lk(h->mu);
    DevGuard dev_guard(h->device);  // host threads start on device 0: the handle's device is the one that counts
    h->model.cfg.refine_iters = refine_iters;
}

int ytk_parseq_forward_crops(ytk_parseq* h, const uint8_t* crops_ptr, int crops_on_device, long long crops_bytes,
                             const ytk_crop* crops, int n_crops, int n_groups, int32_t* ids_out, float* probs_out,
                             int32_t* group_len_out, void* cuda_stream) {
    std::lock_guard<std::mutex> lk(h->mu);
    DevGuard dev_guard(h->device);  // host threads start on device 0: the handle's device is the one that counts
    ytk::ParseqBatch b;
    b.crops = crops_ptr;
    b.crops_on_device = crops_on_device;
    b.crops_bytes = crops_bytes;
    b.ngroups = n_groups;
    b.descs.resize(n_crops);
    const int gh = h->model.gh, pw = h->model.cfg.pw;
    for (int i = 0; i < n_crops; ++i) {
        const ytk_crop& c = crops[i];
        if (c.wp % pw != 0 || c.wp < c.w || c.ntok != gh * (c.wp / pw) || c.group < 0 || c.group >= n_groups ||
            c.wp > h->model.cfg.img_w) {
            ytk::set_error("ytk_parseq_forward_crops: inconsistent crop descriptor %d (w=%d wp=%d ntok=%d group=%d)", i,
                           c.w, c.wp, c.ntok, c.group);
            return YTK_ERR;
        }
        b.descs[i] = ytk::CropDesc{c.pix_off, c.w, c.wp, c.tok_off, c.ntok, c.group};
    }
    return h->engine.forward(b, ids_out, probs_out, group_len_out, nullptr, 0, nullptr,
                             static_cast<cudaStream_t>(cuda_stream))
               ? YTK_ERR
               : YTK_OK;
}

int ytk_parseq_forward_f32(ytk_parseq* h, const float* images, int images_on_device, int B, int W, float* logits_out,
                           int logits_on_device, int32_t* ids_out, float* probs_out, int32_t* steps_out,
                           int32_t* rep_cut_out, float* memory_out, void* cuda_stream) {
    std::lock_guard<std::mutex> lk(h->mu);
    DevGuard dev_guard(h->device);  // host threads start on device 0: the handle's device is the one that counts
    const int pw = h->model.cfg.pw, gh = h->model.gh;
    if (W % pw != 0 || W > h->model.cfg.img_w || W <= 0) {
        ytk::set_error("ytk_parseq_forward_f32: width %d must be a positive multiple of %d and <= %d", W, pw,
                       h->model.cfg.img_w);
        return YTK_ERR;
    }
    ytk::ParseqBatch b;
    b.images_f32 = images;
    b.images_on_device = images_on_device;
    b.image_w = W;
    b.crops_bytes = images_on_device ? 0 : (long long)B * 3 * 32 * W * 4;
    b.ngroups = 1;
    b.descs.resize(B);
    const int ntok = gh * (W / pw);
    for (int i = 0; i < B; ++i) b.descs[i] = ytk::CropDesc{0, W, W, i * ntok, ntok, 0};
    int glen = 0;
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    if (h->engine.forward(b, ids_out, probs_out, &glen, logits_out, logits_on_device, memory_out, st)) return YTK_ERR;
    if (steps_out) *steps_out = glen;
    if (rep_cut_out) {
        if (cudaMemcpy(rep_cut_out, h->engine.ar.rep_cut, sizeof(int) * B, cudaMemcpyDeviceToHost) != cudaSuccess) {
            ytk::set_error("rep_cut copy failed");
            return YTK_ERR;
        }
    }
    return YTK_OK;
}

double ytk_parseq_last_flops(ytk_parseq* h) { return h->engine.flops; }
int ytk_parseq_last_steps(ytk_parseq* h) { return h->engine.last_steps; }
void ytk_parseq_last_phase_ms(ytk_parseq* h, float* ms4) {
    for (int i = 0; i < 4; ++i) ms4[i] = h->engine.phase_ms[i];
}

}  // extern "C"


// ------------------------------------------------------------------------------------------------ RT-DETRv2
struct ytk_rtdetr {
    ytk::RtdetrModel model;
    std::map<int, std::unique_ptr<ytk::RtdetrEngine>> engines;   // per batch size
    std::mutex mu;
    int device = 0;
    cudaEvent_t last_done = nullptr;   // buffers of an engine are shared by all calls: order them (see ytk_dbnet)
    // ytk_rtdetr_forward_u8: device copy of host pages, and the resize scratch (records, coefficients, intermediates)
    uint8_t* pages = nullptr;
    size_t pages_cap = 0;
    uint8_t* scratch = nullptr;
    size_t scratch_cap = 0;
};

// Grows a handle-owned buffer; the previous call may still be reading the old one.
static int rt_reserve(ytk_rtdetr* h, uint8_t** buf, size_t* cap, size_t bytes, const char* what) {
    if (*cap >= bytes) return 0;
    if (h->last_done) cudaEventSynchronize(h->last_done);
    if (*buf) cudaFree(*buf);
    *buf = nullptr;
    *cap = 0;
    if (cudaMalloc(buf, bytes) != cudaSuccess) {
        *buf = nullptr;
        ytk::set_error("cudaMalloc(%zu) for the %s failed", bytes, what);
        return 1;
    }
    *cap = bytes;
    return 0;
}

// Runs the engine on its packed input and copies the outputs (the common tail of both forward entries).
static int rt_finish(ytk_rtdetr* h, ytk::RtdetrEngine* e, int n, float* pred_logits, float* pred_boxes, int out_on_device,
                     cudaStream_t st) {
    if (e->run(st)) return YTK_ERR;
    const int K = h->model.cfg.num_queries, C = h->model.cfg.num_classes;
    const cudaMemcpyKind kind = out_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    cudaError_t err = cudaMemcpyAsync(pred_logits, e->out_logits, (size_t)n * K * C * 4, kind, st);
    if (err == cudaSuccess) err = cudaMemcpyAsync(pred_boxes, e->boxes, (size_t)n * K * 16, kind, st);
    if (!h->last_done) cudaEventCreateWithFlags(&h->last_done, cudaEventDisableTiming);
    if (h->last_done) cudaEventRecord(h->last_done, st);
    if (err == cudaSuccess && !out_on_device) err = cudaStreamSynchronize(st);
    if (err != cudaSuccess) {
        ytk::set_error("RT-DETRv2 output copy failed: %s", cudaGetErrorString(err));
        return YTK_ERR;
    }
    return YTK_OK;
}

static ytk::RtdetrEngine* rt_engine(ytk_rtdetr* h, int n) {
    auto it = h->engines.find(n);
    if (it != h->engines.end()) return it->second.get();
    if (h->engines.size() >= 4) {
        cudaDeviceSynchronize();
        h->engines.erase(h->engines.begin());
    }
    auto e = std::make_unique<ytk::RtdetrEngine>();
    if (e->build(h->model, n)) return nullptr;
    ytk::RtdetrEngine* p = e.get();
    h->engines[n] = std::move(e);
    return p;
}

int ytk_rtdetr_create(const ytk_tensor* tensors, int n_tensors, int num_classes, int num_queries, int img_size,
                      ytk_rtdetr** out) {
    if (!tensors || !out) {
        ytk::set_error("ytk_rtdetr_create: null argument");
        return YTK_ERR;
    }
    ytk::WeightSet ws;
    for (int i = 0; i < n_tensors; ++i) {
        ytk::TensorView v;
        v.data = tensors[i].data;
        v.ndim = tensors[i].ndim;
        for (int d = 0; d < 4; ++d) v.shape[d] = d < v.ndim ? tensors[i].shape[d] : 1;
        ws.map[tensors[i].name] = v;
    }
    auto h = std::make_unique<ytk_rtdetr>();
    cudaGetDevice(&h->device);
    ytk::RtCfg cfg;
    cfg.num_classes = num_classes;
    cfg.num_queries = num_queries;
    cfg.img = img_size;
    if (num_classes < 1 || num_classes > 8 || num_queries < 1) {
        ytk::set_error("ytk_rtdetr_create: num_classes %d (1..8) / num_queries %d unsupported", num_classes, num_queries);
        return YTK_ERR;
    }
    if (h->model.load(ws, cfg)) return YTK_ERR;
    *out = h.release();
    return YTK_OK;
}

void ytk_rtdetr_destroy(ytk_rtdetr* h) {
    if (!h) return;
    DevGuard dev_guard(h->device);
    if (h->last_done) {
        cudaEventSynchronize(h->last_done);
        cudaEventDestroy(h->last_done);
    }
    cudaDeviceSynchronize();
    if (h->pages) cudaFree(h->pages);
    if (h->scratch) cudaFree(h->scratch);
    delete h;
}

int ytk_rtdetr_device(const ytk_rtdetr* h) { return h ? h->device : -1; }

int ytk_rtdetr_forward_f32(ytk_rtdetr* h, const float* x, int x_on_device, int n, float* pred_logits, float* pred_boxes,
                           int out_on_device, void* cuda_stream) {
    if (!h || !x || !pred_logits || !pred_boxes || n < 1) {
        ytk::set_error("ytk_rtdetr_forward_f32: null or empty argument");
        return YTK_ERR;
    }
    std::lock_guard<std::mutex> lk(h->mu);
    DevGuard dev_guard(h->device);
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    ytk::RtdetrEngine* e = rt_engine(h, n);
    if (!e) return YTK_ERR;
    if (h->last_done) cudaStreamWaitEvent(st, h->last_done, 0);
    const int S = h->model.cfg.img;
    const float* src = x;
    if (!x_on_device) {
        if (cudaMemcpyAsync(e->in_f32, x, (size_t)n * 3 * S * S * 4, cudaMemcpyHostToDevice, st) != cudaSuccess) {
            ytk::set_error("H2D copy of the input tensor failed");
            return YTK_ERR;
        }
        src = e->in_f32;
    }
    if (ytk::launch_rt_pack_input(src, n, S, S, e->input, st)) return YTK_ERR;
    return rt_finish(h, e, n, pred_logits, pred_boxes, out_on_device, st);
}

static_assert(sizeof(ytk_rtdetr_src) == sizeof(ytk::RtSrc), "ytk_rtdetr_src and ytk::RtSrc must have one layout");

int ytk_rtdetr_forward_u8(ytk_rtdetr* h, const uint8_t* pages, int pages_on_device, long long pages_bytes,
                          const ytk_rtdetr_src* srcs, int n, float* pred_logits, float* pred_boxes, int out_on_device,
                          void* cuda_stream) {
    if (!h || !pages || !srcs || !pred_logits || !pred_boxes || n < 1 || pages_bytes < 1) {
        ytk::set_error("ytk_rtdetr_forward_u8: null or empty argument");
        return YTK_ERR;
    }
    std::lock_guard<std::mutex> lk(h->mu);
    DevGuard dev_guard(h->device);
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    ytk::ResampleJob job;
    if (ytk::resample_prepare(reinterpret_cast<const ytk::RtSrc*>(srcs), n, h->model.cfg.img, pages_bytes,
                              "ytk_rtdetr_forward_u8", &job))
        return YTK_ERR;
    ytk::RtdetrEngine* e = rt_engine(h, n);
    if (!e) return YTK_ERR;
    if (!pages_on_device && rt_reserve(h, &h->pages, &h->pages_cap, (size_t)pages_bytes, "page staging buffer"))
        return YTK_ERR;
    if (rt_reserve(h, &h->scratch, &h->scratch_cap, (size_t)job.bytes, "resize scratch")) return YTK_ERR;
    if (h->last_done) cudaStreamWaitEvent(st, h->last_done, 0);
    const uint8_t* src = pages;
    if (!pages_on_device) {
        cudaError_t err = cudaMemcpyAsync(h->pages, pages, (size_t)pages_bytes, cudaMemcpyHostToDevice, st);
        if (err != cudaSuccess) {
            ytk::set_error("H2D copy of the pages failed: %s", cudaGetErrorString(err));
            return YTK_ERR;
        }
        src = h->pages;
    }
    if (ytk::launch_resample(src, job, h->scratch, e->input, 1, st)) return YTK_ERR;
    return rt_finish(h, e, n, pred_logits, pred_boxes, out_on_device, st);
}

long long ytk_op_resize_bilinear_scratch_bytes(const ytk_rtdetr_src* srcs, int n, int size) {
    ytk::ResampleJob job;
    if (ytk::resample_prepare(reinterpret_cast<const ytk::RtSrc*>(srcs), n, size, LLONG_MAX,
                              "ytk_op_resize_bilinear_scratch_bytes", &job))
        return -1;
    return job.bytes;
}

int ytk_op_resize_bilinear_u8(const uint8_t* pages_dev, long long pages_bytes, const ytk_rtdetr_src* srcs, int n,
                              int size, uint8_t* scratch_dev, long long scratch_bytes, uint8_t* out_rgb_dev,
                              void* cuda_stream) {
    if (!pages_dev || !srcs || !scratch_dev || !out_rgb_dev) {
        ytk::set_error("ytk_op_resize_bilinear_u8: null argument");
        return YTK_ERR;
    }
    ytk::ResampleJob job;
    if (ytk::resample_prepare(reinterpret_cast<const ytk::RtSrc*>(srcs), n, size, pages_bytes,
                              "ytk_op_resize_bilinear_u8", &job))
        return YTK_ERR;
    if (scratch_bytes < job.bytes) {
        ytk::set_error("ytk_op_resize_bilinear_u8: scratch_dev holds %lld bytes, need %lld", scratch_bytes, job.bytes);
        return YTK_ERR;
    }
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, pages_dev) != cudaSuccess || attr.type != cudaMemoryTypeDevice) {
        cudaGetLastError();
        ytk::set_error("ytk_op_resize_bilinear_u8: pages_dev is not a device pointer");
        return YTK_ERR;
    }
    DevGuard dev_guard(attr.device);
    return ytk::launch_resample(pages_dev, job, scratch_dev, out_rgb_dev, 0, static_cast<cudaStream_t>(cuda_stream))
               ? YTK_ERR
               : YTK_OK;
}

double ytk_rtdetr_flops(ytk_rtdetr* h, int n) {
    std::lock_guard<std::mutex> lk(h->mu);
    DevGuard dev_guard(h->device);
    ytk::RtdetrEngine* e = rt_engine(h, n);
    return e ? e->flops : -1.0;
}

int ytk_rtdetr_debug_tensor(ytk_rtdetr* h, int n, const char* name, float* host_out, long long capacity, int* shape4) {
    std::lock_guard<std::mutex> lk(h->mu);
    DevGuard dev_guard(h->device);
    ytk::RtdetrEngine* e = rt_engine(h, n);
    if (!e) return YTK_ERR;
    auto it = e->dbg.find(name);
    if (it == e->dbg.end() || !it->second.p) {
        ytk::set_error("no debug tensor named '%s'", name);
        return YTK_ERR;
    }
    const ytk::DebugTensor& t = it->second;
    const long long cnt = (long long)t.n * t.h * t.w * t.c;
    shape4[0] = t.n; shape4[1] = t.h; shape4[2] = t.w; shape4[3] = t.c;
    if (cnt > capacity) {
        ytk::set_error("debug tensor '%s' needs %lld floats, capacity %lld", name, cnt, capacity);
        return YTK_ERR;
    }
    cudaDeviceSynchronize();
    if (t.f32) {
        if (cudaMemcpy(host_out, t.p, cnt * 4, cudaMemcpyDeviceToHost) != cudaSuccess) return YTK_ERR;
    } else {
        float* tmp = nullptr;
        if (cudaMalloc(&tmp, cnt * 4) != cudaSuccess) return YTK_ERR;
        ytk::launch_op_to_f32(t.p, tmp, cnt, 0);
        cudaError_t err = cudaMemcpy(host_out, tmp, cnt * 4, cudaMemcpyDeviceToHost);
        cudaFree(tmp);
        if (err != cudaSuccess) return YTK_ERR;
    }
    return YTK_OK;
}
