// PARSeq recognizer on device: model weights + execution engine.  See parseq_engine.cu.
#pragma once
#include <cuda_runtime.h>

#include <string>
#include <vector>

#include "dbnet_engine.h"  // TensorView / WeightSet
#include "gemm_tc.h"
#include "parseq_ops.h"

namespace ytk {

struct ParseqCfg {
    int D, enc_heads, enc_depth, ph, pw, img_h, img_w, num_tokens, max_label_length, dec_heads, mlp_ratio,
        dec_mlp_ratio, refine_iters, rep_on, rep_period_max, rep_min_run_p1, rep_min_repeats, decode_ar;
};

struct LinearW {
    void* w = nullptr;      // bf16 [N][K] (torch nn.Linear layout, K padded to a multiple of 64)
    float* b = nullptr;     // fp32 [N]
    int N = 0, K = 0;
};

struct LnW {
    float* g = nullptr;
    float* b = nullptr;
};

struct EncBlock {
    LnW ln1, ln2;
    LinearW qkv, proj, fc1, fc2;
};

struct ParseqModel {
    ParseqCfg cfg;  // cfg.D is the PADDED width every kernel works with; Dr the model's real embed_dim
    int Dr = 0;
    int S, C, gh, full_gw, Kpatch;
    LinearW patch;
    float* pos_embed = nullptr;  // fp32 [gh*full_gw, D]
    std::vector<EncBlock> blocks;
    LnW enc_norm, norm1, norm2, norm_c, dec_norm;
    LinearW self_kv, self_out, cross_q, cross_kv, cross_out, lin1, lin2, head;
    float* embed = nullptr;   // fp32 [num_tokens, D]
    float* pos_q = nullptr;   // fp32 [S, D]
    void* q_self = nullptr;   // bf16 [S, D]: self-attention query projection of LN_q(pos_queries) (row independent)
    void* ckv0 = nullptr;     // bf16 [2D]: content K/V of position 0 (= BOS, row independent)
    std::vector<void*> owned;
    int load(const WeightSet& ws, const ParseqCfg& cfg);
    ~ParseqModel();
};

// Host-side description of one recognizer call.
struct ParseqBatch {
    const uint8_t* crops = nullptr;   // packed u8 RGB canvases (host or device), or null when images_f32 is used
    int crops_on_device = 0;
    long long crops_bytes = 0;
    const float* images_f32 = nullptr;  // model-level seam: (B,3,32,W) fp32, host or device
    int images_on_device = 0;
    int image_w = 0;
    std::vector<CropDesc> descs;      // per crop
    int ngroups = 0;
};

struct ParseqEngine {
    const ParseqModel* m = nullptr;
    // capacities
    long long cap_tok = 0;
    int cap_rows = 0;
    long long cap_crop_bytes = 0;
    int cap_groups = 0;
    std::vector<void*> bufs;
    // encoder buffers
    uint8_t* crops_dev = nullptr;
    CropDesc* descs_dev = nullptr;
    SeqDesc* seqs_enc = nullptr;
    SeqDesc* seqs_ref = nullptr;
    SeqDesc* seqs_self = nullptr;
    void *A_patch = nullptr, *h = nullptr, *qkv = nullptr, *att = nullptr, *mlp = nullptr, *mem = nullptr,
         *memkv = nullptr;
    float* x = nullptr;
    // decoder buffers (R = rows * S)
    float *x1 = nullptr, *logits = nullptr;
    void *hb = nullptr, *qc = nullptr, *sa = nullptr, *oc = nullptr, *mlpb = nullptr, *cin = nullptr, *ckv = nullptr;
    int logits_rows = 0;
    long long ldl = 0;
    int *row_group = nullptr, *klen = nullptr, *kpad = nullptr, *ids = nullptr;
    int* glen_const = nullptr;  // [2][cap_groups]: context lengths S and 1 for the non-AR decoder passes
    float* probs = nullptr;
    ArState ar{};
    int* ar_block = nullptr;  // backing store of the ArState arrays
    size_t ar_block_ints = 0;
    int* host_flag = nullptr; // pinned: [n_active, step] per AR part
    cudaStream_t st2 = nullptr;  // second stream of the two-part AR loop
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    double flops = 0;         // algorithmic FLOPs of the last forward (GEMMs + attention)
    int last_steps = 0;
    cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};  // start, encoder, AR, refine, end
    float phase_ms[4] = {0, 0, 0, 0};  // encoder, AR decode, refinement, output copies of the last forward

    // Stage read-out for the tests (ytk_parseq_set_debug / ytk_parseq_debug_tensor).  With `debug` on, forward() copies
    // the stages it overwrites in place (the encoder residual stream after the patch GEMM and after every block, x1
    // after the self- and cross-attention sub-layers of the decoder pass, the context tokens of the last pass) into
    // the dbg_* buffers; nothing else changes.  `last` describes the last successful forward, so that a name it did not
    // produce is refused instead of returning stale data.
    int debug = 0;
    struct LastRun {
        bool valid = false, captured = false, ar = false, dec = false;
        long long T = 0;
        int B = 0, groups = 0;
    } last;
    float *dbg_encx = nullptr, *dbg_xself = nullptr, *dbg_xcross = nullptr;
    int* dbg_ctx = nullptr;
    size_t dbg_encx_bytes = 0, dbg_dec_bytes = 0, dbg_ctx_bytes = 0;
    struct View {
        const void* p = nullptr;
        long long rows = 0;
        int cols = 0;
        int kind = 0;  // 0: 16-bit GEMM operand type, 1: fp32, 2: int32
    };
    // The buffer behind a stage name of the last forward (or a model constant); 1 + set_error for an unknown name or
    // one the last forward did not produce.
    int debug_view(const std::string& name, View* out) const;

    int ensure(long long tok, int rows, long long crop_bytes, int groups);
    // Runs encoder + AR decode + refinement.  Outputs (host): ids [rows*S], probs [rows*S], group_len [ngroups];
    // logits_out (optional, host or device): [rows, S, C] fp32 when refine_iters > 0.
    int forward(const ParseqBatch& b, int* ids_out, float* probs_out, int* group_len_out, float* logits_out,
                int logits_on_device, float* memory_out, cudaStream_t st);
    int ensure_debug(long long T, long long R, int B);
    ~ParseqEngine();
};

}  // namespace ytk
