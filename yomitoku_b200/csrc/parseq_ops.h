// Launchers of the non-GEMM PARSeq kernels (parseq_ops.cu).  All return 0 on success.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ytk {

// One crop ("sequence") of the packed recognizer batch.
struct CropDesc {
    long long pix_off;  // byte offset of the crop's u8 RGB canvas [32][w][3] in the packed crop buffer
    int w;              // canvas width actually stored
    int wp;             // padded width the reference batch gave this crop (>= w, multiple of patch width)
    int tok_off;        // first token row of this crop in the packed token matrices
    int ntok;           // gh * (wp / pw)
    int group;          // reference mini-batch id (AR early-stop semantics)
};

// Patchify: packed u8 crops -> A matrix [T, Kpad] bf16 (K order c,py,px = flattened conv weight [D,3,ph,pw]) and the
// residual stream initialised with the cropped positional embedding x[t,:] = pos_embed[(gy*full_gw + gx), :].
int launch_patchify_u8(const uint8_t* crops, const CropDesc* descs, int ncrops, int ph, int pw, int Kpad,
                       const float* pos_embed, int full_gw, int D, void* A, float* x, int T, cudaStream_t st);
// Same from the model-level seam tensor (B,3,32,W) fp32 (every crop has the same width W).
int launch_patchify_f32(const float* images, int B, int W, int ph, int pw, int Kpad, const float* pos_embed,
                        int full_gw, int D, void* A, float* x, cudaStream_t st);

// LayerNorm over the last dim of fp32 rows -> bf16 (and optionally fp32) output.  If addvec != null the row first
// gets addvec[(row % period) + add_row0, :] added (and is written back to x when writeback != 0).
// d_real <= D: statistics run over the first d_real features, the rest is zero padding (ParseqModel::load).
int launch_layernorm(float* x, int M, int D, int d_real, const float* gamma, const float* beta, float eps,
                     void* out_bf16, float* out_f32, const float* addvec, int period, const int* add_row0_dev,
                     int add_row0, int writeback, cudaStream_t st);

// Flash attention over packed sequences, bf16 in/out, fp32 softmax; no mask.
struct SeqDesc {
    int q_off;         // first query row (rows of Q, stride ldq)
    int q_len;
    int o_off;         // first output row (rows of O, stride ldo)
    int k_len;         // number of keys
    long long k_base;  // element offset of key 0 inside K / V (key j at k_base + j * ldkv)
    int kpad;          // masked mode: keys >= kpad are padding
    int pad_;
};
// masked = 0: plain softmax(QK^T)V.  masked = 1: PARSeq refinement self-attention - key j is visible to query i iff
// (i < 2 || j <= i) && j < kpad (reference parseq.py:267-297; rows 0 and 1 of the causal mask are cleared).
// q_rows / kv_rows: number of rows of the Q and K/V matrices (TMA extents of the wgmma path, attn_tc.cu).
// impl: 0 = default (attn_tc_kernel: wgmma + TMA; YTK_ATTN=legacy selects the mma.sync kernel), 1 = legacy mma.sync
// kernel, 2 = wgmma kernel.
int launch_flash_attention(const void* Q, long long ldq, long long q_rows, const void* K, const void* V, long long ldkv,
                           long long kv_rows, void* O, long long ldo, const SeqDesc* seqs, int nseq, int max_q_len,
                           int heads, int head_dim, int masked, cudaStream_t st, int impl = 0);
int launch_attention_tc(const void* Q, long long ldq, long long q_rows, const void* K, const void* V, long long ldkv,
                        long long kv_rows, void* O, long long ldo, const SeqDesc* seqs, int nseq, int heads,
                        int head_dim, int masked, cudaStream_t st);

// Keys per (row, head) the single-query attention holds scores for (its shared-memory row): the most encoder tokens a
// crop may have, and the most AR positions.
constexpr int kMaxMem = 800;

// AR attention, one query per (row, head) (single_query_attn_kernel):
//  self : step i = *step_dev, q = q_shared[i], keys 0..i of the row's content K/V cache [row][S positions][2D] -> out[row]
//  cross: q = qc[row], keys = the row's encoder memory K/V (projected once)                                  -> out[row]
int launch_dec_self_attn(const void* q_shared, const void* ckv, int B, int S, int D, int heads, const int* step_dev,
                         void* out, cudaStream_t st);
int launch_dec_cross_attn(const void* qc, const void* memkv, const CropDesc* descs, int B, int D, int heads, void* out,
                          cudaStream_t st);

struct ArState {
    int* tgt;        // [B][S] AR context tokens (with forced EOS)
    int* raw;        // [B][S] raw arg-max per step
    int* rep_cut;    // [B] (-1 = none)
    int* rep_done;   // [B]
    int* has_eos;    // [B]
    int* group_len;  // [G] number of AR steps the group ran (0 = still running)
    int* n_active;   // [1] groups still running
    int* step;       // [1] current step i
    int* open_rows;  // [G] scratch: rows of the group that hold no EOS yet (zero between steps)
    int* ticket;     // [1] scratch: CTAs of ar_control that are done with the current step (zero between steps)
};
// Arg-max over the head logits + the reference's per-step control logic (parseq.py:220-250) + content embedding of
// the emitted token (text_embed * sqrt(D) + pos_queries[j-1]) normalised by LN_c -> cin bf16 [B, D].
// npart > 0: `logits` holds the float4 partials of the fused head epilogue (gemm_tc EPI_ROWMAX), ldl = partials per row.
int launch_ar_control(const float* logits, long long ldl, int C, int npart, int B, int S, const int* row_group, int g0,
                      int ngroups, ArState st_, int eos_id, int rep_on, int rep_period_max, int rep_min_run_p1, int rep_min_repeats,
                      const float* embed, const float* pos_q, int D, int d_real, const float* g_c, const float* b_c,
                      void* cin, cudaStream_t st);
// Content embeddings for the refinement pass: [B*S, D] bf16 = LN_c(content(row,pos)) from the raw tokens; also
// emits klen (= group_len[group]) and kpad (first EOS position in [BOS, raw...]) per row.
int launch_refine_embed(const int* raw, const int* row_group, const int* group_len, int B, int S, int bos_id, int eos_id,
                        const float* embed, const float* pos_q, int D, int d_real, const float* g_c, const float* b_c,
                        void* cin, int* klen, int* kpad, cudaStream_t st);

// Row-wise softmax statistics of logits: ids = argmax, probs = softmax max; applies the repetition logit patch
// (position == rep_cut[row] -> EOS with probability 1).
// Output index of local row r is r * g_stride + g_off (= crop * S + position).
int launch_softmax_max(const float* logits, long long ldl, int C, int rows, int S, long long g_stride, long long g_off,
                       const int* rep_cut, int eos_id, int* ids, float* probs, cudaStream_t st);
// launch_softmax_max from the partials of the fused head epilogue: partials float4 [rows][ldp], npart valid per row.
int launch_rowmax_finalize(const float* partials, long long ldp, int npart, int C, int rows, int S, long long g_stride,
                           long long g_off, const int* rep_cut, int eos_id, int* ids, float* probs, cudaStream_t st);
int launch_bcast_rows(const void* src, void* dst, int row_bytes, long long dst_stride_bytes, int rows,
                      cudaStream_t st);
int launch_apply_rep_cut(const int* rep_cut, int B, int S, int C, int eos_id, int* ids, float* probs, cudaStream_t st);

int launch_refine_seqs(const int* klen, const int* kpad, int B, int S, int D, SeqDesc* seqs, cudaStream_t st);
int launch_fill_i32(int* p, int v, long long n, cudaStream_t st);

}  // namespace ytk
