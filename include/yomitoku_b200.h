/*
 * yomitoku_b200 C ABI (libytk_b200.so) - the drop-in boundary for the DBNet -> PARSeq hot path.
 *
 * The reference (kotaro-kinoshita/yomitoku) has no FFI: its seam is the Python object protocol
 * `self.model(tensor)` inside TextDetector / TextRecognizer (reference src/yomitoku/text_detector.py:127-131,
 * src/yomitoku/text_recognizer.py:247-256, SURVEY.md section 8b).  These entry points are what a ctypes binding
 * behind those two call sites binds to; INTEGRATION.md shows the stub.  Plain pointers and sizes only, no torch
 * types; all device pointers are caller-owned; every call returns 0 on success and a nonzero code on failure, with a
 * human-readable message from ytk_last_error() (thread-local).  No exceptions cross this boundary.
 */
#ifndef YOMITOKU_B200_H
#define YOMITOKU_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YTK_OK 0
#define YTK_ERR 1

/* activation codes for the op-level entry points */
#define YTK_ACT_NONE 0
#define YTK_ACT_RELU 1
#define YTK_ACT_GELU 2
#define YTK_ACT_SIGMOID 3
#define YTK_ACT_SILU 4

const char* ytk_last_error(void);
int ytk_version(void);
/* number of kernel launches issued by this library on the calling process since load (bench.py gpu_launches) */
long long ytk_launch_count(void);
/* Measurement aid (bench.py roofline): between begin and end every gemm_tc_kernel launch is bracketed by CUDA events on
 * its own stream; end returns the summed algorithmic FLOPs, summed kernel durations (ms) and the launch count. */
void ytk_gemm_profile_begin(void);
int ytk_gemm_profile_end(double* flops, double* ms, long long* launches);

/* ---- op level (kernel parity tests; replaces the cuDNN/cuBLAS call sites listed in SURVEY.md section 2.3) ----
 * Convolution as wgmma implicit GEMM.  in: NHWC fp16 [N,H,W,in_ld] (first Cin channels used), w: fp16
 * [Cout][kh][kw][Cin], bias fp32 [Cout] or NULL, resid: [N,Ho,Wo,ldr] fp16/fp32 or NULL, out: [N,Ho,Wo,ldc]
 * fp16/fp32.  Replaces torch.nn.Conv2d + BatchNorm2d(eval, folded) + ReLU (+ residual add) of
 * torchvision ResNet-50 bottlenecks (reference models/dbnet_plus.py:30-38) and the decoder convs (:56-116).
 * mode 1 = ConvTranspose2d(kernel 2, stride 2) written as a GEMM with a pixel-shuffle epilogue (:111,:114). */
int ytk_op_conv2d_f16(const void* in, int N, int H, int W, int Cin, long long in_ld, const void* w, const float* bias,
                       int kh, int kw, int stride, int pad, int dil, int Cout, const void* resid, int resid_f32,
                       long long ldr, void* out, int out_f32, long long ldc, int act, int mode, void* cuda_stream);

/* Linear layer y = act(A W^T + b (+ resid)); A [M,lda] fp16, W [N,K] fp16 (torch nn.Linear layout), K % 64 == 0.
 * Replaces nn.Linear / timm Mlp / attention projections (reference models/layers/parseq_transformer.py:43-52,
 * models/parseq.py:72). */
int ytk_op_linear_f16(const void* A, long long lda, int M, int K, const void* W, int N, const float* bias,
                       const void* resid, int resid_f32, long long ldr, void* out, int out_f32, long long ldc, int act,
                       void* cuda_stream);

/* One descriptor per packed sequence of ytk_op_attention_f16 (the layout of ytk::SeqDesc, csrc/parseq_ops.h). */
typedef struct ytk_attn_seq {
    int32_t q_off;     /* first query row in Q */
    int32_t q_len;
    int32_t o_off;     /* first output row in O */
    int32_t k_len;     /* number of keys */
    long long k_base;  /* element offset of key 0 inside K / V (key j at k_base + j * ldkv; a multiple of ldkv) */
    int32_t kpad;      /* masked mode: keys >= kpad are padding */
    int32_t pad_;
} ytk_attn_seq;

/* softmax(Q K^T / sqrt(head_dim)) V per (sequence, head) over packed ragged sequences; Q [q_rows, ldq], K / V
 * [kv_rows, ldkv], O [*, ldo] fp16 on the device, head h = columns [h*head_dim, (h+1)*head_dim); seqs_dev: device array.
 * masked != 0: key j visible to query i iff (i < 2 || j <= i) && j < kpad (PARSeq refinement mask, reference
 * models/parseq.py:267-297).  impl: 0 default (wgmma kernel), 1 legacy mma.sync kernel, 2 wgmma kernel.
 * Replaces timm Attention's F.scaled_dot_product_attention (reference
 * models/layers/parseq_transformer.py:206-234) and nn.MultiheadAttention's core (parseq_transformer.py:83-92). */
int ytk_op_attention_f16(const void* Q, long long ldq, long long q_rows, const void* K, const void* V, long long ldkv,
                         long long kv_rows, void* O, long long ldo, const ytk_attn_seq* seqs_dev, int nseq, int max_q_len,
                         int heads, int head_dim, int masked, int impl, void* cuda_stream);

/* Query selection of the RT-DETRv2 decoder (torch.topk over the encoder scores, reference
 * models/layers/rtdetrv2_decoder.py:724-727).  scores_dev: [n, L] fp32 on the device; out_idx_dev: [n, K] int32 on the
 * device = per row the indices of the K largest scores, descending, equal scores in ascending index order (-0 sorts
 * below +0).  1 <= K <= L; L is bounded by shared memory (about 45k on an H100), a larger L is an error, not a launch.
 * Asynchronous on the stream. */
int ytk_op_topk_f32(const float* scores_dev, int n, int L, int K, int* out_idx_dev, void* cuda_stream);

/* Multi-scale deformable attention core of the RT-DETRv2 decoder (reference models/layers/rtdetrv2_decoder.py:306-388,
 * grid_sample bilinear, zero padding, align_corners=False), rows = n_img * K queries.  All pointers on the device:
 *   ow    fp32 [rows, ldo]: per row heads * P * 2 sampling offsets (x, y per point), then heads * P attention logits
 *   ref   fp32 [rows, 4]: reference boxes (cx, cy, w, h); sampling location = ref.xy + off / points[l] * ref.wh * offset_scale
 *   value fp16 level-major: level l of image i is rows [off[l] * n_img + i * h[l] * w[l], ...) with off = prefix sum of
 *         h * w; head hd reads columns [voff + hd * head_dim, ...) of rows with pitch ldv
 *   out   fp16 [rows, ldout]: columns [0, heads * head_dim) are written, nothing else
 * level_h / level_w / level_points: host arrays of n_levels (1..4) entries; head_dim 32 and 12 points per head in all.
 * Asynchronous on the stream; invalid arguments are an error, not a launch. */
int ytk_op_deform_attn_f16(const float* ow, long long ldo, const float* ref, const void* value, long long ldv, int voff,
                           const int* level_h, const int* level_w, const int* level_points, int n_levels, int n_img, int K,
                           int heads, int head_dim, float offset_scale, void* out, long long ldout, void* cuda_stream);

/* LayerNorm over the rows of x fp32 [M, D] (device).  If addvec != NULL every row first gets
 * addvec[(row % period) + r0, :] added, r0 = *add_row0_dev if that is non-NULL, else add_row0; writeback != 0 stores the
 * sum back to x.  Statistics run over the first d_real features (the rest is zero padding: zero in x, gamma, beta and
 * addvec).  Outputs, each optional: out_f16 [M, D] fp16, out_f32 [M, D] fp32.  D <= 1024, D and d_real multiples of 4,
 * 16-byte aligned fp32 pointers.  Asynchronous on the stream; invalid arguments are an error, not a launch. */
int ytk_op_layernorm_f32(float* x, int M, int D, int d_real, const float* gamma, const float* beta, float eps,
                         void* out_f16, float* out_f32, const float* addvec, int period, const int* add_row0_dev,
                         int add_row0, int writeback, void* cuda_stream);

/* ---- Device-side front half of the DBNet post-processing (reference postprocessor/dbnet_postporcessor.py:39-82:
 * binarize, findContours, and the pixel work of minAreaRect / box_score_fast).  One record per horizontal run of an
 * 8-connected component of (prob > thresh). ---- */
typedef struct ytk_db_run {
    int32_t root;  /* raster index of the component's first pixel: component id; OpenCV lists outer contours in
                      descending order of it */
    int32_t y;
    int32_t x0;    /* first column */
    int32_t x1;    /* last column, inclusive */
    double sum;    /* sum of prob over the run */
} ytk_db_run;

/* prob_dev: [n_pages, H, W] fp32 device; scratch_dev: n_pages*H*W*4 bytes device; runs_dev: [n_pages, max_runs_per_page]
 * device; meta_dev: [n_pages, 4] int32 device = {runs found (> max_runs_per_page means truncated), components,
 * 4 * Euler number (8-connectivity: holes = components - Euler number), overflow flag}.  Asynchronous on the stream.
 * The end points of a component's runs have the same minAreaRect as its OpenCV contour, sum / pixel count of the runs is
 * box_score_fast of a component without holes; pages with holes must use the host path (the caller's decision). */
int ytk_dbnet_post_front(const float* prob_dev, int n_pages, int H, int W, float thresh, void* scratch_dev,
                         long long scratch_bytes, ytk_db_run* runs_dev, int max_runs_per_page, int32_t* meta_dev,
                         void* cuda_stream);

/* ---- DBNet text detector: replaces `self.model(tensor)` in reference TextDetector.__call__
 * (src/yomitoku/text_detector.py:127-129 -> models/dbnet_plus.py:243-246) and, in the fused u8 entry, also
 * TextDetector.preprocess (text_detector.py:99-107, data/functions.py:196-264). ---- */
typedef struct ytk_dbnet ytk_dbnet;

/* One entry of the reference-keyed state_dict (host fp32, SURVEY.md Appendix C; the strict key set of
 * DBNet.state_dict() / PARSeq.state_dict() as stored in the HF model.safetensors). */
typedef struct {
    const char* name;
    const float* data;
    int ndim;
    long long shape[4];
} ytk_tensor;

/* Folds BatchNorm, repacks weights to NHWC fp16 and uploads them.  shortest_size / limit_size are cfg.data.* of the
 * detector config (reference configs/cfg_text_detector_dbnet_v2_1.py:23-26). */
int ytk_dbnet_create(const ytk_tensor* tensors, int n_tensors, int shortest_size, int limit_size, ytk_dbnet** out);
void ytk_dbnet_destroy(ytk_dbnet* h);
/* CUDA device ordinal a handle is bound to (the device that was current at create()). */
int ytk_dbnet_device(const ytk_dbnet* h);
/* network input size for an H0 x W0 page = reference resize_shortest_edge (data/functions.py:212-224) */
int ytk_dbnet_input_size(const ytk_dbnet* h, int H0, int W0, int* Hn, int* Wn);
/* pages: [n_pages, H0, W0, 3] uint8 BGR (caller-owned; device pointer iff pages_on_device, else host - pinned for
 * async copies), any size: the resize to (Hn, Wn) is cv2.resize(INTER_AREA) whether the page shrinks or grows.
 * prob_out: [n_pages, Hn, Wn] fp32 sigmoid map = preds["binary"][:, 0] of the reference.  The same as
 * ytk_dbnet_forward_table_u8 (below) with the table of n_pages evenly spaced whole pages. */
int ytk_dbnet_forward_u8(ytk_dbnet* h, const uint8_t* pages, int pages_on_device, int n_pages, int H0, int W0,
                         float* prob_out, int out_on_device, void* cuda_stream);
/* model-level seam: x = normalised (n,3,H,W) fp32 exactly as the reference feeds DBNet.forward; H, W % 32 == 0 */
int ytk_dbnet_forward_f32(ytk_dbnet* h, const float* x_nchw, int x_on_device, int n, int H, int W, float* prob_out,
                          int out_on_device, void* cuda_stream);
/* algorithmic conv FLOPs (2*MAC) of one forward at this shape (roofline accounting) */
double ytk_dbnet_flops(ytk_dbnet* h, int n_pages, int Hn, int Wn);
/* test hook: copy a named intermediate activation (NHWC) of the last run at this shape to host fp32.
 * shape4 receives n,h,w,c.  Names: stem, pool, layer1..layer4, layerL.B, f1..f4, fuse, asf_a, bin1, bin2, prob. */
int ytk_dbnet_debug_tensor(ytk_dbnet* h, int n_pages, int Hn, int Wn, const char* name, float* host_out,
                           long long capacity, int* shape4);

/* ---- PARSeq text recognizer: replaces `self.model(data).softmax(-1)` + tokenizer arg-max in reference
 * TextRecognizer._run_inference / postprocess (src/yomitoku/text_recognizer.py:247-256, 232-245 ->
 * models/parseq.py:159-311, postprocessor/parseq_tokenizer.py:64-88). ---- */
typedef struct ytk_parseq ytk_parseq;

/* values of the recognizer config (reference configs/cfg_text_recognizer_parseq*.py) + repetition-stop knobs
 * (models/parseq.py:93-96) */
typedef struct {
    int embed_dim, enc_heads, enc_depth, patch_h, patch_w, img_h, img_w, num_tokens, max_label_length, dec_heads,
        mlp_ratio, dec_mlp_ratio, refine_iters, repetition_stop, rep_period_max, rep_min_run_p1, rep_min_repeats,
        decode_ar; /* cfg.decode_ar (models/parseq.py:192,252): 0 = one non-autoregressive pass instead of the AR loop */
} ytk_parseq_cfg;

/* One crop of a packed recognizer call.  The canvas is the reference's `dataset.data[i]` (RGB uint8, 32 rows,
 * w columns, black padded, data/functions.py:379-439); wp is the width the reference's _collate would pad it to
 * (max width of its mini-batch, text_recognizer.py:146-156); group = index of that mini-batch (the AR loop stops
 * per mini-batch, models/parseq.py:245-250). */
typedef struct {
    long long pix_off; /* byte offset of the canvas in the packed buffer */
    int w;             /* stored canvas width */
    int wp;            /* padded width (multiple of patch_w, >= w) */
    int tok_off;       /* first encoder token row of this crop (crops are packed back to back) */
    int ntok;          /* (32 / patch_h) * (wp / patch_w) */
    int group;
} ytk_crop;

int ytk_parseq_create(const ytk_tensor* tensors, int n_tensors, const ytk_parseq_cfg* cfg, ytk_parseq** out);
void ytk_parseq_destroy(ytk_parseq* h);
int ytk_parseq_device(const ytk_parseq* h);
void ytk_parseq_set_refine_iters(ytk_parseq* h, int refine_iters);
/* crops: packed canvases; host pointer (pinned memory for async copies) or, iff crops_on_device, a device pointer
 * (the copy is skipped).  Outputs (host): ids / probs
 * [n_crops, max_label_length + 1] = per-position arg-max token and its softmax probability (what
 * BaseTokenizer.decode computes from the full distribution), group_len [n_groups] = AR steps each mini-batch ran
 * (= number of valid positions when refine_iters == 0). */
int ytk_parseq_forward_crops(ytk_parseq* h, const uint8_t* crops, int crops_on_device, long long crops_bytes,
                             const ytk_crop* descs, int n_crops, int n_groups, int32_t* ids_out, float* probs_out,
                             int32_t* group_len_out, void* cuda_stream);
/* model-level seam: images (B,3,32,W) fp32 as fed to PARSeq.forward (one mini-batch).  logits_out (optional)
 * receives (B, S, C) fp32, S = max_label_length + 1 (only the first group_len positions are written when
 * refine_iters == 0), WITHOUT the repetition patch; rep_cut_out [B] (-1 = none) lets the caller apply
 * models/parseq.py:301-309.  memory_out (optional, host) receives the encoder output (B*N, D) fp32. */
int ytk_parseq_forward_f32(ytk_parseq* h, const float* images, int images_on_device, int B, int W, float* logits_out,
                           int logits_on_device, int32_t* ids_out, float* probs_out, int32_t* steps_out,
                           int32_t* rep_cut_out, float* memory_out, void* cuda_stream);
/* algorithmic FLOPs (2*MAC; GEMMs + attention) and AR steps of the last forward call */
double ytk_parseq_last_flops(ytk_parseq* h);
int ytk_parseq_last_steps(ytk_parseq* h);
/* CUDA-event times (ms) of the last forward: encoder, AR decode, refinement, output copies */
void ytk_parseq_last_phase_ms(ytk_parseq* h, float* ms4);

/* op level, for the parity tests: the single-query attention of the AR decoder.  One query per (row, head), head dim
 * D / heads in {32, 48, 64, 96}, fp16 operands with rows of D (queries) and [K | V] rows of 2 * D (keys / values),
 * 16-byte aligned; out [B, D] fp16.
 *   mode 0 (self-attention of AR step i = *step_dev, a device int with 0 <= i < S <= 800): q [S, D], kv [B][S][2D]; row b
 *          attends with q[i] to its keys 0..i
 *   mode 1 (cross-attention): q [B, D], kv = encoder memory [tokens][2D]; row b attends with q[b] to the ntok rows from
 *          tok_off of crops[b] (host records; 1 <= ntok <= 800, the other fields are not read); S and step_dev are unused
 * Asynchronous on the stream (mode 1 uploads the records to a buffer it allocates and frees on the stream); invalid
 * arguments are an error, not a launch. */
int ytk_op_single_query_attn_f16(int mode, const void* q, const void* kv, int B, int S, int D, int heads,
                                 const int* step_dev, const ytk_crop* crops, void* out, void* cuda_stream);

/* op level, for the parity tests: the recognizer's decoding tail, each entry called as the engine calls it.  Device
 * pointers; asynchronous on the stream; invalid arguments are an error, not a launch.  An output row r of the softmax
 * statistics goes to index g = r * g_stride + g_off of ids / probs (crop g / S, position g % S); when rep_cut is given
 * and rep_cut[g / S] == g % S, the position gets eos_id with probability 1 (the repetition patch).
 *   linear_rowmax    the head GEMM with the row-max epilogue: per row of A [M, lda] fp16 times W [N, K] fp16 plus bias
 *                    [N] fp32 (or NULL), npart = 2 * tiles_n float4 partials {max, sum exp(x - max), bit-cast arg-max,
 *                    0} at partials[row * npart ...]; argmax_only != 0 leaves the sums 0 (the AR loop's mode when
 *                    refinement follows).  npart_out / block_n_out (host, optional) receive the layout the plan chose:
 *                    it depends on the SM count.  partials_capacity (float4s) must hold M * npart.
 *   softmax_max      ids / probs from fp32 logits [rows, ldl] (C valid columns, ldl % 4 == 0, 16-byte aligned).
 *   rowmax_finalize  the same from the partials [rows, ldp] of linear_rowmax (npart <= ldp valid per row).
 *   ar_control       one AR step of the engine's loop: arg-max of the step's logits (npart == 0: fp32 logits [B, ldl];
 *                    npart > 0: the partials, ldl float4s per row), the repetition stop, EOS bookkeeping, the ends of
 *                    groups g0 .. g0 + ngroups - 1 (row_group holds global group ids), and cin [B, D] fp16 =
 *                    LN_c(pos_q[j - 1] + sqrt(D) * embed[token]) for the token entering position j = step + 1.  embed is
 *                    the engine's table: rows of D fp32, zero padded from d_real and pre-multiplied by sqrt(d_real / D),
 *                    so sqrt(D) * embed = sqrt(d_real) * E; pos_q [S - 1, D], g_c / b_c [D] likewise zero padded.
 *                    The state (tgt, raw [B][S]; rep_cut, rep_done, has_eos [B]; group_len, open_rows [g0 + ngroups];
 *                    n_active, step, ticket [1]) is read and updated on the device; open_rows and ticket are zero
 *                    between steps.
 *   refine_embed     the refinement context [BOS, raw[0 .. L-2]] of each row, L = group_len[row_group[row]]: cin
 *                    [B][S][D] fp16 (positions >= L get EOS), klen [B] = L, kpad [B] = first EOS position in the
 *                    context (L if none).  Same embedding tables as ar_control; B <= 65535.
 *   apply_rep_cut    the repetition patch alone (refine_iters == 0): ids / probs [B, S], rep_cut [B] (-1 = none). */
typedef struct {
    int32_t* tgt;
    int32_t* raw;
    int32_t* rep_cut;
    int32_t* rep_done;
    int32_t* has_eos;
    int32_t* group_len;
    int32_t* n_active;
    int32_t* step;
    int32_t* open_rows;
    int32_t* ticket;
} ytk_ar_state;   /* ten device pointers, the layout of ytk::ArState (csrc/parseq_ops.h) */

int ytk_op_linear_rowmax_f16(const void* A, long long lda, int M, int K, const void* W, int N, const float* bias,
                             int argmax_only, void* partials, long long partials_capacity, int* npart_out,
                             int* block_n_out, void* cuda_stream);
int ytk_op_softmax_max_f32(const float* logits, long long ldl, int C, int rows, int S, long long g_stride,
                           long long g_off, const int* rep_cut, int eos_id, int* ids, float* probs, void* cuda_stream);
int ytk_op_rowmax_finalize_f32(const void* partials, long long ldp, int npart, int C, int rows, int S,
                               long long g_stride, long long g_off, const int* rep_cut, int eos_id, int* ids,
                               float* probs, void* cuda_stream);
int ytk_op_ar_control(const float* logits, long long ldl, int C, int npart, int B, int S, const int* row_group, int g0,
                      int ngroups, const ytk_ar_state* state, int eos_id, int rep_on, int rep_period_max,
                      int rep_min_run_p1, int rep_min_repeats, const float* embed, const float* pos_q, int D,
                      int d_real, const float* g_c, const float* b_c, void* cin, void* cuda_stream);
int ytk_op_refine_embed(const int* raw, const int* row_group, const int* group_len, int B, int S, int bos_id,
                        int eos_id, const float* embed, const float* pos_q, int D, int d_real, const float* g_c,
                        const float* b_c, void* cin, int* klen, int* kpad, void* cuda_stream);
int ytk_op_apply_rep_cut(const int* rep_cut, int B, int S, int C, int eos_id, int* ids, float* probs,
                         void* cuda_stream);

/* op level, for the parity tests: the DBNet detector's own kernels, each called as the engine calls it.  Activations
 * are NHWC fp16 on the device, 16-byte aligned; weights are the reference's fp32 layouts on the host, packed by the
 * code the engine's loader uses (with no BatchNorm: the bias is the whole shift).  Asynchronous on the stream (weights
 * and scratch go to buffers allocated and freed on it); invalid arguments are an error, not a launch.
 *   preprocess  (ytk_op_dbnet_preprocess_table_u8, declared with the page tables below) n BGR u8 pages -> the stem's
 *               canvas [n, Hn+6, Wn+8, 8], all of it written: pixel (h, w) at (h+3, w+3), channels 0..2 =
 *               cv2.resize(INTER_AREA) / 255 with the mean / std applied by position to B, G, R, zero border and zero
 *               channels 3..7.  Each page gets the rule OpenCV picks for its own scales: area decimation when no axis
 *               grows, else bilinear resampling on both axes with INTER_AREA's "area-mode" coefficients.
 *   stem       7x7 / stride 2 / pad 3 conv (w [64][3][7][7], bias [64]) + ReLU over that canvas -> out
 *               [n, Hn/2, Wn/2, 64]; Hn and Wn multiples of 32.
 *   maxpool     max_pool2d(3, 2, 1): in [n, H, W, C] -> out [n, (H+1)/2, (W+1)/2, C]; C a multiple of 8.
 *   upsample    bilinear, align_corners=False: src [n, Hs, Ws, C] -> channels [coff, coff+C) of dst [n, Hd, Wd, ldd],
 *               written (accumulate = 0) or added (accumulate != 0); coff and ldd multiples of 8, coff + C <= ldd.
 *   asf         the scale fusion after its 3x3 conv: a [n, H, W, 64], fuse [n, H, W, 256] rescaled in place by group;
 *               w1 [16][64] / w2 [64][16] fp32 on the device, sp3 [9] / att [4][64] on the host.  Optional outputs
 *               (device, or NULL): gvec [n, 64] = the channel gate, m [n, H, W] fp32 = the channel-mean map.
 *   head        ConvT(64->64, 2, 2) + ReLU, then ConvT(64->1, 2, 2) + sigmoid in one GEMM epilogue: x [n, H, W, 64]
 *               -> prob [n, 4H, 4W] fp32 (8-byte aligned); w1 [64][64][2][2], b1 [64], w2 [64][1][2][2], b2. */
int ytk_op_dbnet_stem_f16(const void* canvas_dev, int n, int Hn, int Wn, const float* w_host, const float* bias_host,
                          void* out_dev, void* cuda_stream);
int ytk_op_maxpool3x3s2_f16(const void* in, int n, int H, int W, int C, void* out, void* cuda_stream);
int ytk_op_upsample_bilinear_f16(const void* src, int n, int Hs, int Ws, int C, void* dst, int Hd, int Wd, long long ldd,
                                 int coff, int accumulate, void* cuda_stream);
int ytk_op_asf_f16(const void* a, void* fuse, int n, int H, int W, const float* w1_dev, const float* w2_dev,
                   const float* sp3_host, float sp1, const float* att_host, float* gvec_out, float* m_out,
                   void* cuda_stream);
int ytk_op_dbnet_head_f32(const void* x_dev, int n, int H, int W, const float* w1_host, const float* b1_host,
                          const float* w2_host, float b2, float* prob_dev, void* cuda_stream);

/* ---- Device-side crop extraction: replaces the pixel work of ParseqDataset._preprocess_on (reference
 * src/yomitoku/data/dataset.py:106-123): extract_roi_with_perspective (data/functions.py:301-333, cv2.warpPerspective),
 * rotate_text_image (:336-350) and resize_with_padding / resize_with_dynamic_padding (:379-439, cv2.resize INTER_AREA +
 * paste on a black canvas), bit-exact with OpenCV 4.13 for 8UC3.  The scalar decisions (bounding box, output size,
 * rotation, content and canvas size, the inverse perspective matrix) stay on the host: one record per crop
 * (yomitoku_b200/data.py: crop_geometry).  The canvases come out packed exactly as ytk_parseq_forward_crops takes them
 * with crops_on_device = 1, so no crop pixel leaves the GPU. ---- */
typedef struct {
    double minv[9];    /* cv2.invert(cv2.getPerspectiveTransform(quad - (x0,y0), [[0,0],[w,0],[w,h],[0,h]])), row major */
    long long roi_off; /* byte offset of this crop's rectified ROI in scratch_dev: w*h*3 bytes */
    long long pix_off; /* byte offset of this crop's canvas in canvases_dev: canvas_h*canvas_w*3 bytes, RGB */
    int page;          /* index into the page table */
    int x0, y0, rw, rh; /* bounding-box slice of the (int64-truncated) quad inside the page */
    int w, h;          /* rectified size: (int |p0p1|, int |p1p2|) */
    int rot;           /* bit 0: rotate 90 degrees counter-clockwise after the warp (h > 2w); bit 1: then rotate by 180
                          degrees (the orientation fallback's second look, text_recognizer.py:319-328) */
    int cw, ch;        /* content size after the down-scale-only fit (calc_resize_without_padding) */
    int canvas_w, canvas_h;
} ytk_crop_geom;
/* The crop extraction and the source_downscale pyramid read their pages through a page table: see
 * ytk_extract_crops_table_u8 and ytk_halve_pages_table_u8 below. */

/* ---- RT-DETRv2 layout parser / table structure recognizer / table cell detector: replaces `self.model(img_tensor)` in
 * reference LayoutParser.__call__ (src/yomitoku/layout_parser.py:258-262 -> models/rtdetr.py:17-22),
 * TableStructureRecognizer.__call__ (table_structure_recognizer.py:272-276) and CellDetector.__call__
 * (table_cell_detector.py:502-504) and, in the u8 entry, also their `self.transforms` (cvtColor, the table crop, PIL
 * bilinear resize, ToTensor).  One architecture, three weight sets (num_classes 6 / 3 / 6, num_queries
 * 300 / 300 / 1500, img_size 640 / 640 / 960). ---- */
typedef struct ytk_rtdetr ytk_rtdetr;

/* tensors: the reference's state_dict (RTDETRv2(cfg).state_dict() keys, host fp32; the boolean `decoder.valid_mask` may
 * be passed as 0/1 floats or left out - it is derived from the finite entries of `decoder.anchors`).  img_size: the square
 * evaluation size (cfg.data.img_size = eval_spatial_size: 640 or 960, a multiple of 32). */
int ytk_rtdetr_create(const ytk_tensor* tensors, int n_tensors, int num_classes, int num_queries, int img_size,
                      ytk_rtdetr** out);
void ytk_rtdetr_destroy(ytk_rtdetr* h);
int ytk_rtdetr_device(const ytk_rtdetr* h);
/* x: [n, 3, img, img] fp32 in [0, 1] (what the reference's transforms produce), host or device.
 * pred_logits: [n, num_queries, num_classes] fp32, pred_boxes: [n, num_queries, 4] fp32 (cx, cy, w, h in [0, 1]) - the
 * "pred_logits" / "pred_boxes" of the reference's output dict, rows in the decoder's query order (descending encoder
 * score).  Outputs on the host: the call returns after the copy; on the device: asynchronous on the stream. */
int ytk_rtdetr_forward_f32(ytk_rtdetr* h, const float* x, int x_on_device, int n, float* pred_logits, float* pred_boxes,
                           int out_on_device, void* cuda_stream);

/* One model input of the u8 entry: a rectangle of a BGR page.  Invalid records (a page extent beyond pages_bytes, an
 * empty rectangle, a rectangle outside its page) are an error, not a launch. */
typedef struct {
    long long page_off;   /* byte offset of the page in `pages`: H*W*3 bytes, BGR, rows of W*3 bytes */
    int H, W;             /* page size (pages of different sizes may share one buffer) */
    int x0, y0, x1, y1;   /* the model input is page[y0:y1, x0:x1]; 0 <= x0 < x1 <= W, 0 <= y0 < y1 <= H */
} ytk_rtdetr_src;         /* 32 bytes */

/* ---- Page tables: pages of any sizes back to back in one flat uint8 buffer, one record per page, the same record and
 * rules as the RT-DETRv2 sources above.  A same-size [n, H0, W0, 3] buffer is the table {i * H0 * W0 * 3, H0, W0, 0, 0,
 * W0, H0}.  The record is read as a page (its rectangle must be the whole page) by the detector and the pyramid, and
 * as the page a crop record's `page` indexes by the crop extraction.  The records are host arrays (pageable: reusable
 * as soon as the call returns); invalid records (a page beyond pages_bytes, an empty page, a rectangle outside its
 * page or, where whole pages are read, not the whole page) are an error, not a launch.  At most 65535 pages a call. ---- */
typedef ytk_rtdetr_src ytk_page;

/* The DBNet forward of u8 pages: every page is resized to the network input of its own size as ytk_dbnet_forward_u8
 * describes, and all pages of one call must map to the same input (Hn, Wn) (an error names both shapes otherwise);
 * prob_out [n_pages, Hn, Wn].  pages: pages_bytes bytes on the device iff pages_on_device, else on the host. */
int ytk_dbnet_forward_table_u8(ytk_dbnet* h, const uint8_t* pages, int pages_on_device, long long pages_bytes,
                               const ytk_page* table, int n_pages, float* prob_out, int out_on_device,
                               void* cuda_stream);
/* op level, for the parity tests: the pre-processing of ytk_dbnet_forward_table_u8 alone (the DBNet op "preprocess"
 * above), each page resized to (Hn, Wn).  The records are uploaded to a buffer allocated and freed on the stream. */
int ytk_op_dbnet_preprocess_table_u8(const uint8_t* pages_dev, long long pages_bytes, const ytk_page* table, int n,
                                     int Hn, int Wn, void* canvas_dev, void* cuda_stream);
/* The crop extraction: geoms[i].page indexes `table`, the ROI lies inside that page.  pages_dev: the pages in device
 * memory (e.g. the buffer handed to ytk_dbnet_forward_table_u8 with pages_on_device = 1); geoms: host array (pageable:
 * may be reused as soon as the call returns; page-locked: must stay valid until the stream has passed the call);
 * scratch_dev / canvases_dev: caller-owned device buffers.  scratch_dev holds the rectified ROIs (at roi_off) and,
 * 16-byte aligned after the last ROI, a copy of the n_crops records followed by the page table (one upload), so
 * scratch_bytes >= align16(max(roi_off + w*h*3)) + n_crops * sizeof(ytk_crop_geom) + n_pages * sizeof(ytk_page): the
 * call allocates nothing.  Asynchronous on cuda_stream: one H2D copy + two kernel launches. */
int ytk_extract_crops_table_u8(const uint8_t* pages_dev, long long pages_bytes, const ytk_page* table, int n_pages,
                               const ytk_crop_geom* geoms, int n_crops, uint8_t* scratch_dev, long long scratch_bytes,
                               uint8_t* canvases_dev, long long canvases_bytes, void* cuda_stream);
/* One level of the recognizer's source_downscale pyramid (reference data/dataset.py:64-86): page i of src_table ->
 * page i of dst_table = cv2.resize(page, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_AREA), bit-exact with OpenCV
 * 4.13 (2x2 cells round half up; the clipped last column / row of an odd size averages the pixels that exist).  The
 * destination page must be cvRound(H / 2) x cvRound(W / 2) (round half to even) - anything else is rejected.
 * scratch_dev holds the two uploaded tables: scratch_bytes >= 2 * n_pages * sizeof(ytk_page). */
int ytk_halve_pages_table_u8(const uint8_t* src_dev, long long src_bytes, const ytk_page* src_table, int n_pages,
                             uint8_t* dst_dev, long long dst_bytes, const ytk_page* dst_table, uint8_t* scratch_dev,
                             long long scratch_bytes, void* cuda_stream);

/* ---- Pages that are already on the device (a GPU JPEG decode, video frames, an earlier model's output): each source
 * page is an H x W x 3 uint8 array with arbitrary non-negative byte strides, so a contiguous HWC page, a crop or a step
 * of one and the permute(1, 2, 0) of a CHW tensor all go in without a copy. ---- */
typedef struct {
    const uint8_t* data;   /* device pointer of pixel (0, 0), channel 0 */
    long long sh, sw, sc;  /* byte strides of a row, a column and a channel (>= 0) */
    int H, W;              /* page size (>= 1) */
    int rgb;               /* channel order of the source: 0 = B, G, R (the pages of this API); 1 = R, G, B */
    int pad_;
} ytk_page_src;            /* 48 bytes */

/* Packs n source pages into the page-table buffer dst_dev: page i is written as H x W x 3 BGR bytes at
 * table[i].page_off (table[i] must be the whole page, of the source's size).  The copy is exact.  srcs / table: host
 * arrays (pageable: reusable as soon as the call returns); every source and dst_dev on the same device; scratch_dev
 * holds the uploaded records: scratch_bytes >= n * (sizeof(ytk_page_src) + sizeof(ytk_page)).  Asynchronous on
 * cuda_stream: one H2D copy + one kernel launch, nothing allocated; invalid records are an error, not a launch. */
int ytk_pack_pages_u8(const ytk_page_src* srcs, int n, uint8_t* dst_dev, long long dst_bytes, const ytk_page* table,
                      uint8_t* scratch_dev, long long scratch_bytes, void* cuda_stream);

/* The reference's whole input path on the device: per record, the rectangle as RGB,
 * Image.fromarray(rgb_crop).resize((img, img), Image.BILINEAR) bit for bit (Pillow's fixed-point separable resample,
 * horizontal pass first) and ToTensor, then the forward of ytk_rtdetr_forward_f32 with the same outputs, ordering and
 * copy semantics.  The layout parser reads whole pages, the table structure recognizer and the cell detector table
 * crops of them; one upload of the pages serves all three.  pages: pages_bytes bytes on the device iff pages_on_device,
 * else on the host (copied into a buffer the handle owns; page-locked memory must stay valid until the stream has
 * passed the call).  srcs: n host records. */
int ytk_rtdetr_forward_u8(ytk_rtdetr* h, const uint8_t* pages, int pages_on_device, long long pages_bytes,
                          const ytk_rtdetr_src* srcs, int n, float* pred_logits, float* pred_boxes, int out_on_device,
                          void* cuda_stream);
/* op level, for the parity tests: the resize of ytk_rtdetr_forward_u8 alone.  out_rgb_dev = [n][size][size][3] u8 RGB
 * (the resized images, before / 255); scratch_dev holds at least ytk_op_resize_bilinear_scratch_bytes(srcs, n, size)
 * bytes: the call allocates nothing.  Asynchronous on the stream: one H2D copy + two kernel launches. */
int ytk_op_resize_bilinear_u8(const uint8_t* pages_dev, long long pages_bytes, const ytk_rtdetr_src* srcs, int n,
                              int size, uint8_t* scratch_dev, long long scratch_bytes, uint8_t* out_rgb_dev,
                              void* cuda_stream);
/* scratch bytes ytk_op_resize_bilinear_u8 needs for these records (page extents are not checked here), -1 if a record
 * is invalid */
long long ytk_op_resize_bilinear_scratch_bytes(const ytk_rtdetr_src* srcs, int n, int size);
double ytk_rtdetr_flops(ytk_rtdetr* h, int n);

/* ---- Table semantic parser: the word-to-element assignment of reference TableSemanticParser.aggregate
 * (src/yomitoku/table_semantic_parser.py:683-701), every table and the paragraphs of every page in one launch. ---- */
typedef struct {
    int w0, w1;   /* the group's words: word_boxes rows [w0, w1) */
    int e0, e1;   /* its elements (one table's cells, or one page's paragraphs): elem_boxes rows [e0, e1) */
} ytk_overlap_group;

/* For every word of every group, the element of the group that covers the largest share of the word: both boxes
 * truncated toward zero to integers and intersected, ratio = integer intersection area / the word's raw fp64 area,
 * the first element with the largest ratio wins and elements with elem_skip != 0 never do; -1 when no element overlaps
 * the word or the best ratio is below overlap_th.  Bit-exact with the reference's Python (IEEE fp64, no contraction).
 * word_boxes [n_words][4] / elem_boxes [n_elems][4]: fp64 x1, y1, x2, y2 on the device, 16-byte aligned, every
 * coordinate finite with |v| < 2^30 (the caller checks the values; the call cannot); elem_skip [n_elems] bytes on the
 * device.  groups: host array.  Group g's results are best_dev / ratio_dev [off_g, off_g + w1 - w0) with off_g the
 * word count of the groups before it, so out_capacity >= the sum of all w1 - w0.  ratio is the best ratio found (0
 * without overlap) even where best is -1.  Asynchronous on cuda_stream: one H2D copy of the group records and one
 * launch; invalid groups are an error, not a launch. */
int ytk_op_assign_best_overlap_f64(const double* word_boxes_dev, int n_words, const double* elem_boxes_dev,
                                   const uint8_t* elem_skip_dev, int n_elems, const ytk_overlap_group* groups,
                                   int n_groups, double overlap_th, int* best_dev, double* ratio_dev,
                                   long long out_capacity, void* cuda_stream);

/* test hook: copies an intermediate activation (by name, see rtdetr_engine.cu) of the LAST forward of batch size n to
 * the host as fp32; shape4 = {n, h, w, c} (token matrices: {1, 1, rows, c}) */
int ytk_rtdetr_debug_tensor(ytk_rtdetr* h, int n, const char* name, float* host_out, long long capacity, int* shape4);

#ifdef __cplusplus
}
#endif
#endif /* YOMITOKU_B200_H */
