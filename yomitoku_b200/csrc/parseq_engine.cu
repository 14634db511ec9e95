// PARSeq recognizer (ViT encoder + 1-layer two-stream decoder, greedy AR decode + one refinement pass) as a launch
// plan of wgmma GEMMs, tensor-core flash attention and small fused kernels.  Replaces reference
// models/parseq.py:159-311 and models/layers/parseq_transformer.py:69-244 for inference.
//
// What differs from the reference *implementation* while keeping its *results* (SURVEY.md Appendix A):
//  * ragged batches: all crops of a call are packed token-major ([T, D] matrices); each crop keeps the padded width
//    its reference mini-batch would have given it, so pad columns stay real tokens (A9) without dense padding;
//  * K/V caches: encoder memory K/V projected once, content K/V appended per step (exactly output preserving because
//    the decoder has depth 1 and never updates the content stream, A15);
//  * the query-side self-attention projection of LN_q(pos_queries) is row independent and precomputed at load time;
//  * greedy arg-max, EOS bookkeeping, the repetition detector and the per-group early stop run on the device
//    (zero host syncs per step; the host peeks at a pinned counter every few steps);
//  * softmax + per-position max are fused after the head GEMM: only (id, prob) per position leave the device.
// Data layout in HBM: residual stream fp32 [T, D]; GEMM operands bf16; content K/V cache [position][row][2D] bf16.
#include "parseq_engine.h"

#include <cmath>
#include <cstring>
#include <memory>

#include "ptx.cuh"

namespace ytk {

#define CK(x)                                                                   \
    do {                                                                        \
        cudaError_t e_ = (x);                                                   \
        if (e_ != cudaSuccess) {                                                \
            set_error("%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); \
            return 1;                                                           \
        }                                                                       \
    } while (0)

// ---------------------------------------------------------------------------------------------- model
static int up(std::vector<void*>& owned, const void* host, size_t bytes, void** dev) {
    CK(cudaMalloc(dev, bytes));
    CK(cudaMemcpy(*dev, host, bytes, cudaMemcpyHostToDevice));
    owned.push_back(*dev);
    return 0;
}

static int load_linear(std::vector<void*>& owned, const float* w, const float* b, int N, int K, LinearW* out) {
    const int Kp = (K + 63) / 64 * 64;
    std::vector<uint16_t> p((size_t)N * Kp, 0);
    for (int n = 0; n < N; ++n)
        for (int k = 0; k < K; ++k) p[(size_t)n * Kp + k] = f2op_host(w[(size_t)n * K + k]);
    if (up(owned, p.data(), p.size() * 2, &out->w)) return 1;
    void* d = nullptr;
    if (up(owned, b, (size_t)N * 4, &d)) return 1;
    out->b = reinterpret_cast<float*>(d);
    out->N = N;
    out->K = Kp;
    return 0;
}

// Generalised load: output row n goes to row rowmap[n] of an [Np][Kp] matrix (identity when null), input feature k to
// column colmap[k]; rows may be scaled (softmax-scale folding).  Rows / columns that nothing maps to are zero, so
// padded features stay exactly zero through the whole network.
static int load_linear_ex(std::vector<void*>& owned, const float* w, const float* b, int N, int K,
                          const std::vector<int>* rowmap, int Np, const std::vector<int>* colmap, int Kp,
                          const std::vector<float>* rowscale, LinearW* out) {
    if (!rowmap && !colmap && !rowscale && Np == N && Kp == K) return load_linear(owned, w, b, N, K, out);
    std::vector<float> w2((size_t)Np * Kp, 0.f), b2(Np, 0.f);
    for (int n = 0; n < N; ++n) {
        const int r = rowmap ? (*rowmap)[n] : n;
        const float sc = rowscale ? (*rowscale)[n] : 1.f;
        float* dst = &w2[(size_t)r * Kp];
        const float* src = w + (size_t)n * K;
        if (colmap)
            for (int k = 0; k < K; ++k) dst[(*colmap)[k]] = src[k] * sc;
        else
            for (int k = 0; k < K; ++k) dst[k] = src[k] * sc;
        b2[r] = b[n] * sc;
    }
    return load_linear(owned, w2.data(), b2.data(), Np, Kp, out);
}

static int up_padded(std::vector<void*>& owned, const float* src, long long rows, int D, int Dp, float scale,
                     float** dev) {
    void* d = nullptr;
    if (D == Dp && scale == 1.f) {
        if (up(owned, src, (size_t)rows * D * 4, &d)) return 1;
    } else {
        std::vector<float> t((size_t)rows * Dp, 0.f);
        for (long long r = 0; r < rows; ++r)
            for (int k = 0; k < D; ++k) t[(size_t)r * Dp + k] = src[(size_t)r * D + k] * scale;
        if (up(owned, t.data(), t.size() * 4, &d)) return 1;
    }
    *dev = reinterpret_cast<float*>(d);
    return 0;
}

static int load_linear_named(std::vector<void*>& owned, const WeightSet& ws, const std::string& wn,
                             const std::string& bn, int N, int K, LinearW* out) {
    const TensorView *w = ws.need(wn, (long long)N * K), *b = ws.need(bn, N);
    if (!w || !b) return 1;
    return load_linear(owned, w->data, b->data, N, K, out);
}

static int load_ln(std::vector<void*>& owned, const WeightSet& ws, const std::string& p, int D, int Dp, LnW* out) {
    const TensorView *g = ws.need(p + ".weight", D), *b = ws.need(p + ".bias", D);
    if (!g || !b) return 1;
    // zero gamma / beta on the padded features: LayerNorm then writes exact zeros there
    return up_padded(owned, g->data, 1, D, Dp, 1.f, &out->g) || up_padded(owned, b->data, 1, D, Dp, 1.f, &out->b);
}

static void host_ln(const float* x, const float* g, const float* b, int D, float eps, float* y) {
    double s = 0;
    for (int i = 0; i < D; ++i) s += x[i];
    const double mean = s / D;
    double q = 0;
    for (int i = 0; i < D; ++i) q += (x[i] - mean) * (x[i] - mean);
    const double rstd = 1.0 / std::sqrt(q / D + eps);
    for (int i = 0; i < D; ++i) y[i] = (float)((x[i] - mean) * rstd) * g[i] + b[i];
}

int ParseqModel::load(const WeightSet& ws, const ParseqCfg& c) {
    cfg = c;
    const int D = c.D;  // real embed_dim
    Dr = D;
    S = c.max_label_length + 1;
    C = c.num_tokens - 2;
    gh = c.img_h / c.ph;
    full_gw = c.img_w / c.pw;
    if (D % c.enc_heads != 0 || D % c.dec_heads != 0 || (D & 3) != 0) {
        set_error("PARSeq: embed_dim %d must be a multiple of 4 and of the head counts %d/%d", D, c.enc_heads,
                  c.dec_heads);
        return 1;
    }
    // The kernels want embed_dim % 64 == 0 and head dims that are multiples of 16 (tensor-core fragments).  Models
    // that do not fit (parseq-tiny: D 368, 8 heads of 46) run as the mathematically identical zero-padded model:
    // every head is padded to hdp features whose weights are zero, the residual stream to Dp = heads * hdp columns
    // that stay exactly zero, LayerNorm statistics use the real D (launch_layernorm's d_real), and the 1/sqrt(hd)
    // and sqrt(D) factors of the real model are folded into the q projections / the embedding table.
    const int hd_e = D / c.enc_heads, hd_d = D / c.dec_heads;
    int hdp_e = (hd_e + 15) / 16 * 16;
    while ((c.enc_heads * hdp_e) % 64 != 0) hdp_e += 16;
    const int Dp = c.enc_heads * hdp_e;
    const int hdp_d = Dp / c.dec_heads;
    if (Dp % c.dec_heads != 0 || hdp_d < hd_d || hdp_d % 16 != 0 || hdp_e > 96 || hdp_d > 96 || Dp > 1024) {
        set_error("PARSeq device engine: cannot lay out embed_dim %d with %d/%d heads (padded width %d, head dims %d/%d; "
                  "supported head dims 32/48/64/96, width <= 1024)",
                  D, c.enc_heads, c.dec_heads, Dp, hdp_e, hdp_d);
        return 1;
    }
    if (hdp_e != 32 && hdp_e != 48 && hdp_e != 64 && hdp_e != 96) {
        set_error("PARSeq device engine: encoder head dim %d (padded %d) unsupported (32/48/64/96)", hd_e, hdp_e);
        return 1;
    }
    if (hdp_d != 32 && hdp_d != 48 && hdp_d != 64 && hdp_d != 96) {
        set_error("PARSeq device engine: decoder head dim %d (padded %d) unsupported (32/48/64/96)", hd_d, hdp_d);
        return 1;
    }
    if (S > 101) {  // kMaxS in parseq_ops.cu; shorter label lengths fit, longer do not
        set_error("max_label_length %d > 100 unsupported", c.max_label_length);
        return 1;
    }
    cfg.D = Dp;
    const bool padded = Dp != D;
    std::vector<int> he(D), hdm(D);  // real feature -> padded per-head position (encoder / decoder head layout)
    for (int i = 0; i < D; ++i) {
        he[i] = (i / hd_e) * hdp_e + i % hd_e;
        hdm[i] = (i / hd_d) * hdp_d + i % hd_d;
    }
    const std::vector<int>* HE = padded ? &he : nullptr;
    const std::vector<int>* HD = padded ? &hdm : nullptr;
    const float qs_e = std::sqrt((float)hdp_e / (float)hd_e), qs_d = std::sqrt((float)hdp_d / (float)hd_d);
    const float es = std::sqrt((float)D / (float)Dp);  // kernels multiply the embedding by sqrt(Dp)
    const std::string e = "encoder.";
    // patch embedding conv as a GEMM: weight [D,3,ph,pw] flattened to K = 3*ph*pw (order c,py,px)
    {
        const int K = 3 * c.ph * c.pw;
        const TensorView *w = ws.need(e + "patch_embed.proj.weight", (long long)D * K),
                         *b = ws.need(e + "patch_embed.proj.bias", D);
        if (!w || !b) return 1;
        if (load_linear_ex(owned, w->data, b->data, D, K, nullptr, Dp, nullptr, K, nullptr, &patch)) return 1;
        Kpatch = patch.K;
        const TensorView* pe = ws.need(e + "pos_embed", (long long)gh * full_gw * D);
        if (!pe) return 1;
        if (up_padded(owned, pe->data, (long long)gh * full_gw, D, Dp, 1.f, &pos_embed)) return 1;
    }
    blocks.resize(c.enc_depth);
    std::vector<int> qkv_map;
    std::vector<float> qkv_scale;
    if (padded) {
        qkv_map.resize(3 * D);
        qkv_scale.assign(3 * D, 1.f);
        for (int w3 = 0; w3 < 3; ++w3)
            for (int i = 0; i < D; ++i) {
                qkv_map[w3 * D + i] = w3 * Dp + he[i];
                if (w3 == 0) qkv_scale[i] = qs_e;
            }
    }
    for (int i = 0; i < c.enc_depth; ++i) {
        const std::string p = e + "blocks." + std::to_string(i) + ".";
        EncBlock& bk = blocks[i];
        if (load_ln(owned, ws, p + "norm1", D, Dp, &bk.ln1) || load_ln(owned, ws, p + "norm2", D, Dp, &bk.ln2))
            return 1;
        const TensorView *qw = ws.need(p + "attn.qkv.weight", 3LL * D * D), *qb = ws.need(p + "attn.qkv.bias", 3 * D),
                         *pw_ = ws.need(p + "attn.proj.weight", (long long)D * D),
                         *pb = ws.need(p + "attn.proj.bias", D),
                         *w1 = ws.need(p + "mlp.fc1.weight", (long long)c.mlp_ratio * D * D),
                         *b1 = ws.need(p + "mlp.fc1.bias", c.mlp_ratio * D),
                         *w2 = ws.need(p + "mlp.fc2.weight", (long long)c.mlp_ratio * D * D),
                         *b2 = ws.need(p + "mlp.fc2.bias", D);
        if (!qw || !qb || !pw_ || !pb || !w1 || !b1 || !w2 || !b2) return 1;
        if (load_linear_ex(owned, qw->data, qb->data, 3 * D, D, padded ? &qkv_map : nullptr, 3 * Dp, nullptr, Dp,
                           padded ? &qkv_scale : nullptr, &bk.qkv))
            return 1;
        if (load_linear_ex(owned, pw_->data, pb->data, D, D, nullptr, Dp, HE, Dp, nullptr, &bk.proj)) return 1;
        if (load_linear_ex(owned, w1->data, b1->data, c.mlp_ratio * D, D, nullptr, c.mlp_ratio * D, nullptr, Dp, nullptr,
                           &bk.fc1))
            return 1;
        if (load_linear_ex(owned, w2->data, b2->data, D, c.mlp_ratio * D, nullptr, Dp, nullptr, c.mlp_ratio * D, nullptr,
                           &bk.fc2))
            return 1;
    }
    if (load_ln(owned, ws, e + "norm", D, Dp, &enc_norm)) return 1;
    const std::string d = "decoder.layers.0.";
    if (load_ln(owned, ws, d + "norm1", D, Dp, &norm1) || load_ln(owned, ws, d + "norm2", D, Dp, &norm2) ||
        load_ln(owned, ws, d + "norm_c", D, Dp, &norm_c) || load_ln(owned, ws, "decoder.norm", D, Dp, &dec_norm))
        return 1;
    const TensorView *sw = ws.need(d + "self_attn.in_proj_weight", 3LL * D * D),
                     *sb = ws.need(d + "self_attn.in_proj_bias", 3 * D),
                     *cw = ws.need(d + "cross_attn.in_proj_weight", 3LL * D * D),
                     *cb = ws.need(d + "cross_attn.in_proj_bias", 3 * D);
    if (!sw || !sb || !cw || !cb) return 1;
    std::vector<int> kv_map;
    std::vector<float> q_scale;
    if (padded) {
        kv_map.resize(2 * D);
        for (int w2 = 0; w2 < 2; ++w2)
            for (int i = 0; i < D; ++i) kv_map[w2 * D + i] = w2 * Dp + hdm[i];
        q_scale.assign(D, qs_d);
    }
    const std::vector<int>* KV = padded ? &kv_map : nullptr;
    if (load_linear_ex(owned, sw->data + (size_t)D * D, sb->data + D, 2 * D, D, KV, 2 * Dp, nullptr, Dp, nullptr,
                       &self_kv))
        return 1;
    if (load_linear_ex(owned, cw->data, cb->data, D, D, HD, Dp, nullptr, Dp, padded ? &q_scale : nullptr, &cross_q))
        return 1;
    if (load_linear_ex(owned, cw->data + (size_t)D * D, cb->data + D, 2 * D, D, KV, 2 * Dp, nullptr, Dp, nullptr,
                       &cross_kv))
        return 1;
    {
        const TensorView *ow = ws.need(d + "self_attn.out_proj.weight", (long long)D * D),
                         *ob = ws.need(d + "self_attn.out_proj.bias", D),
                         *xw = ws.need(d + "cross_attn.out_proj.weight", (long long)D * D),
                         *xb = ws.need(d + "cross_attn.out_proj.bias", D),
                         *l1w = ws.need(d + "linear1.weight", (long long)c.dec_mlp_ratio * D * D),
                         *l1b = ws.need(d + "linear1.bias", c.dec_mlp_ratio * D),
                         *l2w = ws.need(d + "linear2.weight", (long long)c.dec_mlp_ratio * D * D),
                         *l2b = ws.need(d + "linear2.bias", D), *hw = ws.need("head.weight", (long long)C * D),
                         *hb_ = ws.need("head.bias", C);
        if (!ow || !ob || !xw || !xb || !l1w || !l1b || !l2w || !l2b || !hw || !hb_) return 1;
        if (load_linear_ex(owned, ow->data, ob->data, D, D, nullptr, Dp, HD, Dp, nullptr, &self_out)) return 1;
        if (load_linear_ex(owned, xw->data, xb->data, D, D, nullptr, Dp, HD, Dp, nullptr, &cross_out)) return 1;
        if (load_linear_ex(owned, l1w->data, l1b->data, c.dec_mlp_ratio * D, D, nullptr, c.dec_mlp_ratio * D, nullptr,
                           Dp, nullptr, &lin1))
            return 1;
        if (load_linear_ex(owned, l2w->data, l2b->data, D, c.dec_mlp_ratio * D, nullptr, Dp, nullptr,
                           c.dec_mlp_ratio * D, nullptr, &lin2))
            return 1;
        if (load_linear_ex(owned, hw->data, hb_->data, C, D, nullptr, C, nullptr, Dp, nullptr, &head)) return 1;
    }
    const TensorView *em = ws.need("text_embed.embedding.weight", (long long)c.num_tokens * D),
                     *pq = ws.need("pos_queries", (long long)S * D);
    if (!em || !pq) return 1;
    if (up_padded(owned, em->data, c.num_tokens, D, Dp, es, &embed)) return 1;
    if (up_padded(owned, pq->data, S, D, Dp, 1.f, &pos_q)) return 1;
    // ---- row-independent precomputation (fp32 on the host, in the real model's feature space)
    const TensorView *gq = ws.need(d + "norm_q.weight", D), *bq = ws.need(d + "norm_q.bias", D),
                     *gc = ws.need(d + "norm_c.weight", D), *bc = ws.need(d + "norm_c.bias", D);
    if (!gq || !bq || !gc || !bc) return 1;
    {
        std::vector<float> ln(D);
        std::vector<uint16_t> q((size_t)S * Dp, 0);
        for (int i = 0; i < S; ++i) {
            host_ln(pq->data + (size_t)i * D, gq->data, bq->data, D, 1e-5f, ln.data());
            for (int n = 0; n < D; ++n) {
                const float* wr = sw->data + (size_t)n * D;
                double acc = sb->data[n];
                for (int k = 0; k < D; ++k) acc += (double)wr[k] * ln[k];
                q[(size_t)i * Dp + hdm[n]] = f2op_host((float)acc * (padded ? qs_d : 1.f));
            }
        }
        if (up(owned, q.data(), q.size() * 2, &q_self)) return 1;
        // content position 0 = sqrt(D) * E[BOS] (no positional term), LN_c, K/V projection
        std::vector<float> c0(D), l0(D);
        const float sq = std::sqrt((float)D);
        const int bos = c.num_tokens - 2;
        for (int k = 0; k < D; ++k) c0[k] = sq * em->data[(size_t)bos * D + k];
        host_ln(c0.data(), gc->data, bc->data, D, 1e-5f, l0.data());
        std::vector<uint16_t> kv(2 * Dp, 0);
        for (int n = 0; n < 2 * D; ++n) {
            const float* wr = sw->data + (size_t)(D + n) * D;
            double acc = sb->data[D + n];
            for (int k = 0; k < D; ++k) acc += (double)wr[k] * l0[k];
            kv[(n / D) * Dp + hdm[n % D]] = f2op_host((float)acc);
        }
        if (up(owned, kv.data(), kv.size() * 2, &ckv0)) return 1;
    }
    return 0;
}

ParseqModel::~ParseqModel() {
    for (void* p : owned) cudaFree(p);
}

// ---------------------------------------------------------------------------------------------- engine
static int dmalloc(std::vector<void*>& bufs, void** p, size_t bytes) {
    if (bytes == 0) bytes = 16;
    CK(cudaMalloc(p, bytes));
    bufs.push_back(*p);
    return 0;
}

int ParseqEngine::ensure(long long tok, int rows, long long crop_bytes, int groups) {
    if (tok <= cap_tok && rows <= cap_rows && crop_bytes <= cap_crop_bytes && groups <= cap_groups) return 0;
    for (void* p : bufs) cudaFree(p);
    bufs.clear();
    cap_tok = std::max(cap_tok, tok);
    cap_rows = std::max(cap_rows, rows);
    cap_crop_bytes = std::max(cap_crop_bytes, crop_bytes);
    cap_groups = std::max(cap_groups, groups);
    const int D = m->cfg.D, S = m->S;
    const long long T = (cap_tok + 127) / 128 * 128;
    const long long B = cap_rows;
    const long long R = B * S;
    const long long Rp = (R + 127) / 128 * 128;
    const int Hm = std::max(m->cfg.mlp_ratio, m->cfg.dec_mlp_ratio) * D;
#define DM(ptr, bytes)                                                             \
    do {                                                                           \
        void* t_ = nullptr;                                                        \
        if (dmalloc(bufs, &t_, (size_t)(bytes))) return 1;                         \
        ptr = reinterpret_cast<decltype(ptr)>(t_);                                 \
    } while (0)
    DM(crops_dev, cap_crop_bytes + 64);
    DM(descs_dev, sizeof(CropDesc) * B);
    DM(seqs_enc, sizeof(SeqDesc) * B);
    DM(seqs_ref, sizeof(SeqDesc) * B);
    DM(seqs_self, sizeof(SeqDesc) * B);
    DM(A_patch, T * m->Kpatch * 2);
    DM(x, T * D * 4);
    DM(h, T * D * 2);
    DM(qkv, T * 3 * D * 2);
    DM(att, T * D * 2);
    DM(mlp, std::max(T, Rp) * Hm * 2);
    DM(mem, T * D * 2);
    DM(memkv, T * 2 * D * 2);
    DM(x1, Rp * D * 4);
    DM(hb, Rp * D * 2);
    DM(qc, Rp * D * 2);
    DM(sa, Rp * D * 2);
    DM(oc, Rp * D * 2);
    mlpb = mlp;
    DM(cin, Rp * D * 2);
    DM(ckv, Rp * 2 * D * 2);
    ldl = (m->C + 255) / 256 * 256;
    logits_rows = (int)std::min<long long>(Rp, 16384);
    if (logits_rows < B) logits_rows = (int)((B + 127) / 128 * 128);
    DM(logits, (long long)logits_rows * ldl * 4);
    DM(row_group, 4 * B);
    DM(glen_const, 4 * 2 * (size_t)std::max(cap_groups, 1));
    DM(klen, 4 * B);
    DM(kpad, 4 * B);
    DM(ids, 4 * R);
    DM(probs, 4 * R);
    ar_block_ints = (size_t)(2 * R + 3 * B + 2 * cap_groups + 8);
    DM(ar_block, 4 * ar_block_ints);
#undef DM
    ar.tgt = ar_block;
    ar.raw = ar.tgt + R;
    ar.rep_cut = ar.raw + R;
    ar.rep_done = ar.rep_cut + B;
    ar.has_eos = ar.rep_done + B;
    ar.group_len = ar.has_eos + B;
    ar.open_rows = ar.group_len + cap_groups;
    // per-part scalars (the AR loop may run as two row ranges on two streams): [n_active, step, ticket, pad] x 2
    ar.n_active = ar.open_rows + cap_groups;
    ar.step = ar.n_active + 1;
    ar.ticket = ar.n_active + 2;
    if (!host_flag) CK(cudaMallocHost(reinterpret_cast<void**>(&host_flag), 4 * sizeof(int)));
    if (!st2) CK(cudaStreamCreateWithFlags(&st2, cudaStreamNonBlocking));
    if (!ev_fork) CK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
    if (!ev_join) CK(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
    for (int i = 0; i < 5; ++i)
        if (!ev[i]) CK(cudaEventCreate(&ev[i]));
    return 0;
}

ParseqEngine::~ParseqEngine() {
    for (void* p : bufs) cudaFree(p);
    if (host_flag) cudaFreeHost(host_flag);
    if (st2) cudaStreamDestroy(st2);
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_join) cudaEventDestroy(ev_join);
    for (int i = 0; i < 5; ++i)
        if (ev[i]) cudaEventDestroy(ev[i]);
}

namespace {
struct Lin {
    // small helper: build + launch a linear layer plan
    static int run(const void* A, long long lda, int M, const LinearW& w, void* out, long long ldc, int out_f32, int act,
                   const void* resid, int resid_f32, long long ldr, cudaStream_t st, double* flops,
                   GemmPlan* keep = nullptr) {
        Epilogue e;
        e.bias = w.b;
        e.resid = resid;
        e.resid_f32 = resid_f32;
        e.ldr = ldr;
        e.out = out;
        e.out_f32 = out_f32;
        e.ldc = ldc;
        e.act = act;
        GemmPlan local;
        GemmPlan* p = keep ? keep : &local;
        if (gemm_plan_create(p, A, lda, M, w.K, w.w, w.N, e)) return 1;
        if (flops) *flops += p->flops;
        return gemm_plan_launch(p, st);
    }
};
}  // namespace

int ParseqEngine::forward(const ParseqBatch& b, int* ids_out, float* probs_out, int* group_len_out, float* logits_out,
                          int logits_on_device, float* memory_out, cudaStream_t st) {
    const ParseqCfg& c = m->cfg;
    const int D = c.D, S = m->S, C = m->C;
    const int B = (int)b.descs.size();
    if (B == 0) return 0;
    long long T = 0;
    int max_ntok = 0;
    for (const CropDesc& d : b.descs) {
        T = std::max<long long>(T, (long long)d.tok_off + d.ntok);
        max_ntok = std::max(max_ntok, d.ntok);
        if (d.ntok > kMaxMem) {
            set_error("crop with %d encoder tokens exceeds the supported %d", d.ntok, kMaxMem);
            return 1;
        }
    }
    if (ensure(T, B, b.crops_bytes, b.ngroups)) return 1;
    flops = 0;
    const int R = B * S;
    const int eos = 0, bos = c.num_tokens - 2, pad_id = c.num_tokens - 1;
    // ---------------- upload descriptors (+ crops)
    std::vector<SeqDesc> se(B), sr(B);
    std::vector<int> rg(B);
    for (int i = 0; i < B; ++i) {
        const CropDesc& cd = b.descs[i];
        // encoder self-attention: q, k, v are column blocks of the packed qkv matrix (row stride 3D)
        se[i] = SeqDesc{cd.tok_off, cd.ntok, cd.tok_off, cd.ntok, (long long)cd.tok_off * 3 * D, cd.ntok, 0};
        // refinement cross-attention: queries = the row's 101 positions, keys = its encoder memory (row stride 2D)
        sr[i] = SeqDesc{i * S, S, i * S, cd.ntok, (long long)cd.tok_off * 2 * D, cd.ntok, 0};
        rg[i] = b.descs[i].group;
    }
    CK(cudaMemcpyAsync(descs_dev, b.descs.data(), sizeof(CropDesc) * B, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(seqs_enc, se.data(), sizeof(SeqDesc) * B, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(seqs_ref, sr.data(), sizeof(SeqDesc) * B, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(row_group, rg.data(), 4 * B, cudaMemcpyHostToDevice, st));
    if (b.images_f32) {
        const float* img = b.images_f32;
        if (!b.images_on_device) {
            const size_t bytes = (size_t)B * 3 * 32 * b.image_w * 4;
            CK(cudaMemcpyAsync(crops_dev, img, bytes, cudaMemcpyHostToDevice, st));
            img = reinterpret_cast<const float*>(crops_dev);
        }
        if (launch_patchify_f32(img, B, b.image_w, c.ph, c.pw, m->Kpatch, m->pos_embed, m->full_gw, D, A_patch, x, st))
            return 1;
    } else {
        const uint8_t* cp = b.crops;
        if (!b.crops_on_device) {
            CK(cudaMemcpyAsync(crops_dev, b.crops, b.crops_bytes, cudaMemcpyHostToDevice, st));
            cp = crops_dev;
        }
        if (launch_patchify_u8(cp, descs_dev, B, c.ph, c.pw, m->Kpatch, m->pos_embed, m->full_gw, D, A_patch, x,
                               (int)T, st))
            return 1;
    }
    // the host vectors above must outlive the async copies
    CK(cudaStreamSynchronize(st));
    // ---------------- encoder (reference Encoder.forward, parseq_transformer.py:206-234)
    CK(cudaEventRecord(ev[0], st));
    const int Ti = (int)T;
    if (Lin::run(A_patch, m->Kpatch, Ti, m->patch, x, D, 1, ACT_NONE, x, 1, D, st, &flops)) return 1;
    const int hd_e = D / c.enc_heads;
    for (const EncBlock& bk : m->blocks) {
        if (launch_layernorm(x, Ti, D, m->Dr, bk.ln1.g, bk.ln1.b, 1e-6f, h, nullptr, nullptr, 1, nullptr, 0, 0, st)) return 1;
        if (Lin::run(h, D, Ti, bk.qkv, qkv, 3 * D, 0, ACT_NONE, nullptr, 0, 0, st, &flops)) return 1;
        const op_t* q = reinterpret_cast<const op_t*>(qkv);
        if (launch_flash_attention(q, 3 * D, Ti, q + D, q + 2 * D, 3 * D, Ti, att, D, seqs_enc, B, max_ntok, c.enc_heads,
                                   hd_e, 0, st))
            return 1;
        if (Lin::run(att, D, Ti, bk.proj, x, D, 1, ACT_NONE, x, 1, D, st, &flops)) return 1;
        if (launch_layernorm(x, Ti, D, m->Dr, bk.ln2.g, bk.ln2.b, 1e-6f, h, nullptr, nullptr, 1, nullptr, 0, 0, st)) return 1;
        if (Lin::run(h, D, Ti, bk.fc1, mlp, bk.fc1.N, 0, ACT_GELU, nullptr, 0, 0, st, &flops)) return 1;
        if (Lin::run(mlp, bk.fc1.N, Ti, bk.fc2, x, D, 1, ACT_NONE, x, 1, D, st, &flops)) return 1;
    }
    for (const CropDesc& d : b.descs) flops += 4.0 * d.ntok * (double)d.ntok * D * c.enc_depth;
    // memory = final LayerNorm (fp32 copy into x1-sized scratch only when the caller wants it)
    if (launch_layernorm(x, Ti, D, m->Dr, m->enc_norm.g, m->enc_norm.b, 1e-6f, mem, memory_out ? x : nullptr, nullptr, 1,
                         nullptr, 0, 0, st))
        return 1;
    if (memory_out)  // [T, real D] for the caller
        CK(cudaMemcpy2DAsync(memory_out, (size_t)m->Dr * 4, x, (size_t)D * 4, (size_t)m->Dr * 4, Ti,
                             cudaMemcpyDeviceToHost, st));
    // memory K/V once (the reference re-projects it in every AR step)
    if (Lin::run(mem, D, Ti, m->cross_kv, memkv, 2 * D, 0, ACT_NONE, nullptr, 0, 0, st, &flops)) return 1;
    // ---------------- AR decode (reference parseq.py:192-252)
    CK(cudaEventRecord(ev[1], st));
    // the ArState arrays live at capacity-based offsets: clear the whole block, not just the first rows
    CK(cudaMemsetAsync(ar_block, 0, 4 * ar_block_ints, st));
    if (launch_fill_i32(ar.tgt, pad_id, R, st)) return 1;
    if (launch_fill_i32(ar.rep_cut, -1, B, st)) return 1;
    {
        std::vector<int> first(B, bos);  // tgt[:, 0] = BOS
        CK(cudaMemcpy2DAsync(ar.tgt, sizeof(int) * S, first.data(), sizeof(int), sizeof(int), B, cudaMemcpyHostToDevice,
                             st));
        CK(cudaStreamSynchronize(st));
    }
    int steps_run = 0;
    const int hd_d = D / c.dec_heads;
    if (c.decode_ar) {
        // content K/V cache [row][position 0..S-1][2D]; position 0 (<bos>) is the same for every row
        if (launch_bcast_rows(m->ckv0, ckv, 2 * D * 2, (long long)S * 2 * D * 2, B, st)) return 1;
        // The decode loop can run as two PARTS (row ranges that end on a group boundary), each on its own stream, so
        // that one part's GEMMs overlap the other part's HBM-bound attention.  The step's kernels are latency-bound: halving
        // M does not halve their time, and the persistent GEMM CTAs (over 200 KB of shared memory each) do not co-reside -
        // so it is OFF unless YTK_AR_SPLIT_MIN=<rows> asks for it (tests/test_gpu_parseq.py runs both ways and compares them).  Parts share nothing but read-only weights / memory K/V.
        struct Part {
            int r0, rows, g0, ng;
            ArState a;
            cudaStream_t st;
            GemmPlan p_so, p_cq, p_co, p_l1, p_l2, p_hd, p_kv;
            double step_flops;
            int* flag;
            bool done;
        };
        int nparts = 1, split_row = B;
        {
            const char* ev_ = getenv("YTK_AR_SPLIT_MIN");
            const int split_min = ev_ ? atoi(ev_) : 0;
            bool sorted = true;
            int best = -1;
            for (int r = 1; r < B; ++r) {
                if (rg[r] < rg[r - 1]) sorted = false;
                if (rg[r] != rg[r - 1] && (best < 0 || std::abs(r - B / 2) < std::abs(best - B / 2))) best = r;
            }
            if (sorted && best > 0 && B >= split_min && split_min > 0) {
                nparts = 2;
                split_row = best;
            }
        }
        auto b16 = [](void* p, size_t elems) { return static_cast<void*>(reinterpret_cast<op_t*>(p) + elems); };
        // the [rows, C] logits are materialised only when the caller wants the AR logits themselves
        const bool fused_head = !(logits_out && c.refine_iters == 0) && getenv("YTK_NO_FUSED_HEAD") == nullptr;
        Part parts[2];
        for (int k = 0; k < nparts; ++k) {
            Part& p = parts[k];
            p.r0 = k == 0 ? 0 : split_row;
            p.rows = k == 0 ? split_row : B - split_row;
            if (nparts == 1) p.rows = B;
            p.g0 = nparts == 1 ? 0 : rg[p.r0];
            p.ng = nparts == 1 ? b.ngroups : rg[p.r0 + p.rows - 1] - p.g0 + 1;
            p.a = ar;
            p.a.tgt = ar.tgt + (size_t)p.r0 * S;
            p.a.raw = ar.raw + (size_t)p.r0 * S;
            p.a.rep_cut = ar.rep_cut + p.r0;
            p.a.rep_done = ar.rep_done + p.r0;
            p.a.has_eos = ar.has_eos + p.r0;
            p.a.n_active = ar.n_active + 4 * k;
            p.a.step = ar.step + 4 * k;
            p.a.ticket = ar.ticket + 4 * k;
            p.st = k == 0 ? st : st2;
            p.flag = host_flag + 2 * k;
            p.done = false;
            const size_t r0 = (size_t)p.r0;
            auto mk = [&](GemmPlan* pl, const void* A, long long lda, const LinearW& w, void* out, long long ldc,
                          int out_f32, int act, const void* resid, int resid_f32, long long ldr) {
                Epilogue ep;
                ep.bias = w.b;
                ep.resid = resid;
                ep.resid_f32 = resid_f32;
                ep.ldr = ldr;
                ep.out = out;
                ep.out_f32 = out_f32;
                ep.ldc = ldc;
                ep.act = act;
                return gemm_plan_create(pl, A, lda, p.rows, w.K, w.w, w.N, ep);
            };
            float* x1p = x1 + r0 * D;
            if (mk(&p.p_so, b16(sa, r0 * D), D, m->self_out, x1p, D, 1, ACT_NONE, nullptr, 0, 0)) return 1;
            if (mk(&p.p_cq, b16(hb, r0 * D), D, m->cross_q, b16(qc, r0 * D), D, 0, ACT_NONE, nullptr, 0, 0)) return 1;
            if (mk(&p.p_co, b16(oc, r0 * D), D, m->cross_out, x1p, D, 1, ACT_NONE, x1p, 1, D)) return 1;
            if (mk(&p.p_l1, b16(hb, r0 * D), D, m->lin1, b16(mlpb, r0 * m->lin1.N), m->lin1.N, 0, ACT_GELU, nullptr, 0, 0))
                return 1;
            if (mk(&p.p_l2, b16(mlpb, r0 * m->lin1.N), m->lin1.N, m->lin2, x1p, D, 1, ACT_NONE, x1p, 1, D)) return 1;
            if (fused_head) {
                // head GEMM with the row-max epilogue: (max, sum exp, arg-max) partials instead of [rows, C] fp32 logits
                // (the partials live in the logits buffer: 16 bytes x 2 * tiles_n per row)
                Epilogue ep;
                ep.bias = m->head.b;
                ep.out = logits + r0 * ldl;
                ep.out_f32 = 1;
                ep.mode = EPI_ROWMAX;
                ep.act = c.refine_iters == 0 ? ACT_NONE : ACT_RELU;   // arg-max only unless the AR logits ARE the output
                if (gemm_plan_create(&p.p_hd, b16(hb, r0 * D), D, p.rows, m->head.K, m->head.w, m->head.N, ep)) return 1;
                // partial rows start at float4 index row * ldc: re-base this part's output inside the shared buffer
                p.p_hd.args.out = reinterpret_cast<float4*>(logits) + r0 * p.p_hd.args.ldc;
            } else if (mk(&p.p_hd, b16(hb, r0 * D), D, m->head, logits + r0 * ldl, ldl, 1, ACT_NONE, nullptr, 0, 0)) return 1;
            if (mk(&p.p_kv, b16(cin, r0 * D), D, m->self_kv, b16(ckv, r0 * S * 2 * D), (long long)S * 2 * D, 0, ACT_NONE,
                   nullptr, 0, 0))
                return 1;
            p.step_flops = p.p_so.flops + p.p_cq.flops + p.p_co.flops + p.p_l1.flops + p.p_l2.flops + p.p_hd.flops +
                           p.p_kv.flops;
        }
        if (nparts > 1) {  // fork: the second stream starts after everything issued so far
            CK(cudaEventRecord(ev_fork, st));
            CK(cudaStreamWaitEvent(st2, ev_fork, 0));
        }
        auto launch_step = [&](Part& p, int i) -> int {
            const size_t r0 = (size_t)p.r0;
            cudaStream_t ps = p.st;
            float* x1p = x1 + r0 * D;
            void* hbp = b16(hb, r0 * D);
            float* lg = logits + r0 * ldl;
            const long long ldp = p.p_hd.args.ldc;              // fused head: float4 partials per row
            const int npart = fused_head ? (int)ldp : 0;
            if (fused_head) lg = reinterpret_cast<float*>(reinterpret_cast<float4*>(logits) + r0 * ldp);
            if (launch_dec_self_attn(m->q_self, b16(ckv, r0 * S * 2 * D), p.rows, S, D, c.dec_heads, p.a.step,
                                     b16(sa, r0 * D), ps))
                return 1;
            if (gemm_plan_launch(&p.p_so, ps)) return 1;
            // x1 += pos_queries[i] (the query stream's residual input), then norm1
            if (launch_layernorm(x1p, p.rows, D, m->Dr, m->norm1.g, m->norm1.b, 1e-5f, hbp, nullptr, m->pos_q, 1, p.a.step, 0,
                                 1, ps))
                return 1;
            if (gemm_plan_launch(&p.p_cq, ps)) return 1;
            if (launch_dec_cross_attn(b16(qc, r0 * D), memkv, descs_dev + p.r0, p.rows, D, c.dec_heads, b16(oc, r0 * D), ps))
                return 1;
            if (gemm_plan_launch(&p.p_co, ps)) return 1;
            if (launch_layernorm(x1p, p.rows, D, m->Dr, m->norm2.g, m->norm2.b, 1e-5f, hbp, nullptr, nullptr, 1, nullptr, 0, 0,
                                 ps))
                return 1;
            if (gemm_plan_launch(&p.p_l1, ps)) return 1;
            if (gemm_plan_launch(&p.p_l2, ps)) return 1;
            if (launch_layernorm(x1p, p.rows, D, m->Dr, m->dec_norm.g, m->dec_norm.b, 1e-5f, hbp, nullptr, nullptr, 1, nullptr,
                                 0, 0, ps))
                return 1;
            if (gemm_plan_launch(&p.p_hd, ps)) return 1;
            if (c.refine_iters == 0) {
                if (fused_head) {
                    if (launch_rowmax_finalize(lg, ldp, npart, C, p.rows, S, S, i, nullptr, eos, ids + r0 * S,
                                               probs + r0 * S, ps))
                        return 1;
                } else if (launch_softmax_max(lg, ldl, C, p.rows, S, S, i, nullptr, eos, ids + r0 * S, probs + r0 * S, ps))
                    return 1;
                if (logits_out)
                    CK(cudaMemcpy2DAsync(logits_out + (r0 * S + (size_t)i) * C, (size_t)S * C * 4, lg, ldl * 4,
                                         (size_t)C * 4, p.rows,
                                         logits_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, ps));
            }
            if (launch_ar_control(lg, fused_head ? ldp : ldl, C, npart, p.rows, S, row_group + p.r0, p.g0, p.ng, p.a, eos,
                                  c.rep_on, c.rep_period_max,
                                  c.rep_min_run_p1, c.rep_min_repeats, m->embed, m->pos_q, D, m->Dr, m->norm_c.g, m->norm_c.b,
                                  b16(cin, r0 * D), ps))
                return 1;
            flops += p.step_flops;
            if (i + 1 < S) {
                // K/V of the token that just entered the context: position i+1 of every row of the part
                if (gemm_plan_set_out(&p.p_kv, reinterpret_cast<op_t*>(ckv) + r0 * S * 2 * D + (size_t)(i + 1) * 2 * D))
                    return 1;
                if (gemm_plan_launch(&p.p_kv, ps)) return 1;
            }
            return 0;
        };
        for (int i = 0; i < S; ++i) {
            bool any = false;
            for (int k = 0; k < nparts; ++k)
                if (!parts[k].done) {
                    if (launch_step(parts[k], i)) return 1;
                    any = true;
                }
            if (!any) break;
            steps_run = i + 1;
            // early stop: peek at the device-side counters every 4 steps (no sync on the other steps)
            if ((i & 3) == 3 || i + 1 == S) {
                for (int k = 0; k < nparts; ++k)
                    if (!parts[k].done)
                        CK(cudaMemcpyAsync(parts[k].flag, parts[k].a.n_active, 2 * sizeof(int), cudaMemcpyDeviceToHost,
                                           parts[k].st));
                bool all = true;
                for (int k = 0; k < nparts; ++k)
                    if (!parts[k].done) {
                        CK(cudaStreamSynchronize(parts[k].st));
                        if (parts[k].flag[0] == 0) parts[k].done = true;
                        else all = false;
                    }
                if (all) break;
            }
        }
        if (nparts > 1) {  // join
            CK(cudaEventRecord(ev_join, st2));
            CK(cudaStreamWaitEvent(st, ev_join, 0));
        }
    } else {
        // decode_ar == 0 (parseq.py:252-262): no AR loop; the first decoder pass below sees only <bos> as context
        if (launch_fill_i32(ar.group_len, S, b.ngroups, st)) return 1;
        steps_run = S;
    }
    last_steps = steps_run;
    CK(cudaEventRecord(ev[2], st));
    if (c.decode_ar)
        for (const CropDesc& d : b.descs) flops += 4.0 * d.ntok * (double)D * steps_run;  // cross attention
    // Decoder passes over all S queries (reference parseq.py:252-299): with decode_ar == 0 a first pass whose context is
    // <bos> alone, then `refine_iters` passes whose context is [<bos>, arg-max of the previous logits[:, :-1]].
    const int n_pass = c.refine_iters + (c.decode_ar ? 0 : 1);
    if (n_pass == 0) {
        if (launch_apply_rep_cut(ar.rep_cut, B, S, C, eos, ids, probs, st)) return 1;
    } else {
        if (launch_fill_i32(glen_const, S, b.ngroups, st)) return 1;
        if (launch_fill_i32(glen_const + cap_groups, 1, b.ngroups, st)) return 1;
    }
    for (int pass = 0; pass < n_pass; ++pass) {
        const bool first = pass == 0, final = pass + 1 == n_pass;
        // context tokens: raw[row][p-1] is the token at position p >= 1; L (per group) = context length
        const int* raw = (first && c.decode_ar) ? ar.raw : ids;
        const int* glen = first ? (c.decode_ar ? ar.group_len : glen_const + cap_groups) : glen_const;
        if (launch_refine_embed(raw, row_group, glen, B, S, bos, eos, m->embed, m->pos_q, D, m->Dr, m->norm_c.g,
                                m->norm_c.b, cin, klen, kpad, st))
            return 1;
        if (Lin::run(cin, D, R, m->self_kv, ckv, 2 * D, 0, ACT_NONE, nullptr, 0, 0, st, &flops)) return 1;
        // masked tensor-core attention: 101 shared queries x the row's content keys (cache layout [row][pos][2D]);
        // rows 0/1 see every key, row q >= 2 the keys <= q, nobody sees keys at/after the first EOS (Appendix A1)
        if (launch_refine_seqs(klen, kpad, B, S, D, seqs_self, st)) return 1;
        {
            const op_t* ck = reinterpret_cast<const op_t*>(ckv);
            if (launch_flash_attention(m->q_self, D, S, ck, ck + D, 2 * D, R, sa, D, seqs_self, B, S,
                                       c.dec_heads, hd_d, 1, st))
                return 1;
        }
        if (Lin::run(sa, D, R, m->self_out, x1, D, 1, ACT_NONE, nullptr, 0, 0, st, &flops)) return 1;
        if (launch_layernorm(x1, R, D, m->Dr, m->norm1.g, m->norm1.b, 1e-5f, hb, nullptr, m->pos_q, S, nullptr, 0, 1, st))
            return 1;
        if (Lin::run(hb, D, R, m->cross_q, qc, D, 0, ACT_NONE, nullptr, 0, 0, st, &flops)) return 1;
        const op_t* kv = reinterpret_cast<const op_t*>(memkv);
        if (launch_flash_attention(qc, D, R, kv, kv + D, 2 * D, Ti, oc, D, seqs_ref, B, S, c.dec_heads, hd_d, 0, st))
            return 1;
        for (const CropDesc& d : b.descs) flops += 4.0 * S * (double)d.ntok * D;
        if (Lin::run(oc, D, R, m->cross_out, x1, D, 1, ACT_NONE, x1, 1, D, st, &flops)) return 1;
        if (launch_layernorm(x1, R, D, m->Dr, m->norm2.g, m->norm2.b, 1e-5f, hb, nullptr, nullptr, 1, nullptr, 0, 0, st))
            return 1;
        if (Lin::run(hb, D, R, m->lin1, mlpb, m->lin1.N, 0, ACT_GELU, nullptr, 0, 0, st, &flops)) return 1;
        if (Lin::run(mlpb, m->lin1.N, R, m->lin2, x1, D, 1, ACT_NONE, x1, 1, D, st, &flops)) return 1;
        if (launch_layernorm(x1, R, D, m->Dr, m->dec_norm.g, m->dec_norm.b, 1e-5f, hb, nullptr, nullptr, 1, nullptr, 0, 0, st))
            return 1;
        for (int r0 = 0; r0 < R; r0 += logits_rows) {
            const int rows = std::min(logits_rows, R - r0);
            const op_t* a = reinterpret_cast<const op_t*>(hb) + (size_t)r0 * D;
            const bool want_logits = logits_out && final;
            if (!want_logits && getenv("YTK_NO_FUSED_HEAD") == nullptr) {
                // head GEMM -> softmax statistics in the epilogue: only (id, probability) per position exist in HBM
                Epilogue ep;
                ep.bias = m->head.b;
                ep.out = logits;
                ep.out_f32 = 1;
                ep.mode = EPI_ROWMAX;
                GemmPlan hp;
                if (gemm_plan_create(&hp, a, D, rows, m->head.K, m->head.w, m->head.N, ep)) return 1;
                flops += hp.flops;
                if (gemm_plan_launch(&hp, st)) return 1;
                if (launch_rowmax_finalize(logits, hp.args.ldc, (int)hp.args.ldc, C, rows, S, 1, r0,
                                           final ? ar.rep_cut : nullptr, eos, ids, probs, st))
                    return 1;
                continue;
            }
            if (Lin::run(a, D, rows, m->head, logits, ldl, 1, ACT_NONE, nullptr, 0, 0, st, &flops)) return 1;
            // the repetition patch (parseq.py:301-309) applies to the final logits only
            if (launch_softmax_max(logits, ldl, C, rows, S, 1, r0, final ? ar.rep_cut : nullptr, eos, ids, probs, st))
                return 1;
            if (logits_out && final) {
                // model-level seam: materialise the (B, 101, C) logits; the repetition patch is applied by the caller
                CK(cudaMemcpy2DAsync(logits_out + (size_t)r0 * C, (size_t)C * 4, logits, ldl * 4, (size_t)C * 4, rows,
                                     logits_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st));
            }
        }
    }
    CK(cudaEventRecord(ev[3], st));
    CK(cudaMemcpyAsync(ids_out, ids, 4 * (size_t)R, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(probs_out, probs, 4 * (size_t)R, cudaMemcpyDeviceToHost, st));
    if (group_len_out) CK(cudaMemcpyAsync(group_len_out, ar.group_len, 4 * (size_t)b.ngroups, cudaMemcpyDeviceToHost, st));
    CK(cudaEventRecord(ev[4], st));
    CK(cudaStreamSynchronize(st));
    for (int i = 0; i < 4; ++i) cudaEventElapsedTime(&phase_ms[i], ev[i], ev[i + 1]);
    return 0;
}

}  // namespace ytk
