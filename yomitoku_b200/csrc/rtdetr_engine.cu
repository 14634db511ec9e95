// RT-DETRv2 (PResNet-50d backbone + HybridEncoder + 6-layer deformable decoder) as a static launch plan: every
// convolution and linear layer is a wgmma implicit GEMM (gemm_tc.cu), the two kinds of self-attention run on the wgmma
// attention kernel (attn_tc.cu), the rest are the small kernels of rtdetr_ops.cu.  Replaces, for inference, reference
// models/rtdetr.py:9-22 = layers/rtdetr_backbone.py:245-334 + layers/rtdetr_hybrid_encoder.py:216-410 +
// layers/rtdetrv2_decoder.py:446-815 (the layout parser, the table structure recognizer and the table cell detector share
// the architecture; the image size and the query count come from the config: 640 / 300 or 960 / 1500).
//
// Data layout in HBM: activations NHWC fp16 (BatchNorm folded into weights / bias, RepVgg blocks re-parameterised into
// one 3x3 convolution); the decoder's token matrices are level-major (rtdetr_ops.h) so that a level IS the NHWC output of
// its 1x1 projection; the decoder state (num_queries rows per image) is fp32 with an fp16 copy as GEMM operand; the value
// projections of all six decoder layers are one GEMM (256 -> 1536) over the memory.
#include "rtdetr_engine.h"

#include <cmath>
#include <cstring>

#include "dbnet_ops.h"
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

namespace {

int up(std::vector<void*>& owned, const void* host, size_t bytes, void** dev) {
    CK(cudaMalloc(dev, bytes));
    CK(cudaMemcpy(*dev, host, bytes, cudaMemcpyHostToDevice));
    owned.push_back(*dev);
    return 0;
}

int bn_fold(const WeightSet& ws, const std::string& p, int C, std::vector<float>& scale, std::vector<float>& shift) {
    const TensorView *g = ws.need(p + ".weight", C), *b = ws.need(p + ".bias", C), *m = ws.need(p + ".running_mean", C),
                     *v = ws.need(p + ".running_var", C);
    if (!g || !b || !m || !v) return 1;
    scale.resize(C);
    shift.resize(C);
    for (int c = 0; c < C; ++c) {
        const float s = g->data[c] / std::sqrt(v->data[c] + 1e-5f);
        scale[c] = s;
        shift[c] = b->data[c] - m->data[c] * s;
    }
    return 0;
}

// fp32 [Cout][Cin][k][k] (already scaled) -> fp16 [CoutP][k][k][CinP] on the device, zero padded; bias [CoutP]
int upload_conv(std::vector<void*>& owned, const std::vector<float>& w, const std::vector<float>& bias, int Cout, int Cin,
                int k, int stride, ConvW* out) {
    const int CinP = (Cin + 63) / 64 * 64, CoutP = Cout < 64 ? 64 : Cout;
    std::vector<uint16_t> p((size_t)CoutP * k * k * CinP, 0);
    for (int co = 0; co < Cout; ++co)
        for (int ci = 0; ci < Cin; ++ci)
            for (int r = 0; r < k; ++r)
                for (int s = 0; s < k; ++s)
                    p[(((size_t)co * k + r) * k + s) * CinP + ci] = f2op_host(w[(((size_t)co * Cin + ci) * k + r) * k + s]);
    std::vector<float> b(CoutP, 0.f);
    for (int c = 0; c < Cout; ++c) b[c] = bias[c];
    void* d = nullptr;
    if (up(owned, p.data(), p.size() * 2, &out->w) || up(owned, b.data(), b.size() * 4, &d)) return 1;
    out->bias = reinterpret_cast<float*>(d);
    out->Cout = CoutP;
    out->Cin = CinP;
    out->k = k;
    out->stride = stride;
    out->pad = (k - 1) / 2;
    out->dil = 1;
    return 0;
}

// ConvNormLayer (conv without bias + BatchNorm, rtdetr_backbone.py:32-56 / rtdetr_hybrid_encoder.py:25-50)
int load_conv_norm(std::vector<void*>& owned, const WeightSet& ws, const std::string& p, int Cout, int Cin, int k,
                   int stride, ConvW* out) {
    const TensorView* w = ws.need(p + ".conv.weight", (long long)Cout * Cin * k * k);
    std::vector<float> scale, shift;
    if (!w || bn_fold(ws, p + ".norm", Cout, scale, shift)) return 1;
    std::vector<float> f((size_t)Cout * Cin * k * k);
    const size_t per = (size_t)Cin * k * k;
    for (int co = 0; co < Cout; ++co)
        for (size_t i = 0; i < per; ++i) f[co * per + i] = w->data[co * per + i] * scale[co];
    return upload_conv(owned, f, shift, Cout, Cin, k, stride, out);
}

// RepVggBlock (rtdetr_hybrid_encoder.py:125-178): conv3x3+BN and conv1x1+BN summed -> one 3x3 kernel + bias
int load_repvgg(std::vector<void*>& owned, const WeightSet& ws, const std::string& p, int C, ConvW* out) {
    const TensorView *w3 = ws.need(p + ".conv1.conv.weight", (long long)C * C * 9),
                     *w1 = ws.need(p + ".conv2.conv.weight", (long long)C * C);
    std::vector<float> s3, b3, s1, b1;
    if (!w3 || !w1 || bn_fold(ws, p + ".conv1.norm", C, s3, b3) || bn_fold(ws, p + ".conv2.norm", C, s1, b1)) return 1;
    std::vector<float> f((size_t)C * C * 9), bias(C);
    for (int co = 0; co < C; ++co) {
        for (int ci = 0; ci < C; ++ci) {
            for (int t = 0; t < 9; ++t) f[((size_t)co * C + ci) * 9 + t] = w3->data[((size_t)co * C + ci) * 9 + t] * s3[co];
            f[((size_t)co * C + ci) * 9 + 4] += w1->data[(size_t)co * C + ci] * s1[co];
        }
        bias[co] = b3[co] + b1[co];
    }
    return upload_conv(owned, f, bias, C, C, 3, 1, out);
}

int upload_linear(std::vector<void*>& owned, const float* w, const float* b, int N, int K, RtLinear* out) {
    const int Kp = (K + 63) / 64 * 64;
    std::vector<uint16_t> p((size_t)N * Kp, 0);
    for (int n = 0; n < N; ++n)
        for (int k = 0; k < K; ++k) p[(size_t)n * Kp + k] = f2op_host(w[(size_t)n * K + k]);
    void* d = nullptr;
    if (up(owned, p.data(), p.size() * 2, &out->w) || up(owned, b, (size_t)N * 4, &d)) return 1;
    out->b = reinterpret_cast<float*>(d);
    out->N = N;
    out->K = Kp;
    return 0;
}

int load_linear(std::vector<void*>& owned, const WeightSet& ws, const std::string& p, int N, int K, RtLinear* out) {
    const TensorView *w = ws.need(p + ".weight", (long long)N * K), *b = ws.need(p + ".bias", N);
    if (!w || !b) return 1;
    return upload_linear(owned, w->data, b->data, N, K, out);
}

// rows [r0, r1) of a packed in_proj (nn.MultiheadAttention) as their own linear layer
int load_in_proj(std::vector<void*>& owned, const WeightSet& ws, const std::string& p, int D, int r0, int r1,
                 RtLinear* out) {
    const TensorView *w = ws.need(p + ".in_proj_weight", 3LL * D * D), *b = ws.need(p + ".in_proj_bias", 3LL * D);
    if (!w || !b) return 1;
    return upload_linear(owned, w->data + (size_t)r0 * D, b->data + r0, r1 - r0, D, out);
}

int load_ln(std::vector<void*>& owned, const WeightSet& ws, const std::string& p, int D, RtLn* out) {
    const TensorView *g = ws.need(p + ".weight", D), *b = ws.need(p + ".bias", D);
    void *dg = nullptr, *db = nullptr;
    if (!g || !b || up(owned, g->data, D * 4, &dg) || up(owned, b->data, D * 4, &db)) return 1;
    out->g = reinterpret_cast<float*>(dg);
    out->b = reinterpret_cast<float*>(db);
    return 0;
}

}  // namespace

int RtdetrModel::load(const WeightSet& ws, const RtCfg& c) {
    cfg = c;
    const int D = c.hidden;
    if (D != 256 || c.heads != 8 || c.img % 32 || c.num_points != 4) {
        set_error("RT-DETRv2: hidden %d / heads %d / img %d / points %d unsupported", D, c.heads, c.img, c.num_points);
        return 1;
    }
    // ---- backbone (PResNet-50, variant d)
    const std::string bb = "backbone.";
    if (load_conv_norm(owned, ws, bb + "conv1.conv1_1", 32, 3, 3, 2, &stem[0])) return 1;
    if (load_conv_norm(owned, ws, bb + "conv1.conv1_2", 32, 32, 3, 1, &stem[1])) return 1;
    if (load_conv_norm(owned, ws, bb + "conv1.conv1_3", 64, 32, 3, 1, &stem[2])) return 1;
    const int planes[4] = {64, 128, 256, 512}, nblk[4] = {3, 4, 6, 3};
    int cin = 64;
    for (int s = 0; s < 4; ++s)
        for (int b = 0; b < nblk[s]; ++b) {
            RtBottleneck bk;
            const std::string p = bb + "res_layers." + std::to_string(s) + ".blocks." + std::to_string(b);
            const int stride = (b == 0 && s != 0) ? 2 : 1;
            if (load_conv_norm(owned, ws, p + ".branch2a", planes[s], cin, 1, 1, &bk.a)) return 1;
            if (load_conv_norm(owned, ws, p + ".branch2b", planes[s], planes[s], 3, stride, &bk.b)) return 1;
            if (load_conv_norm(owned, ws, p + ".branch2c", planes[s] * 4, planes[s], 1, 1, &bk.c)) return 1;
            bk.has_short = (b == 0);
            bk.pool = (stride == 2);
            if (bk.has_short &&
                load_conv_norm(owned, ws, p + (bk.pool ? ".short.conv" : ".short"), planes[s] * 4, cin, 1, 1, &bk.shortc))
                return 1;
            blocks[s].push_back(bk);
            cin = planes[s] * 4;
        }
    // ---- hybrid encoder
    const std::string en = "encoder.";
    const int cins[3] = {512, 1024, 2048};
    for (int i = 0; i < 3; ++i) {
        // input_proj.{i} = conv + norm under the names "conv" / "norm": the ConvNormLayer key pattern
        if (load_conv_norm(owned, ws, en + "input_proj." + std::to_string(i), D, cins[i], 1, 1, &enc_proj[i])) return 1;
        if (load_conv_norm(owned, ws, "decoder.input_proj." + std::to_string(i), D, D, 1, 1, &dec_proj[i])) return 1;
    }
    {
        const std::string p = en + "encoder.0.layers.0";
        if (load_in_proj(owned, ws, p + ".self_attn", D, 0, 2 * D, &aifi_qk)) return 1;
        if (load_in_proj(owned, ws, p + ".self_attn", D, 2 * D, 3 * D, &aifi_v)) return 1;
        if (load_linear(owned, ws, p + ".self_attn.out_proj", D, D, &aifi_out)) return 1;
        if (load_linear(owned, ws, p + ".linear1", c.ffn, D, &aifi_l1)) return 1;
        if (load_linear(owned, ws, p + ".linear2", D, c.ffn, &aifi_l2)) return 1;
        if (load_ln(owned, ws, p + ".norm1", D, &aifi_n1) || load_ln(owned, ws, p + ".norm2", D, &aifi_n2)) return 1;
    }
    auto load_csp = [&](const std::string& p, RtCsp* out) {
        if (load_conv_norm(owned, ws, p + ".conv1", D, 2 * D, 1, 1, &out->conv1)) return 1;
        if (load_conv_norm(owned, ws, p + ".conv2", D, 2 * D, 1, 1, &out->conv2)) return 1;
        for (int i = 0; i < 3; ++i)
            if (load_repvgg(owned, ws, p + ".bottlenecks." + std::to_string(i), D, &out->rep[i])) return 1;
        return 0;
    };
    for (int i = 0; i < 2; ++i) {
        if (load_conv_norm(owned, ws, en + "lateral_convs." + std::to_string(i), D, D, 1, 1, &lateral[i])) return 1;
        if (load_conv_norm(owned, ws, en + "downsample_convs." + std::to_string(i), D, D, 3, 2, &down[i])) return 1;
        if (load_csp(en + "fpn_blocks." + std::to_string(i), &fpn[i])) return 1;
        if (load_csp(en + "pan_blocks." + std::to_string(i), &pan[i])) return 1;
    }
    {
        // 2-D sin-cos position embedding of the stride-32 map (rtdetr_hybrid_encoder.py:334-354): rows in raster order
        // (h major), features [sin(w omega), cos(w omega), sin(h omega), cos(h omega)]
        const int g = c.img / 32, pd = D / 4;
        std::vector<float> pe((size_t)g * g * D);
        for (int h = 0; h < g; ++h)
            for (int w = 0; w < g; ++w)
                for (int k = 0; k < pd; ++k) {
                    const float omega = 1.0f / std::pow(10000.0f, (float)k / (float)pd);
                    // the reference flattens a meshgrid(indexing="ij") over (w, h): row index = w_idx * h_count + h_idx
                    // with grid_w = w_idx and grid_h = h_idx; the token at raster position (y, x) is row y * g + x, so
                    // the reference pairs token r with grid_w = r / g and grid_h = r % g
                    float* row = &pe[((size_t)h * g + w) * D];
                    const float a = (float)h * omega, b2 = (float)w * omega;
                    row[k] = std::sin(a);
                    row[pd + k] = std::cos(a);
                    row[2 * pd + k] = std::sin(b2);
                    row[3 * pd + k] = std::cos(b2);
                }
        void* d = nullptr;
        if (up(owned, pe.data(), pe.size() * 4, &d)) return 1;
        pos_embed = reinterpret_cast<float*>(d);
    }
    // ---- decoder
    const std::string de = "decoder.";
    lv.n = 3;
    lv.off[0] = 0;
    for (int l = 0; l < 3; ++l) {
        lv.h[l] = lv.w[l] = c.img / (8 << l);
        lv.points[l] = c.num_points;
        lv.off[l + 1] = lv.off[l] + lv.h[l] * lv.w[l];
    }
    lv.total = lv.off[3];
    {
        const TensorView *a = ws.need(de + "anchors", (long long)lv.total * 4), *v = ws.find(de + "valid_mask");
        if (!a) return 1;
        std::vector<int> bad;
        for (int i = 0; i < lv.total; ++i) {
            bool ok = true;
            for (int k = 0; k < 4; ++k) ok = ok && std::isfinite(a->data[(size_t)i * 4 + k]);
            if (v && v->numel() == lv.total) ok = v->data[i] != 0.f;
            if (!ok) bad.push_back(i);
        }
        void *da = nullptr, *dv = nullptr;
        if (up(owned, a->data, (size_t)lv.total * 16, &da)) return 1;
        anchors = reinterpret_cast<float*>(da);
        n_invalid = (int)bad.size();
        if (n_invalid) {
            if (up(owned, bad.data(), bad.size() * 4, &dv)) return 1;
            invalid = reinterpret_cast<int*>(dv);
        }
    }
    if (load_linear(owned, ws, de + "enc_output.proj", D, D, &enc_out) || load_ln(owned, ws, de + "enc_output.norm", D, &enc_out_ln))
        return 1;
    if (load_linear(owned, ws, de + "enc_score_head", c.num_classes, D, &enc_score)) return 1;
    if (load_linear(owned, ws, de + "enc_bbox_head.layers.0", D, D, &enc_box0) ||
        load_linear(owned, ws, de + "enc_bbox_head.layers.1", D, D, &enc_box1) ||
        load_linear(owned, ws, de + "enc_bbox_head.layers.2", 4, D, &enc_box2))
        return 1;
    {
        const TensorView *w = ws.need(de + "query_pos_head.layers.0.weight", 2LL * D * 4),
                         *b = ws.need(de + "query_pos_head.layers.0.bias", 2LL * D);
        void *dw = nullptr, *db = nullptr;
        if (!w || !b || up(owned, w->data, (size_t)2 * D * 16, &dw) || up(owned, b->data, (size_t)2 * D * 4, &db)) return 1;
        qpos0_w = reinterpret_cast<float*>(dw);
        qpos0_b = reinterpret_cast<float*>(db);
        if (load_linear(owned, ws, de + "query_pos_head.layers.1", D, 2 * D, &qpos1)) return 1;
    }
    const int P = 3 * c.num_points;
    std::vector<float> vw((size_t)c.num_layers * D * D), vb((size_t)c.num_layers * D);
    layers.resize(c.num_layers);
    for (int i = 0; i < c.num_layers; ++i) {
        RtDecLayer& L = layers[i];
        const std::string p = de + "decoder.layers." + std::to_string(i);
        if (load_in_proj(owned, ws, p + ".self_attn", D, 0, 2 * D, &L.qk) ||
            load_in_proj(owned, ws, p + ".self_attn", D, 2 * D, 3 * D, &L.v) ||
            load_linear(owned, ws, p + ".self_attn.out_proj", D, D, &L.out))
            return 1;
        {
            const std::string ca = p + ".cross_attn";
            const TensorView *so_w = ws.need(ca + ".sampling_offsets.weight", (long long)c.heads * P * 2 * D),
                             *so_b = ws.need(ca + ".sampling_offsets.bias", (long long)c.heads * P * 2),
                             *aw_w = ws.need(ca + ".attention_weights.weight", (long long)c.heads * P * D),
                             *aw_b = ws.need(ca + ".attention_weights.bias", (long long)c.heads * P),
                             *v_w = ws.need(ca + ".value_proj.weight", (long long)D * D), *v_b = ws.need(ca + ".value_proj.bias", D);
            if (!so_w || !so_b || !aw_w || !aw_b || !v_w || !v_b) return 1;
            const int n_so = c.heads * P * 2, n_aw = c.heads * P;
            std::vector<float> w((size_t)(n_so + n_aw) * D), b(n_so + n_aw);
            memcpy(w.data(), so_w->data, (size_t)n_so * D * 4);
            memcpy(w.data() + (size_t)n_so * D, aw_w->data, (size_t)n_aw * D * 4);
            memcpy(b.data(), so_b->data, n_so * 4);
            memcpy(b.data() + n_so, aw_b->data, n_aw * 4);
            if (upload_linear(owned, w.data(), b.data(), n_so + n_aw, D, &L.ow)) return 1;
            memcpy(&vw[(size_t)i * D * D], v_w->data, (size_t)D * D * 4);
            memcpy(&vb[(size_t)i * D], v_b->data, D * 4);
            if (load_linear(owned, ws, ca + ".output_proj", D, D, &L.cross_out)) return 1;
        }
        if (load_linear(owned, ws, p + ".linear1", c.ffn, D, &L.lin1) || load_linear(owned, ws, p + ".linear2", D, c.ffn, &L.lin2))
            return 1;
        if (load_ln(owned, ws, p + ".norm1", D, &L.n1) || load_ln(owned, ws, p + ".norm2", D, &L.n2) ||
            load_ln(owned, ws, p + ".norm3", D, &L.n3))
            return 1;
        const std::string bh = de + "dec_bbox_head." + std::to_string(i) + ".layers.";
        if (load_linear(owned, ws, bh + "0", D, D, &L.box0) || load_linear(owned, ws, bh + "1", D, D, &L.box1) ||
            load_linear(owned, ws, bh + "2", 4, D, &L.box2))
            return 1;
    }
    if (upload_linear(owned, vw.data(), vb.data(), c.num_layers * D, D, &value_all)) return 1;
    if (load_linear(owned, ws, de + "dec_score_head." + std::to_string(c.num_layers - 1), c.num_classes, D, &score_last))
        return 1;
    return 0;
}

RtdetrModel::~RtdetrModel() {
    for (void* p : owned) cudaFree(p);
}

// ---------------------------------------------------------------------------------------------- engine
int RtdetrEngine::alloc(const std::string& name, long long rows, int c, bool f32, void** out, int n, int h, int w) {
    const size_t bytes = (size_t)rows * c * (f32 ? 4 : 2);
    void* p = nullptr;
    CK(cudaMalloc(&p, bytes));
    CK(cudaMemset(p, 0, bytes));
    bufs.push_back(p);
    total_bytes += bytes;
    if (!name.empty()) dbg[name] = n ? DebugTensor{p, n, h, w, c, f32} : DebugTensor{p, 1, 1, (int)rows, c, f32};
    *out = p;
    return 0;
}

int RtdetrEngine::conv(const ConvW& cw, const void* in, int n, int h, int w, long long in_ld, void* out, long long ldc,
                       int act, const void* resid, long long ldr) {
    ConvGeom g{n, h, w, cw.Cin, in_ld, cw.k, cw.k, cw.stride, cw.pad, cw.dil, cw.Cout};
    Epilogue e;
    e.bias = cw.bias;
    e.resid = resid;
    e.ldr = ldr;
    e.out = out;
    e.ldc = ldc;
    e.act = act;
    auto plan = std::make_shared<GemmPlan>();
    if (conv_plan_create(plan.get(), in, g, cw.w, e)) return 1;
    flops += plan->flops;
    steps.push_back([plan](cudaStream_t st) { return gemm_plan_launch(plan.get(), st); });
    return 0;
}

int RtdetrEngine::linear(const RtLinear& w, const void* A, long long lda, int M, void* out, long long ldc, bool out_f32,
                         int act, const void* resid, bool resid_f32, long long ldr) {
    Epilogue e;
    e.bias = w.b;
    e.resid = resid;
    e.resid_f32 = resid_f32 ? 1 : 0;
    e.ldr = ldr;
    e.out = out;
    e.out_f32 = out_f32 ? 1 : 0;
    e.ldc = ldc;
    e.act = act;
    auto plan = std::make_shared<GemmPlan>();
    if (gemm_plan_create(plan.get(), A, lda, M, w.K, w.w, w.N, e)) return 1;
    flops += plan->flops;
    steps.push_back([plan](cudaStream_t st) { return gemm_plan_launch(plan.get(), st); });
    return 0;
}

// CSPRepLayer (rtdetr_hybrid_encoder.py:181-213, expansion 1.0): out = RepVgg^3(conv1(x)) + conv2(x)
int RtdetrEngine::csp(const RtCsp& c, const std::string& name, const void* cat, int n, int h, int w, void* out) {
    const int D = m->cfg.hidden;
    const long long rows = (long long)n * h * w;
    void *t1, *t2, *x2;
    if (alloc(name + ".t1", rows, D, false, &t1, n, h, w) || alloc(name + ".t2", rows, D, false, &t2, n, h, w) ||
        alloc(name + ".x2", rows, D, false, &x2, n, h, w))
        return 1;
    if (conv(c.conv1, cat, n, h, w, 2 * D, t1, D, ACT_SILU)) return 1;
    if (conv(c.rep[0], t1, n, h, w, D, t2, D, ACT_SILU)) return 1;
    if (conv(c.rep[1], t2, n, h, w, D, t1, D, ACT_SILU)) return 1;
    if (conv(c.rep[2], t1, n, h, w, D, t2, D, ACT_SILU)) return 1;
    if (conv(c.conv2, cat, n, h, w, 2 * D, x2, D, ACT_SILU)) return 1;
    steps.push_back([=](cudaStream_t st) { return launch_rt_add(t2, x2, nullptr, D, 1, out, rows, st); });
    return 0;
}

int RtdetrEngine::build(const RtdetrModel& model, int n) {
    m = &model;
    N = n;
    const RtCfg& c = model.cfg;
    const int D = c.hidden, S = c.img, K = c.num_queries, C = c.num_classes;
    const RtLevels lv = model.lv;
    // ---- input + stem
    void *x0, *s1, *s2, *s3, *pool;
    if (alloc("input", (long long)N * S * S, 64, false, &x0, N, S, S)) return 1;
    input = x0;
    {
        void* f = nullptr;
        CK(cudaMalloc(&f, (size_t)N * 3 * S * S * 4));
        bufs.push_back(f);
        in_f32 = reinterpret_cast<float*>(f);
    }
    const int S2 = S / 2, S4 = S / 4;
    if (alloc("stem1", (long long)N * S2 * S2, 64, false, &s1, N, S2, S2) ||
        alloc("stem2", (long long)N * S2 * S2, 64, false, &s2, N, S2, S2) ||
        alloc("stem3", (long long)N * S2 * S2, 64, false, &s3, N, S2, S2) ||
        alloc("pool", (long long)N * S4 * S4, 64, false, &pool, N, S4, S4))
        return 1;
    if (conv(model.stem[0], x0, N, S, S, 64, s1, 64, ACT_RELU)) return 1;
    if (conv(model.stem[1], s1, N, S2, S2, 64, s2, 64, ACT_RELU)) return 1;
    if (conv(model.stem[2], s2, N, S2, S2, 64, s3, 64, ACT_RELU)) return 1;
    steps.push_back([=](cudaStream_t st) { return launch_maxpool(s3, pool, N, S2, S2, 64, st); });
    // ---- residual stages
    const void* x = pool;
    int h = S4, w = S4, cch = 64;
    void* feat[4];
    const int planes[4] = {64, 128, 256, 512};
    for (int s = 0; s < 4; ++s) {
        for (size_t b = 0; b < model.blocks[s].size(); ++b) {
            const RtBottleneck& bk = model.blocks[s][b];
            const int ho = bk.pool ? h / 2 : h, wo = bk.pool ? w / 2 : w;
            const std::string nm = "res" + std::to_string(s) + "." + std::to_string(b);
            void *t1, *t2, *o, *sc = nullptr;
            if (alloc("", (long long)N * h * w, planes[s], false, &t1) || alloc("", (long long)N * ho * wo, planes[s], false, &t2) ||
                alloc(nm, (long long)N * ho * wo, planes[s] * 4, false, &o, N, ho, wo))
                return 1;
            if (conv(bk.a, x, N, h, w, cch, t1, planes[s], ACT_RELU)) return 1;
            if (conv(bk.b, t1, N, h, w, planes[s], t2, planes[s], ACT_RELU)) return 1;
            const void* res = x;
            if (bk.has_short) {
                if (alloc("", (long long)N * ho * wo, planes[s] * 4, false, &sc)) return 1;
                const void* sin = x;
                if (bk.pool) {
                    void* pl;
                    if (alloc("", (long long)N * ho * wo, cch, false, &pl)) return 1;
                    const void* xin = x;
                    const int hh = h, ww = w, cc = cch;
                    steps.push_back([=](cudaStream_t st) { return launch_rt_avgpool2(xin, pl, N, hh, ww, cc, st); });
                    sin = pl;
                }
                if (conv(bk.shortc, sin, N, ho, wo, cch, sc, planes[s] * 4, ACT_NONE)) return 1;
                res = sc;
            }
            if (conv(bk.c, t2, N, ho, wo, planes[s], o, planes[s] * 4, ACT_RELU, res, planes[s] * 4)) return 1;
            x = o;
            h = ho;
            w = wo;
            cch = planes[s] * 4;
        }
        feat[s] = const_cast<void*>(x);
        dbg["c" + std::to_string(s + 2)] = dbg["res" + std::to_string(s) + "." + std::to_string(model.blocks[s].size() - 1)];
    }
    // ---- hybrid encoder.  Concat buffers: the producers write their halves in place.
    const int g3 = S / 8, g4 = S / 16, g5 = S / 32;
    void *cat4, *cat3, *pcat4, *pcat5;     // [.., 512]: FPN (up | low) at strides 16 / 8, PAN (down | lateral) at 16 / 32
    if (alloc("cat4", (long long)N * g4 * g4, 2 * D, false, &cat4, N, g4, g4) ||
        alloc("cat3", (long long)N * g3 * g3, 2 * D, false, &cat3, N, g3, g3) ||
        alloc("pcat4", (long long)N * g4 * g4, 2 * D, false, &pcat4, N, g4, g4) ||
        alloc("pcat5", (long long)N * g5 * g5, 2 * D, false, &pcat5, N, g5, g5))
        return 1;
    op_t* cat4h = reinterpret_cast<op_t*>(cat4);
    op_t* cat3h = reinterpret_cast<op_t*>(cat3);
    op_t* pcat4h = reinterpret_cast<op_t*>(pcat4);
    op_t* pcat5h = reinterpret_cast<op_t*>(pcat5);
    void* p5;
    if (alloc("proj5", (long long)N * g5 * g5, D, false, &p5, N, g5, g5)) return 1;
    if (conv(model.enc_proj[0], feat[1], N, g3, g3, 512, cat3h + D, 2 * D, ACT_NONE)) return 1;
    if (conv(model.enc_proj[1], feat[2], N, g4, g4, 1024, cat4h + D, 2 * D, ACT_NONE)) return 1;
    if (conv(model.enc_proj[2], feat[3], N, g5, g5, 2048, p5, D, ACT_NONE)) return 1;
    // AIFI: one post-norm transformer layer over the stride-32 tokens (rtdetr_hybrid_encoder.py:71-122, 360-378)
    const int T5 = g5 * g5;
    const long long R5 = (long long)N * T5;
    void *aq, *aqkv, *aatt, *ay, *as32, *as16, *affn, *p5o;
    if (alloc("aifi.q", R5, D, false, &aq) || alloc("aifi.qkv", R5, 3 * D, false, &aqkv) || alloc("aifi.att", R5, D, false, &aatt) ||
        alloc("aifi.y", R5, D, true, &ay) || alloc("aifi.s32", R5, D, true, &as32) || alloc("aifi.s16", R5, D, false, &as16) ||
        alloc("aifi.ffn", R5, c.ffn, false, &affn) || alloc("aifi.out", R5, D, false, &p5o, N, g5, g5))
        return 1;
    SeqDesc* seq5 = nullptr;
    SeqDesc* seqq = nullptr;
    {
        std::vector<SeqDesc> s5(N), sq(N);
        for (int i = 0; i < N; ++i) {
            s5[i] = SeqDesc{i * T5, T5, i * T5, T5, (long long)i * T5 * 3 * D, T5, 0};
            sq[i] = SeqDesc{i * K, K, i * K, K, (long long)i * K * 3 * D, K, 0};
        }
        void *d5 = nullptr, *dq = nullptr;
        CK(cudaMalloc(&d5, sizeof(SeqDesc) * N));
        CK(cudaMalloc(&dq, sizeof(SeqDesc) * N));
        CK(cudaMemcpy(d5, s5.data(), sizeof(SeqDesc) * N, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(dq, sq.data(), sizeof(SeqDesc) * N, cudaMemcpyHostToDevice));
        bufs.push_back(d5);
        bufs.push_back(dq);
        seq5 = reinterpret_cast<SeqDesc*>(d5);
        seqq = reinterpret_cast<SeqDesc*>(dq);
    }
    const RtdetrModel* mp = &model;
    steps.push_back([=](cudaStream_t st) { return launch_rt_add(p5, nullptr, mp->pos_embed, D, T5, aq, R5, st); });
    op_t* aqkvh = reinterpret_cast<op_t*>(aqkv);
    if (linear(model.aifi_qk, aq, D, (int)R5, aqkvh, 3 * D, false, ACT_NONE)) return 1;
    if (linear(model.aifi_v, p5, D, (int)R5, aqkvh + 2 * D, 3 * D, false, ACT_NONE)) return 1;
    steps.push_back([=](cudaStream_t st) {
        return launch_flash_attention(aqkvh, 3 * D, R5, aqkvh + D, aqkvh + 2 * D, 3 * D, R5, aatt, D, seq5, N, T5, c.heads,
                                      D / c.heads, 0, st);
    });
    flops += 4.0 * N * (double)T5 * T5 * D;
    if (linear(model.aifi_out, aatt, D, (int)R5, ay, D, true, ACT_NONE, p5, false, D)) return 1;
    steps.push_back([=](cudaStream_t st) {
        return launch_layernorm(reinterpret_cast<float*>(ay), (int)R5, D, D, mp->aifi_n1.g, mp->aifi_n1.b, 1e-5f, as16,
                                reinterpret_cast<float*>(as32), nullptr, 1, nullptr, 0, 0, st);
    });
    if (linear(model.aifi_l1, as16, D, (int)R5, affn, c.ffn, false, ACT_GELU)) return 1;
    if (linear(model.aifi_l2, affn, c.ffn, (int)R5, ay, D, true, ACT_NONE, as32, true, D)) return 1;
    steps.push_back([=](cudaStream_t st) {
        return launch_layernorm(reinterpret_cast<float*>(ay), (int)R5, D, D, mp->aifi_n2.g, mp->aifi_n2.b, 1e-5f, p5o, nullptr,
                                nullptr, 1, nullptr, 0, 0, st);
    });
    // top-down FPN (rtdetr_hybrid_encoder.py:380-393)
    void *f4, *l4 = pcat4h + D, *f3, *o4, *o5;
    void* l5 = pcat5h + D;            // lateral outputs live in the second half of the PAN concat buffers
    if (alloc("fpn4", (long long)N * g4 * g4, D, false, &f4, N, g4, g4) || alloc("enc_out3", (long long)N * g3 * g3, D, false, &f3, N, g3, g3) ||
        alloc("enc_out4", (long long)N * g4 * g4, D, false, &o4, N, g4, g4) || alloc("enc_out5", (long long)N * g5 * g5, D, false, &o5, N, g5, g5))
        return 1;
    if (conv(model.lateral[0], p5o, N, g5, g5, D, l5, 2 * D, ACT_SILU)) return 1;
    steps.push_back([=](cudaStream_t st) { return launch_rt_upsample_nearest2(l5, 2 * D, N, g5, g5, D, cat4, 2 * D, 0, st); });
    if (csp(model.fpn[0], "fpn0", cat4, N, g4, g4, f4)) return 1;
    if (conv(model.lateral[1], f4, N, g4, g4, D, l4, 2 * D, ACT_SILU)) return 1;
    steps.push_back([=](cudaStream_t st) { return launch_rt_upsample_nearest2(l4, 2 * D, N, g4, g4, D, cat3, 2 * D, 0, st); });
    if (csp(model.fpn[1], "fpn1", cat3, N, g3, g3, f3)) return 1;
    // bottom-up PAN (:395-408)
    if (conv(model.down[0], f3, N, g3, g3, D, pcat4, 2 * D, ACT_SILU)) return 1;
    if (csp(model.pan[0], "pan0", pcat4, N, g4, g4, o4)) return 1;
    if (conv(model.down[1], o4, N, g4, g4, D, pcat5, 2 * D, ACT_SILU)) return 1;
    if (csp(model.pan[1], "pan1", pcat5, N, g5, g5, o5)) return 1;
    // ---- decoder input: level-major memory, encoder heads, query selection (rtdetrv2_decoder.py:596-746)
    const long long RM = (long long)lv.total * N, RQ = (long long)N * K;
    void *mem, *val, *eo32, *om32, *om16, *elog, *escore;
    if (alloc("memory", RM, D, false, &mem) || alloc("value", RM, c.num_layers * D, false, &val) || alloc("enc.y", RM, D, true, &eo32) ||
        alloc("enc.om32", RM, D, true, &om32) || alloc("enc.om16", RM, D, false, &om16) || alloc("enc.logits", RM, 8, true, &elog) ||
        alloc("enc.scores", (long long)N * lv.total, 1, true, &escore))
        return 1;
    op_t* memh = reinterpret_cast<op_t*>(mem);
    void* enc_outs[3] = {f3, o4, o5};
    for (int l = 0; l < 3; ++l)
        if (conv(model.dec_proj[l], enc_outs[l], N, lv.h[l], lv.w[l], D, memh + (long long)lv.off[l] * N * D, D, ACT_NONE)) return 1;
    if (linear(model.value_all, mem, D, (int)RM, val, c.num_layers * D, false, ACT_NONE)) return 1;
    if (linear(model.enc_out, mem, D, (int)RM, eo32, D, true, ACT_NONE)) return 1;
    steps.push_back([=](cudaStream_t st) {
        return launch_rt_mask_invalid(reinterpret_cast<float*>(eo32), D, mp->enc_out.b, mp->invalid, mp->n_invalid, lv, N, st);
    });
    steps.push_back([=](cudaStream_t st) {
        return launch_layernorm(reinterpret_cast<float*>(eo32), (int)RM, D, D, mp->enc_out_ln.g, mp->enc_out_ln.b, 1e-5f, om16,
                                reinterpret_cast<float*>(om32), nullptr, 1, nullptr, 0, 0, st);
    });
    if (linear(model.enc_score, om16, D, (int)RM, elog, 8, true, ACT_NONE)) return 1;
    void *tk, *tgt32, *tgt16, *asel, *ref, *h1, *h2, *delta;
    if (alloc("topk", RQ, 1, true, &tk) || alloc("tgt32", RQ, D, true, &tgt32) || alloc("tgt16", RQ, D, false, &tgt16) ||
        alloc("anchor_sel", RQ, 4, true, &asel) || alloc("ref", RQ, 4, true, &ref) || alloc("box.h1", RQ, D, false, &h1) ||
        alloc("box.h2", RQ, D, false, &h2) || alloc("box.delta", RQ, 4, true, &delta))
        return 1;
    topk = reinterpret_cast<int*>(tk);
    boxes = reinterpret_cast<float*>(ref);
    steps.push_back([=](cudaStream_t st) {
        return launch_rt_enc_scores(reinterpret_cast<float*>(elog), 8, C, lv, N, reinterpret_cast<float*>(escore), st);
    });
    steps.push_back([=](cudaStream_t st) {
        return launch_rt_topk(reinterpret_cast<float*>(escore), N, lv.total, K, reinterpret_cast<int*>(tk), st);
    });
    steps.push_back([=](cudaStream_t st) {
        return launch_rt_gather_queries(reinterpret_cast<float*>(om32), D, reinterpret_cast<int*>(tk), K, lv, N,
                                        reinterpret_cast<float*>(tgt32), tgt16, mp->anchors, reinterpret_cast<float*>(asel), st);
    });
    if (linear(model.enc_box0, tgt16, D, (int)RQ, h1, D, false, ACT_RELU) || linear(model.enc_box1, h1, D, (int)RQ, h2, D, false, ACT_RELU) ||
        linear(model.enc_box2, h2, D, (int)RQ, delta, 4, true, ACT_NONE))
        return 1;
    steps.push_back([=](cudaStream_t st) {
        return launch_rt_ref_update(reinterpret_cast<float*>(delta), 4, reinterpret_cast<float*>(asel),
                                    reinterpret_cast<float*>(ref), (int)RQ, st);
    });
    // ---- decoder layers (rtdetrv2_decoder.py:225-303, 402-444)
    void *qp0, *qp16, *tq, *qkv, *att, *y, *ow, *samp, *ffn, *lg;
    const int n_ow = c.heads * 3 * c.num_points * 3;
    if (alloc("dec.qp0", RQ, 2 * D, false, &qp0) || alloc("dec.qpos", RQ, D, false, &qp16) || alloc("dec.tq", RQ, D, false, &tq) ||
        alloc("dec.qkv", RQ, 3 * D, false, &qkv) || alloc("dec.att", RQ, D, false, &att) || alloc("dec.y", RQ, D, true, &y) ||
        alloc("dec.ow", RQ, n_ow, true, &ow) || alloc("dec.samp", RQ, D, false, &samp) || alloc("dec.ffn", RQ, c.ffn, false, &ffn) ||
        alloc("logits", RQ, 8, true, &lg) )
        return 1;
    logits = reinterpret_cast<float*>(lg);
    ld_logits = 8;
    {
        void* ol = nullptr;
        CK(cudaMalloc(&ol, (size_t)RQ * C * 4));
        bufs.push_back(ol);
        out_logits = reinterpret_cast<float*>(ol);
    }
    op_t* qkvh = reinterpret_cast<op_t*>(qkv);
    for (int i = 0; i < c.num_layers; ++i) {
        const RtDecLayer* L = &model.layers[i];
        steps.push_back([=](cudaStream_t st) {
            return launch_rt_qpos_l0(reinterpret_cast<float*>(ref), mp->qpos0_w, mp->qpos0_b, 2 * D, qp0, (int)RQ, st);
        });
        if (linear(model.qpos1, qp0, 2 * D, (int)RQ, qp16, D, false, ACT_NONE)) return 1;
        steps.push_back([=](cudaStream_t st) { return launch_rt_add(tgt16, qp16, nullptr, D, 1, tq, RQ, st); });
        if (linear(L->qk, tq, D, (int)RQ, qkvh, 3 * D, false, ACT_NONE)) return 1;
        if (linear(L->v, tgt16, D, (int)RQ, qkvh + 2 * D, 3 * D, false, ACT_NONE)) return 1;
        steps.push_back([=](cudaStream_t st) {
            return launch_flash_attention(qkvh, 3 * D, RQ, qkvh + D, qkvh + 2 * D, 3 * D, RQ, att, D, seqq, N, K, c.heads,
                                          D / c.heads, 0, st);
        });
        flops += 4.0 * N * (double)K * K * D;
        if (linear(L->out, att, D, (int)RQ, y, D, true, ACT_NONE, tgt32, true, D)) return 1;
        steps.push_back([=](cudaStream_t st) {
            return launch_layernorm(reinterpret_cast<float*>(y), (int)RQ, D, D, L->n1.g, L->n1.b, 1e-5f, tgt16,
                                    reinterpret_cast<float*>(tgt32), nullptr, 1, nullptr, 0, 0, st);
        });
        // multi-scale deformable cross-attention
        steps.push_back([=](cudaStream_t st) { return launch_rt_add(tgt16, qp16, nullptr, D, 1, tq, RQ, st); });
        if (linear(L->ow, tq, D, (int)RQ, ow, n_ow, true, ACT_NONE)) return 1;
        steps.push_back([=](cudaStream_t st) {
            return launch_rt_deform_attn(reinterpret_cast<float*>(ow), n_ow, reinterpret_cast<float*>(ref), val,
                                         (long long)c.num_layers * D, i * D, lv, N, K, c.heads, D / c.heads, c.offset_scale,
                                         samp, D, st);
        });
        if (linear(L->cross_out, samp, D, (int)RQ, y, D, true, ACT_NONE, tgt32, true, D)) return 1;
        steps.push_back([=](cudaStream_t st) {
            return launch_layernorm(reinterpret_cast<float*>(y), (int)RQ, D, D, L->n2.g, L->n2.b, 1e-5f, tgt16,
                                    reinterpret_cast<float*>(tgt32), nullptr, 1, nullptr, 0, 0, st);
        });
        if (linear(L->lin1, tgt16, D, (int)RQ, ffn, c.ffn, false, ACT_RELU)) return 1;
        if (linear(L->lin2, ffn, c.ffn, (int)RQ, y, D, true, ACT_NONE, tgt32, true, D)) return 1;
        steps.push_back([=](cudaStream_t st) {
            return launch_layernorm(reinterpret_cast<float*>(y), (int)RQ, D, D, L->n3.g, L->n3.b, 1e-5f, tgt16,
                                    reinterpret_cast<float*>(tgt32), nullptr, 1, nullptr, 0, 0, st);
        });
        // iterative box refinement (:428-441)
        if (linear(L->box0, tgt16, D, (int)RQ, h1, D, false, ACT_RELU) || linear(L->box1, h1, D, (int)RQ, h2, D, false, ACT_RELU) ||
            linear(L->box2, h2, D, (int)RQ, delta, 4, true, ACT_NONE))
            return 1;
        steps.push_back([=](cudaStream_t st) {
            return launch_rt_ref_update(reinterpret_cast<float*>(delta), 4, nullptr, reinterpret_cast<float*>(ref), (int)RQ, st);
        });
    }
    if (linear(model.score_last, tgt16, D, (int)RQ, lg, 8, true, ACT_NONE)) return 1;
    steps.push_back([=](cudaStream_t st) {
        return launch_rt_copy_cols(reinterpret_cast<float*>(lg), 8, C, out_logits, RQ, st);
    });
    return 0;
}

int RtdetrEngine::run(cudaStream_t st) {
    for (auto& s : steps)
        if (s(st)) {
            if (!last_error()[0]) set_error("RT-DETRv2 step launch failed: %s", cudaGetErrorString(cudaGetLastError()));
            return 1;
        }
    return 0;
}

RtdetrEngine::~RtdetrEngine() {
    for (void* p : bufs) cudaFree(p);
}

}  // namespace ytk
