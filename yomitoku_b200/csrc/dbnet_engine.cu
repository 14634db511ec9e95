// DBNet++ (ResNet-50 dilated backbone + FPN decoder + Adaptive Scale Fusion + binarize head) as a static launch plan
// of wgmma implicit-GEMM convolutions and a few memory-bound kernels.  Replaces reference
// models/dbnet_plus.py:13-246 + models/layers/dbnet_feature_attention.py:36-160 for inference.
//
// Data layout in HBM: every activation is NHWC bf16 (channels innermost, 16-byte vectors), batch-norm is folded into
// the conv weights/bias at load time, weights are [Cout][kh][kw][Cin] bf16 (K-major for the UMMA B operand).
// One Engine = one (pages, H, W) shape: all buffers and TMA descriptors are created once and reused.
#include "dbnet_engine.h"

#include <cmath>
#include <cstring>
#include <memory>

#include "dbnet_ops.h"
#include "ptx.cuh"

namespace ytk {

// ---------------------------------------------------------------------------------------------- helpers
#define CK(x)                                                                   \
    do {                                                                        \
        cudaError_t e_ = (x);                                                   \
        if (e_ != cudaSuccess) {                                                \
            set_error("%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); \
            return 1;                                                           \
        }                                                                       \
    } while (0)

const TensorView* WeightSet::find(const std::string& name) const {
    auto it = map.find(name);
    return it == map.end() ? nullptr : &it->second;
}
const TensorView* WeightSet::need(const std::string& name, long long numel) const {
    const TensorView* t = find(name);
    if (!t) {
        set_error("state_dict is missing '%s'", name.c_str());
        return nullptr;
    }
    if (numel >= 0 && t->numel() != numel) {
        set_error("state_dict tensor '%s' has %lld elements, expected %lld", name.c_str(), t->numel(), numel);
        return nullptr;
    }
    return t;
}

static int upload(const void* host, size_t bytes, void** dev) {
    CK(cudaMalloc(dev, bytes));
    CK(cudaMemcpy(*dev, host, bytes, cudaMemcpyHostToDevice));
    return 0;
}

// Fold eval-mode BatchNorm into (scale, shift) per output channel.
static int bn_fold(const WeightSet& ws, const std::string& p, int C, std::vector<float>& scale,
                   std::vector<float>& shift) {
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

// conv weight [Cout][Cin][kh][kw] fp32 (+ optional per-channel scale) -> [Cout][kh][kw][Cin] bf16 on the device
static int pack_conv(const TensorView* w, int Cout, int Cin, int kh, int kw, const float* scale, void** dev) {
    std::vector<uint16_t> p((size_t)Cout * kh * kw * Cin);
    for (int co = 0; co < Cout; ++co)
        for (int ci = 0; ci < Cin; ++ci)
            for (int r = 0; r < kh; ++r)
                for (int s = 0; s < kw; ++s) {
                    const float v = w->data[(((size_t)co * Cin + ci) * kh + r) * kw + s] * (scale ? scale[co] : 1.f);
                    p[(((size_t)co * kh + r) * kw + s) * Cin + ci] = f2op_host(v);
                }
    return upload(p.data(), p.size() * 2, dev);
}

void pack_stem_weights(const float* w, const float* scale, std::vector<uint16_t>* out) {
    std::vector<uint16_t>& p = *out;
    p.assign((size_t)64 * 7 * 64, 0);
    for (int co = 0; co < 64; ++co)
        for (int c = 0; c < 3; ++c)
            for (int r = 0; r < 7; ++r)
                for (int s = 0; s < 7; ++s)
                    p[((size_t)co * 7 + r) * 64 + s * 8 + c] =
                        f2op_host(w[(((size_t)co * 3 + c) * 7 + r) * 7 + s] * (scale ? scale[co] : 1.f));
}

void pack_convt_head(const float* w1, const float* b1, const float* scale, const float* shift, const float* w2,
                     std::vector<uint16_t>* w_rows, std::vector<float>* bias, std::vector<float>* fin_w) {
    std::vector<uint16_t>& p = *w_rows;
    p.resize((size_t)256 * 64);
    bias->resize(256);
    for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 2; ++j)
            for (int co = 0; co < 64; ++co) {
                const int row = (i * 2 + j) * 64 + co;
                const float sc = scale ? scale[co] : 1.f;
                for (int ci = 0; ci < 64; ++ci)
                    p[(size_t)row * 64 + ci] = f2op_host(w1[(((size_t)ci * 64 + co) * 2 + i) * 2 + j] * sc);
                (*bias)[row] = b1[co] * sc + (shift ? shift[co] : 0.f);
            }
    // [ci][1][i'][j'] -> [k = i'*2+j'][ci] for the fused epilogue
    fin_w->resize(4 * 64);
    for (int ci = 0; ci < 64; ++ci)
        for (int k = 0; k < 4; ++k) (*fin_w)[k * 64 + ci] = w2[ci * 4 + k];
}

int DbnetModel::load_conv(const WeightSet& ws, const std::string& wname, const std::string& bnname, int Cout, int Cin,
                          int k, int stride, int pad, int dil, const std::string& biasname, ConvW* out) {
    const TensorView* w = ws.need(wname, (long long)Cout * Cin * k * k);
    if (!w) return 1;
    std::vector<float> scale, shift;
    const float* sc = nullptr;
    std::vector<float> bias;
    if (!bnname.empty()) {
        if (bn_fold(ws, bnname, Cout, scale, shift)) return 1;
        sc = scale.data();
        bias = shift;
    }
    if (!biasname.empty()) {
        const TensorView* b = ws.need(biasname, Cout);
        if (!b) return 1;
        if (bias.empty()) bias.assign(Cout, 0.f);
        for (int c = 0; c < Cout; ++c) bias[c] += b->data[c] * (sc ? sc[c] : 1.f);
    }
    out->Cout = Cout;
    out->Cin = Cin;
    out->k = k;
    out->stride = stride;
    out->pad = pad;
    out->dil = dil;
    if (pack_conv(w, Cout, Cin, k, k, sc, &out->w)) return 1;
    out->bias = nullptr;
    if (!bias.empty()) {
        void* d = nullptr;
        if (upload(bias.data(), bias.size() * 4, &d)) return 1;
        out->bias = reinterpret_cast<float*>(d);
    }
    owned.push_back(out->w);
    if (out->bias) owned.push_back(out->bias);
    return 0;
}

int DbnetModel::load(const WeightSet& ws) {
    const std::string bb = "backbone.body.";
    // ---- stem: 7x7/s2 conv + BN, packed as [64][7 rows][8 px * 8 ch] (pixels 0..6 and channels 0..2 non-zero)
    {
        const TensorView* w = ws.need(bb + "conv1.weight", 64LL * 3 * 7 * 7);
        if (!w) return 1;
        std::vector<float> scale, shift;
        if (bn_fold(ws, bb + "bn1", 64, scale, shift)) return 1;
        std::vector<uint16_t> p;
        pack_stem_weights(w->data, scale.data(), &p);
        if (upload(p.data(), p.size() * 2, &stem.w)) return 1;
        void* d = nullptr;
        if (upload(shift.data(), 64 * 4, &d)) return 1;
        stem.bias = reinterpret_cast<float*>(d);
        stem.Cout = 64;
        owned.push_back(stem.w);
        owned.push_back(stem.bias);
    }
    // ---- bottlenecks (torchvision resnet50, layer4 stride replaced by dilation; SURVEY.md Appendix A6)
    const int planes[4] = {64, 128, 256, 512}, nblk[4] = {3, 4, 6, 3};
    int inpl = 64;
    for (int l = 0; l < 4; ++l) {
        for (int b = 0; b < nblk[l]; ++b) {
            Bottleneck bk;
            const std::string p = bb + "layer" + std::to_string(l + 1) + "." + std::to_string(b) + ".";
            int stride = (b == 0 && (l == 1 || l == 2)) ? 2 : 1;
            int dil = (l == 3 && b > 0) ? 2 : 1;
            if (load_conv(ws, p + "conv1.weight", p + "bn1", planes[l], inpl, 1, 1, 0, 1, "", &bk.c1)) return 1;
            if (load_conv(ws, p + "conv2.weight", p + "bn2", planes[l], planes[l], 3, stride, dil, dil, "", &bk.c2))
                return 1;
            if (load_conv(ws, p + "conv3.weight", p + "bn3", planes[l] * 4, planes[l], 1, 1, 0, 1, "", &bk.c3)) return 1;
            bk.has_down = (b == 0);
            if (bk.has_down &&
                load_conv(ws, p + "downsample.0.weight", p + "downsample.1", planes[l] * 4, inpl, 1, stride, 0, 1, "",
                          &bk.down))
                return 1;
            blocks[l].push_back(bk);
            inpl = planes[l] * 4;
        }
    }
    // ---- decoder
    const std::string d = "decoder.";
    const int cin[4] = {256, 512, 1024, 2048};
    for (int i = 0; i < 4; ++i) {
        const std::string n = std::to_string(i + 1);
        if (load_conv(ws, d + "input_proj.layer" + n + ".weight", "", 256, cin[i], 1, 1, 0, 1, "", &lateral[i])) return 1;
        const std::string on = (i == 0) ? d + "out_proj.layer1.weight" : d + "out_proj.layer" + n + ".0.weight";
        if (load_conv(ws, on, "", 64, 256, 3, 1, 1, 1, "", &outproj[i])) return 1;
    }
    const std::string ca = d + "concat_attention.";
    if (load_conv(ws, ca + "conv.weight", "", 64, 256, 3, 1, 1, 1, ca + "conv.bias", &asf_conv)) return 1;
    {
        const std::string e = ca + "enhanced_attention.";
        const TensorView *w1 = ws.need(e + "channel_wise.1.weight", 16 * 64), *w2 = ws.need(e + "channel_wise.3.weight", 64 * 16),
                         *s3 = ws.need(e + "spatial_wise.0.weight", 9), *s1 = ws.need(e + "spatial_wise.2.weight", 1),
                         *at = ws.need(e + "attention_wise.0.weight", 4 * 64);
        if (!w1 || !w2 || !s3 || !s1 || !at) return 1;
        void* p = nullptr;
        if (upload(w1->data, 16 * 64 * 4, &p)) return 1;
        asf_w1 = reinterpret_cast<float*>(p);
        if (upload(w2->data, 64 * 16 * 4, &p)) return 1;
        asf_w2 = reinterpret_cast<float*>(p);
        owned.push_back(asf_w1);
        owned.push_back(asf_w2);
        memcpy(asf_sp3, s3->data, 9 * 4);
        asf_sp1 = s1->data[0];
        memcpy(asf_att, at->data, 4 * 64 * 4);
    }
    const std::string bz = d + "binarize.";
    if (load_conv(ws, bz + "0.weight", bz + "1", 64, 256, 3, 1, 1, 1, "", &bin_conv)) return 1;
    {
        // ConvTranspose2d(64,64,2,2) + BN (folded) + ReLU, then ConvTranspose2d(64,1,2,2): see pack_convt_head
        const TensorView *w = ws.need(bz + "3.weight", 64LL * 64 * 4), *b = ws.need(bz + "3.bias", 64);
        const TensorView *w2 = ws.need(bz + "6.weight", 64 * 4), *b2 = ws.need(bz + "6.bias", 1);
        if (!w || !b || !w2 || !b2) return 1;
        std::vector<float> scale, shift;
        if (bn_fold(ws, bz + "4", 64, scale, shift)) return 1;
        std::vector<uint16_t> p;
        std::vector<float> bias, fw;
        pack_convt_head(w->data, b->data, scale.data(), shift.data(), w2->data, &p, &bias, &fw);
        if (upload(p.data(), p.size() * 2, &convt1.w)) return 1;
        void* q = nullptr;
        if (upload(bias.data(), 256 * 4, &q)) return 1;
        convt1.bias = reinterpret_cast<float*>(q);
        convt1.Cout = 256;
        convt1.Cin = 64;
        owned.push_back(convt1.w);
        owned.push_back(convt1.bias);
        void* fd = nullptr;
        if (upload(fw.data(), fw.size() * 4, &fd)) return 1;
        convt2_w_dev = reinterpret_cast<float*>(fd);
        owned.push_back(fd);
        convt2_b = b2->data[0];
    }
    return 0;
}

DbnetModel::~DbnetModel() {
    for (void* p : owned) cudaFree(p);
}

// ---------------------------------------------------------------------------------------------- engine
void dbnet_input_size(int H0, int W0, int shortest, int limit, int* Hn, int* Wn) {
    // reference resize_shortest_edge, data/functions.py:212-224 (int() truncations, floor to multiples of 32)
    const double scale = (double)shortest / (double)(H0 < W0 ? H0 : W0);
    int nh, nw;
    if (H0 < W0) {
        nh = shortest;
        nw = (int)(W0 * scale);
    } else {
        nh = (int)(H0 * scale);
        nw = shortest;
    }
    const int mx = nh > nw ? nh : nw;
    if (mx > limit) {
        const double s2 = (double)limit / (double)mx;
        nh = (int)(nh * s2);
        nw = (int)(nw * s2);
    }
    *Wn = (nw / 32) * 32 > 32 ? (nw / 32) * 32 : 32;
    *Hn = (nh / 32) * 32 > 32 ? (nh / 32) * 32 : 32;
}

int DbnetEngine::alloc(const std::string& name, int n, int h, int w, int c, bool f32, void** out) {
    const size_t bytes = (size_t)n * h * w * c * (f32 ? 4 : 2);
    void* p = nullptr;
    CK(cudaMalloc(&p, bytes));
    bufs.push_back(p);
    total_bytes += bytes;
    dbg[name] = DebugTensor{p, n, h, w, c, f32};
    *out = p;
    return 0;
}

int DbnetEngine::add_conv(const ConvW& cw, const void* in, int n, int h, int w, long long in_ld, void* out,
                          long long ldc, int act, const void* resid, long long ldr, bool out_f32) {
    ConvGeom g{n, h, w, cw.Cin, in_ld, cw.k, cw.k, cw.stride, cw.pad, cw.dil, cw.Cout};
    Epilogue e;
    e.bias = cw.bias;
    e.resid = resid;
    e.ldr = ldr;
    e.out = out;
    e.ldc = ldc;
    e.out_f32 = out_f32 ? 1 : 0;
    e.act = act;
    auto plan = std::make_shared<GemmPlan>();
    if (conv_plan_create(plan.get(), in, g, cw.w, e)) return 1;
    flops += plan->flops;
    steps.push_back([plan](cudaStream_t st) { return gemm_plan_launch(plan.get(), st); });
    return 0;
}

int DbnetEngine::build(const DbnetModel& m, int n, int Hn_, int Wn_) {
    N = n;
    Hn = Hn_;
    Wn = Wn_;
    if (Hn % 32 || Wn % 32) {
        set_error("DBNet input must be a multiple of 32, got %dx%d", Hn, Wn);
        return 1;
    }
    const int H2 = Hn / 2, W2 = Wn / 2, H4 = Hn / 4, W4 = Wn / 4, H8 = Hn / 8, W8 = Wn / 8, H16 = Hn / 16, W16 = Wn / 16;
    void *in_pad, *stem_o, *pool_o;
    {
        const size_t bytes = (size_t)N * (Hn + 6) * (Wn + 8) * 8 * 2;
        CK(cudaMalloc(&in_pad, bytes));
        bufs.push_back(in_pad);
        total_bytes += bytes;
        input = in_pad;
    }
    if (alloc("stem", N, H2, W2, 64, false, &stem_o)) return 1;
    if (alloc("pool", N, H4, W4, 64, false, &pool_o)) return 1;
    // ---- stem through overlapping TMA boxes on the padded 8-channel canvas
    {
        Epilogue e;
        e.bias = m.stem.bias;
        e.out = stem_o;
        e.ldc = 64;
        e.act = ACT_RELU;
        auto plan = std::make_shared<GemmPlan>();
        if (stem_plan_create(plan.get(), in_pad, N, Hn, Wn, m.stem.w, e)) return 1;
        flops += 2.0 * N * H2 * W2 * 64.0 * 147.0;  // algorithmic (the padded K=448 GEMM does more)
        steps.push_back([plan](cudaStream_t st) { return gemm_plan_launch(plan.get(), st); });
    }
    steps.push_back([=](cudaStream_t st) { return launch_maxpool(stem_o, pool_o, N, H2, W2, 64, st); });
    // ---- residual stages
    const void* x = pool_o;
    int h = H4, w = W4, c = 64;
    void* feat[4];
    const int planes[4] = {64, 128, 256, 512};
    for (int l = 0; l < 4; ++l) {
        for (size_t b = 0; b < m.blocks[l].size(); ++b) {
            const Bottleneck& bk = m.blocks[l][b];
            const int ho = (bk.c2.stride == 2) ? h / 2 : h, wo = (bk.c2.stride == 2) ? w / 2 : w;
            const std::string nm = "layer" + std::to_string(l + 1) + "." + std::to_string(b);
            void *t1, *t2, *o, *idn = nullptr;
            if (alloc(nm + ".t1", N, h, w, planes[l], false, &t1)) return 1;
            if (alloc(nm + ".t2", N, ho, wo, planes[l], false, &t2)) return 1;
            if (alloc(nm, N, ho, wo, planes[l] * 4, false, &o)) return 1;
            if (add_conv(bk.c1, x, N, h, w, c, t1, planes[l], ACT_RELU)) return 1;
            if (add_conv(bk.c2, t1, N, h, w, planes[l], t2, planes[l], ACT_RELU)) return 1;
            const void* res = x;
            if (bk.has_down) {
                if (alloc(nm + ".down", N, ho, wo, planes[l] * 4, false, &idn)) return 1;
                if (add_conv(bk.down, x, N, h, w, c, idn, planes[l] * 4, ACT_NONE)) return 1;
                res = idn;
            }
            if (add_conv(bk.c3, t2, N, ho, wo, planes[l], o, planes[l] * 4, ACT_RELU, res, planes[l] * 4)) return 1;
            x = o;
            h = ho;
            w = wo;
            c = planes[l] * 4;
        }
        feat[l] = const_cast<void*>(x);
        dbg["layer" + std::to_string(l + 1)] = dbg["layer" + std::to_string(l + 1) + "." +
                                                   std::to_string(m.blocks[l].size() - 1)];
    }
    // ---- FPN laterals + cumulative top-down sums (reference dbnet_plus.py:201-220)
    const int fh[4] = {H4, H8, H16, H16}, fw[4] = {W4, W8, W16, W16}, fc[4] = {256, 512, 1024, 2048};
    void* f[4];
    for (int i = 0; i < 4; ++i)
        if (alloc("f" + std::to_string(i + 1), N, fh[i], fw[i], 256, false, &f[i])) return 1;
    if (add_conv(m.lateral[3], feat[3], N, fh[3], fw[3], fc[3], f[3], 256, ACT_NONE)) return 1;
    // layer3 and layer4 maps have the same size: the top-down add is a plain residual in the lateral conv's epilogue
    if (add_conv(m.lateral[2], feat[2], N, fh[2], fw[2], fc[2], f[2], 256, ACT_NONE, f[3], 256)) return 1;
    for (int i = 1; i >= 0; --i) {
        if (add_conv(m.lateral[i], feat[i], N, fh[i], fw[i], fc[i], f[i], 256, ACT_NONE)) return 1;
        void *src = f[i + 1], *dst = f[i];
        const int hs = fh[i + 1], ws_ = fw[i + 1], hd = fh[i], wd = fw[i];
        steps.push_back([=](cudaStream_t st) { return launch_upsample(src, N, hs, ws_, 256, dst, hd, wd, 256, 0, 1, st); });
    }
    // ---- out_proj 3x3 convs written (through bilinear upsampling) into the concat buffer, order p4,p3,p2,p1
    void* fuse;
    if (alloc("fuse", N, H4, W4, 256, false, &fuse)) return 1;
    if (add_conv(m.outproj[0], f[0], N, H4, W4, 256, reinterpret_cast<op_t*>(fuse) + 192, 256, ACT_NONE))
        return 1;
    for (int i = 1; i < 4; ++i) {
        void* p;
        if (alloc("p" + std::to_string(i + 1), N, fh[i], fw[i], 64, false, &p)) return 1;
        if (add_conv(m.outproj[i], f[i], N, fh[i], fw[i], 256, p, 64, ACT_NONE)) return 1;
        const int hs = fh[i], ws_ = fw[i], coff = 64 * (3 - i);
        steps.push_back([=](cudaStream_t st) { return launch_upsample(p, N, hs, ws_, 64, fuse, H4, W4, 256, coff, 0, st); });
    }
    // ---- Adaptive Scale Fusion
    void *asf_a, *gsum, *gvec, *gmean, *mmap;
    if (alloc("asf_a", N, H4, W4, 64, false, &asf_a)) return 1;
    if (add_conv(m.asf_conv, fuse, N, H4, W4, 256, asf_a, 64, ACT_NONE)) return 1;
    CK(cudaMalloc(&gsum, sizeof(float) * 64 * kAsfPoolChunks * N));
    CK(cudaMalloc(&gvec, sizeof(float) * 64 * N));
    CK(cudaMalloc(&gmean, sizeof(float) * N));
    bufs.push_back(gsum);
    bufs.push_back(gvec);
    bufs.push_back(gmean);
    if (alloc("asf_m", N, H4, W4, 1, true, &mmap)) return 1;
    {
        const DbnetModel* mp = &m;
        steps.push_back([=](cudaStream_t st) {
            return launch_asf(asf_a, fuse, N, H4, W4, mp->asf_w1, mp->asf_w2, mp->asf_sp3, mp->asf_sp1, mp->asf_att,
                              reinterpret_cast<float*>(gsum), reinterpret_cast<float*>(gvec),
                              reinterpret_cast<float*>(gmean), reinterpret_cast<float*>(mmap), st);
        });
    }
    // ---- binarize head
    void *b1, *prob_;
    if (alloc("bin1", N, H4, W4, 64, false, &b1)) return 1;
    if (add_conv(m.bin_conv, fuse, N, H4, W4, 256, b1, 64, ACT_RELU)) return 1;
    if (alloc("prob", N, Hn, Wn, 1, true, &prob_)) return 1;
    prob = reinterpret_cast<float*>(prob_);
    {
        // ConvT(64->64,2,2)+BN+ReLU and ConvT(64->1,2,2)+sigmoid fused into one GEMM epilogue: the 64x(H/2)x(W/2)
        // intermediate never touches HBM.
        ConvGeom g{N, H4, W4, 64, 64, 1, 1, 1, 0, 1, 256};
        Epilogue e;
        e.bias = m.convt1.bias;
        e.out = prob_;
        e.out_f32 = 1;
        e.ldc = 4;
        e.mode = EPI_CONVT_FINAL;
        e.fin_w = m.convt2_w_dev;
        e.fin_b = m.convt2_b;
        auto plan = std::make_shared<GemmPlan>();
        if (conv_plan_create(plan.get(), b1, g, m.convt1.w, e)) return 1;
        flops += plan->flops + 2.0 * N * H2 * W2 * 64.0 * 4.0;
        steps.push_back([plan](cudaStream_t st) { return gemm_plan_launch(plan.get(), st); });
    }
    return 0;
}

int DbnetEngine::run(cudaStream_t st) {
    for (auto& s : steps)
        if (s(st)) {
            if (!last_error()[0]) set_error("DBNet step launch failed: %s", cudaGetErrorString(cudaGetLastError()));
            return 1;
        }
    return 0;
}

DbnetEngine::~DbnetEngine() {
    for (void* p : bufs) cudaFree(p);
}

}  // namespace ytk
