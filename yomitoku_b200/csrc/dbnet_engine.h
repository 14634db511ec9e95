// DBNet++ model (device weights) and per-shape execution engine.  See dbnet_engine.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <functional>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "gemm_tc.h"

namespace ytk {

struct TensorView {
    const float* data;
    int ndim;
    long long shape[4];
    long long numel() const {
        long long n = 1;
        for (int i = 0; i < ndim; ++i) n *= shape[i];
        return n;
    }
};

// The reference-keyed state_dict handed over the C ABI (host fp32 tensors, SURVEY.md Appendix C).
struct WeightSet {
    std::unordered_map<std::string, TensorView> map;
    const TensorView* find(const std::string& name) const;
    const TensorView* need(const std::string& name, long long numel) const;
};

struct ConvW {
    void* w = nullptr;      // bf16 [Cout][k][k][Cin], BN scale folded in
    float* bias = nullptr;  // fp32 [Cout] (BN shift and/or conv bias) or null
    int Cout = 0, Cin = 0, k = 1, stride = 1, pad = 0, dil = 1;
};

struct Bottleneck {
    ConvW c1, c2, c3, down;
    bool has_down = false;
};

struct DbnetModel {
    ConvW stem;
    std::vector<Bottleneck> blocks[4];
    ConvW lateral[4], outproj[4], asf_conv, bin_conv, convt1;
    float *asf_w1 = nullptr, *asf_w2 = nullptr;  // device: channel_wise 1x1 convs (16x64, 64x16)
    float asf_sp3[9], asf_sp1, asf_att[4 * 64];  // host copies of the tiny attention weights
    float* convt2_w_dev = nullptr;  // device [4][64]: last transposed conv, k = i'*2+j'
    float convt2_b = 0.f;
    std::vector<void*> owned;
    int load(const WeightSet& ws);
    int load_conv(const WeightSet& ws, const std::string& wname, const std::string& bnname, int Cout, int Cin, int k,
                  int stride, int pad, int dil, const std::string& biasname, ConvW* out);
    ~DbnetModel();
};

struct DebugTensor {
    void* p = nullptr;
    int n = 0, h = 0, w = 0, c = 0;
    bool f32 = false;
};

struct DbnetEngine {
    int N = 0, Hn = 0, Wn = 0;
    void* input = nullptr;   // padded NHWC8 bf16 canvas [N, Hn+6, Wn+8, 8]
    float* prob = nullptr;   // [N, Hn, Wn] fp32
    double flops = 0;        // algorithmic conv FLOPs per run (2*MAC)
    size_t total_bytes = 0;
    std::vector<void*> bufs;
    std::vector<std::function<int(cudaStream_t)>> steps;
    std::map<std::string, DebugTensor> dbg;
    int build(const DbnetModel& m, int n, int Hn, int Wn);
    int run(cudaStream_t st);
    int alloc(const std::string& name, int n, int h, int w, int c, bool f32, void** out);
    int add_conv(const ConvW& cw, const void* in, int n, int h, int w, long long in_ld, void* out, long long ldc,
                 int act, const void* resid = nullptr, long long ldr = 0, bool out_f32 = false);
    ~DbnetEngine();
};

void dbnet_input_size(int H0, int W0, int shortest, int limit, int* Hn, int* Wn);

// Weight packing shared by DbnetModel::load (BatchNorm folded in: per-channel scale / shift) and the op-level entries
// (identity: scale and shift null).
// Stem: conv1.weight [64][3][7][7] fp32 -> [64][7 rows][8 px * 8 ch] 16-bit (pixel 7 and channels 3..7 zero).
void pack_stem_weights(const float* w, const float* scale, std::vector<uint16_t>* out);
// Binarize head: ConvTranspose2d(64,64,2,2) weight [ci][co][i][j] and bias -> GEMM rows ordered (i, j, co), w_rows
// [256][64] 16-bit and bias [256] fp32; ConvTranspose2d(64,1,2,2) weight [ci][1][i'][j'] -> fin_w [k = i'*2+j'][ci] fp32.
void pack_convt_head(const float* w1, const float* b1, const float* scale, const float* shift, const float* w2,
                     std::vector<uint16_t>* w_rows, std::vector<float>* bias, std::vector<float>* fin_w);

}  // namespace ytk
