// RT-DETRv2 (layout parser / table structure recognizer of the reference) model + per-batch-size execution engine.
// See rtdetr_engine.cu.
#pragma once
#include <cuda_runtime.h>

#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "dbnet_engine.h"   // TensorView / WeightSet / ConvW / DebugTensor
#include "parseq_ops.h"     // SeqDesc
#include "rtdetr_ops.h"

namespace ytk {

struct RtCfg {
    int num_classes = 6;
    int hidden = 256, heads = 8, ffn = 1024;
    int num_queries = 300, num_layers = 6;
    int img = 640;                 // square eval size (cfg.data.img_size / eval_spatial_size)
    int num_points = 4;            // per level
    float offset_scale = 0.5f;
};

struct RtLinear {
    void* w = nullptr;   // fp16 [N][Kp]
    float* b = nullptr;  // fp32 [N]
    int N = 0, K = 0;    // K = padded to a multiple of 64
};
struct RtLn {
    float *g = nullptr, *b = nullptr;
};
struct RtBottleneck {
    ConvW a, b, c, shortc;
    bool has_short = false, pool = false;
};
struct RtCsp {
    ConvW conv1, conv2, rep[3];    // rep: RepVggBlock re-parameterised (3x3 + 1x1 + both BNs -> one 3x3 + bias)
};
struct RtDecLayer {
    RtLinear qk, v, out, ow, cross_out, lin1, lin2;   // ow = sampling_offsets ++ attention_weights
    RtLn n1, n2, n3;
    RtLinear box0, box1, box2;                          // dec_bbox_head[i]
};

struct RtdetrModel {
    RtCfg cfg;
    ConvW stem[3];
    std::vector<RtBottleneck> blocks[4];
    ConvW enc_proj[3], lateral[2], down[2], dec_proj[3];
    RtLinear aifi_qk, aifi_v, aifi_out, aifi_l1, aifi_l2;
    RtLn aifi_n1, aifi_n2;
    RtCsp fpn[2], pan[2];
    float* pos_embed = nullptr;                        // fp32 [(img/32)^2, hidden]
    RtLinear value_all;                                // the value_proj of all decoder layers: hidden -> layers * hidden
    RtLinear enc_out, enc_score, enc_box0, enc_box1, enc_box2, qpos1, score_last;
    RtLn enc_out_ln;
    float *qpos0_w = nullptr, *qpos0_b = nullptr;      // query_pos_head.layers.0 (fp32, K = 4)
    float* anchors = nullptr;                          // fp32 [L, 4] logit space (inf where invalid)
    int* invalid = nullptr;                            // anchors outside the valid mask (device list)
    int n_invalid = 0;
    std::vector<RtDecLayer> layers;
    RtLevels lv;
    std::vector<void*> owned;
    int load(const WeightSet& ws, const RtCfg& cfg);
    ~RtdetrModel();
};

struct RtdetrEngine {
    const RtdetrModel* m = nullptr;
    int N = 0;
    void* input = nullptr;       // fp16 NHWC [N, img, img, 64]
    float* in_f32 = nullptr;     // staging for host inputs: [N, 3, img, img]
    float* logits = nullptr;     // fp32 [N * K, ld_logits] (first num_classes columns)
    int ld_logits = 0;
    float* boxes = nullptr;      // fp32 [N * K, 4] cxcywh in [0, 1]
    int* topk = nullptr;         // [N, K] selected anchors
    float* out_logits = nullptr; // packed [N, K, C]
    double flops = 0;
    size_t total_bytes = 0;
    std::vector<void*> bufs;
    std::vector<std::function<int(cudaStream_t)>> steps;
    std::map<std::string, DebugTensor> dbg;
    // Stage read-out for the tests (ytk_rtdetr_set_debug / ytk_rtdetr_debug_tensor).  Stages the engine later overwrites
    // in place are registered as captures: with `debug` on, run() copies each into its own buffer (allocated on the
    // first such run, owned by the engine) right after the step that produced it.  With `debug` off the captures
    // neither allocate nor run.  `ran` / `captured` describe the last run, so that a stage it did not produce is refused
    // instead of read as zeros or stale data.
    struct Capture {
        size_t after = 0;      // runs before step `after` (after all steps built before it)
        const void* src = nullptr;
        DebugTensor t;         // t.p: the capture buffer (null until the first run with capture on)
        size_t bytes = 0;
    };
    std::map<std::string, Capture> caps;
    std::vector<const Capture*> cap_order;
    bool ran = false, captured = false;
    int build(const RtdetrModel& model, int n);
    int run(cudaStream_t st, bool debug = false);
    // The buffer behind a stage name of the last run; 1 + set_error for an unknown name or one the last run did not
    // produce.
    int debug_view(const std::string& name, DebugTensor* out) const;
    ~RtdetrEngine();

  private:
    int alloc(const std::string& name, long long rows, int c, bool f32, void** out, int n = 0, int h = 0, int w = 0);
    void capture(const std::string& name, const void* src, long long rows, int c, bool f32, int n = 0, int h = 0,
                 int w = 0);
    int conv(const ConvW& cw, const void* in, int n, int h, int w, long long in_ld, void* out, long long ldc, int act,
             const void* resid = nullptr, long long ldr = 0);
    int linear(const RtLinear& w, const void* A, long long lda, int M, void* out, long long ldc, bool out_f32, int act,
               const void* resid = nullptr, bool resid_f32 = false, long long ldr = 0);
    int csp(const RtCsp& c, const std::string& name, const void* cat, int n, int h, int w, void* out);
};

}  // namespace ytk
