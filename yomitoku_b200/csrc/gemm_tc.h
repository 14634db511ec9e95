// Implicit-GEMM convolution / linear layer on wgmma tensor cores (sm_90a).
//
//   D[pixel, co] = act( sum_{tap, ci} A[pixel + tap, ci] * W[co, tap, ci] + bias[co] (+ resid[pixel, co]) )
//
// A is an NHWC bf16 activation tensor read through 4-D TMA tensor maps: one 128-pixel M tile is a BH x BW spatial
// patch (BH*BW = 128), and a filter tap is just a shifted TMA box whose out-of-bounds part is zero-filled by the
// hardware (= convolution padding).  Stride-2 convolutions read through up to four "phase" tensor maps (even/odd
// rows x even/odd columns).  A plain linear layer is the degenerate case H = 1, W = M, one tap.
// W is a K-major bf16 matrix [Cout][taps*Cin] read through a 2-D TMA map.  Accumulators live in the registers of two
// consumer warpgroups (fp32); the TMA producer fills the K ring for tile i+1 while they store tile i (persistent CTAs,
// one per SM).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ytk {

constexpr int kMaxTaps = 9;

enum Act : int { ACT_NONE = 0, ACT_RELU = 1, ACT_GELU = 2, ACT_SIGMOID = 3, ACT_SILU = 4 };
enum EpiMode : int {
    EPI_NORMAL = 0,
    EPI_SHUFFLE2X = 1,  // ConvTranspose2d(k=2,s=2): column block (i,j) of width Cout/4 goes to pixel (2h+i, 2w+j)
    // DBNet binarize tail: ConvT(64->64,2,2)+BN+ReLU as above (Cout = 256) immediately followed by
    // ConvT(64->1,2,2)+sigmoid evaluated in registers; out = fp32 probability map [N, 4*Ho, 4*Wo]
    EPI_CONVT_FINAL = 2,
    // Row-wise softmax statistics instead of the output matrix (the PARSeq head, K9 of SURVEY.md section 2.3): for every
    // row and every 32-column slice owner (two epilogue warps per row and N tile) the running (max, sum exp(x - max),
    // arg-max) of x = acc + bias over the columns < Cout; `out` is a float4 array [rows][2 * tiles_n] = {max, sum,
    // bit-cast index, 0}.  The [rows, Cout] fp32 logits never touch HBM; a tiny kernel merges the partials
    // (parseq_ops.cu: ar_control_kernel / rowmax_finalize_kernel).  act == ACT_RELU skips the sum (arg-max only).
    EPI_ROWMAX = 3,
};

struct ConvTap {
    int32_t map;  // which A tensor map (stride-2 phase)
    int32_t dh;   // row offset added to the tile origin (in the phase map's coordinates)
    int32_t dw;   // column offset
};

struct alignas(64) GemmMaps {
    CUtensorMap a[4];
    CUtensorMap b;
    // TMA epilogue (args.epi_tma): the output tensor [n_img][Ho][Wo][Cout] and the residual tensor of the same shape,
    // 128-byte-swizzled boxes of 16 tile rows x 128 bytes (one epilogue warp's pass)
    CUtensorMap out;
    CUtensorMap resid;
    CUtensorMap resid_pf;   // the residual tensor again, box = a whole output tile (L2 prefetch one tile ahead)
};

struct GemmArgs {
    int Ho, Wo, n_img;             // output spatial extent (per image) and image count
    int bw_log2;                   // tile patch: BW = 1 << bw_log2 columns, BH = 128 >> bw_log2 rows
    int tiles_w, tiles_h, tiles_n; // tile grid
    int Cout;                      // true number of output columns (<= tiles_n * BLOCK_N)
    int kpt;                       // 64-channel K blocks per tap
    int ntaps;
    ConvTap taps[kMaxTaps];
    const float* bias;             // [Cout] fp32 or null
    const void* resid;             // [pixels, ldr] bf16 or fp32, or null; same pixel indexing as out
    int resid_f32;
    long long ldr;
    void* out;                     // [pixels, ldc] bf16 or fp32
    int out_f32;
    long long ldc;
    int act;
    int mode;
    const float* fin_w;            // EPI_CONVT_FINAL: device [4][64] fp32, k = i'*2+j' of the last transposed conv
    float fin_b;
    int epi_tma;                   // 1: the epilogue moves residual and output tiles with TMA (EPI_NORMAL plans whose
                                   // residual, if any, has the output's element size); 0: per-thread global accesses
    int epi_swz;                   // 1: the TMA epilogue's boxes are 128-byte swizzled (conflict-free row accesses)
    int epi_pf;                    // 1: the TMA producer prefetches the next tile's residual rows into L2 (whole rows of
                                   // the tile in one request instead of 64-byte pieces fetched from DRAM one by one)
};

struct Epilogue {
    const float* bias = nullptr;
    const void* resid = nullptr;
    int resid_f32 = 0;
    long long ldr = 0;
    void* out = nullptr;
    int out_f32 = 0;
    long long ldc = 0;
    int act = ACT_NONE;
    int mode = EPI_NORMAL;
    const float* fin_w = nullptr;
    float fin_b = 0.f;
};

struct ConvGeom {
    int N, H, W, Cin;      // input NHWC (Cin multiple of 64)
    long long in_ld;       // channel stride of the input buffer in elements (>= Cin)
    int kh, kw, stride, pad, dil;
    int Cout;
};

// A prepared launch: tensor maps + arguments.  Built once per (layer, buffer set), launched many times.
struct GemmPlan {
    GemmMaps maps;
    GemmArgs args;
    int block_n;
    int grid;      // CTAs to launch
    double flops;  // 2*M*N*K of the true problem (for roofline accounting)
};

// All return 0 on success, nonzero on failure (message via ytk::last_error()).
int conv_plan_create(GemmPlan* plan, const void* in, const ConvGeom& g, const void* w_packed, const Epilogue& e);
// A: [M, lda] bf16 row-major (K multiple of 64, first K columns used); Wt: [N, K] bf16 row-major.
int gemm_plan_create(GemmPlan* plan, const void* A, long long lda, int M, int K, const void* Wt, int N,
                     const Epilogue& e);
// ResNet stem: 7x7 stride-2 pad-3 conv over a zero-padded 8-channel NHWC canvas [N, Hn+6, Wn+8, 8] (pixel (h,w) at
// (h+3, w+3)).  One K block = one filter row = 8 pixels x 8 channels = 64 contiguous bf16, fetched with TMA boxes whose
// rows overlap in memory (W stride = 2 pixels).  w_packed: [Cout][7][64] bf16.
int stem_plan_create(GemmPlan* plan, const void* in_padded, int N, int Hn, int Wn, const void* w_packed,
                     const Epilogue& e);
// Same but the M extent can be changed per launch (rows beyond M are never stored).
void gemm_plan_set_m(GemmPlan* plan, int M);
// Points a prepared plan at another output buffer of the same shape and pitch (the AR loop's K/V cache slot of the
// step); re-encodes the output tensor map when the plan stores through TMA.  Returns 0 on success.
int gemm_plan_set_out(GemmPlan* plan, void* out);
int gemm_plan_launch(const GemmPlan* plan, cudaStream_t stream);

// Generic 4-D tiled bf16 tensor map with 128B swizzle (dims/strides innermost first; strides in bytes for dims 1..3).
int make_tmap_op_4d(CUtensorMap* m, const void* base, const uint64_t dims[4], const uint64_t strides_b[3],
                      const uint32_t box[4]);

// Launch attribute set for kernels that call pdl_wait() (ptx.cuh): programmatic stream serialization when YTK_PDL=1
// (off by default, see gemm_tc.cu).  Returns the number of attributes written to attr[0..].
int pdl_launch_attr(cudaLaunchAttribute* attr);
void set_error(const char* fmt, ...);
const char* last_error();
int num_sms();
// Function attributes (the dynamic shared memory limit) are per device: returns true the first time it is called for
// `*mask` on the calling thread's current device (bit d of the mask = done on device d).
bool first_launch_on_device(unsigned long long* mask);
void count_launch(int n = 1);
long long launch_count();
// Timing window over gemm_tc_kernel launches: CUDA events on the launching stream around every launch between begin and
// end; end() returns the summed algorithmic FLOPs, the summed kernel durations (ms) and the launch count.
void gemm_profile_begin();
int gemm_profile_end(double* flops, double* ms, long long* launches);

}  // namespace ytk
