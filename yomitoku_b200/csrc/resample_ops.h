// Device resize of u8 BGR pages (resample_ops.cu): Pillow's BILINEAR or LANCZOS resize of page rectangles, each to its
// own output size, written as the RT-DETRv2 engine input, as u8 RGB or as planar u8 RGB.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "resample_math.h"

namespace ytk {

// One source of a call: the rectangle of a page, its output size and where its output starts (bytes into `out`).
struct ResampleSrc {
    RtSrc src;
    int out_w, out_h;
    long long out_off;
};

// Device copy of one source with where its coefficients and its first-pass intermediate live.
struct ResamplePlan {
    RtSrc src;
    long long cx_off, cy_off;  // int offsets of the cw -> out_w and ch -> out_h coefficient tables in the table block
    long long inter_off;       // byte offset of the u8 RGB intermediate in the scratch buffer
    long long out_off;         // byte offset of the output in `out`
    int kx, ky;                // ksize of the two tables
    int out_w, out_h;
    int passes, icols;         // resample_passes bits; columns of the intermediate (0: none)
    int pad_[2];
};

// Output layouts: the RT-DETRv2 engine input (NHWC, 64 16-bit channels, 3 real: the values pack_input_kernel makes of
// ToTensor's output), [out_h][out_w][3] u8 RGB, or [3][out_h][out_w] u8 RGB (what torchvision's encode_jpeg takes).
enum ResampleOut : int { kOutEngine = 0, kOutRGB = 1, kOutPlanar = 2 };

// One call's scratch buffer: [plans][coefficient tables][intermediates], 16-byte aligned parts.  `host` is the first
// two parts, uploaded with one copy.
struct ResampleJob {
    int n = 0;
    std::vector<unsigned char> host;
    long long coef_off = 0, bytes = 0;
    long long max_inter = 0;   // most intermediate pixels of one source (0: no source needs two passes)
    long long max_out = 0;     // most output pixels of one source
};

// Validates the records (a page extent inside pages_bytes, a non-empty rectangle inside its page, an output of at
// least 1 x 1, a known filter) and builds the plans and coefficient tables on the host.  Returns 0, or 1 with
// ytk_last_error set.
int resample_prepare(const ResampleSrc* srcs, int n, int filter, long long pages_bytes, const char* who,
                     ResampleJob* job);
// The sources of the RT-DETRv2 input resize: every rectangle to S x S, output i at i * S * S * pixel_bytes.
std::vector<ResampleSrc> square_sources(const RtSrc* srcs, int n, int S, long long pixel_bytes);
// Uploads job.host to scratch and runs the passes: the first kernel only when some source needs two passes.
int launch_resample(const uint8_t* pages, const ResampleJob& job, uint8_t* scratch, void* out, ResampleOut layout,
                    cudaStream_t st);

}  // namespace ytk
