// Device-side RT-DETRv2 input resize (resample_ops.cu): Pillow's BILINEAR resize of page rectangles to S x S.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "resample_math.h"

namespace ytk {

// Device copy of one source with where its coefficients and its first-pass intermediate live.
struct ResamplePlan {
    RtSrc src;
    long long cx_off, cy_off;  // int offsets of the crop_w -> S and crop_h -> S coefficient tables in the table block
    long long inter_off;       // byte offset of the u8 RGB intermediate in the scratch buffer
    int kx, ky;                // ksize of the two tables
};

// One call's scratch buffer: [plans][coefficient tables][intermediates], 16-byte aligned parts.  `host` is the first
// two parts, uploaded with one copy.
struct ResampleJob {
    int n = 0, S = 0;
    std::vector<unsigned char> host;
    long long coef_off = 0, bytes = 0;
    long long max_inter = 0;   // most intermediate pixels of one source
};

// Validates the records (a page extent inside pages_bytes, a non-empty rectangle inside its page) and builds the plans
// and coefficient tables on the host.  Returns 0, or 1 with ytk_last_error set.
int resample_prepare(const RtSrc* srcs, int n, int S, long long pages_bytes, const char* who, ResampleJob* job);
// Uploads job.host to scratch and runs both passes.  pack = 1: writes the RT-DETRv2 engine input (NHWC, 64 channels
// of op_t, 3 real: the values pack_input_kernel makes of ToTensor's output); pack = 0: [n][S][S][3] u8 RGB.
int launch_resample(const uint8_t* pages, const ResampleJob& job, uint8_t* scratch, void* out, int pack,
                    cudaStream_t st);

}  // namespace ytk
