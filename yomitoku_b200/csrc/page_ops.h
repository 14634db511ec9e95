// Launcher of the page packing kernel (page_ops.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "resample_math.h"  // RtSrc: the page record of a page table

namespace ytk {

// One source page of the pack: the layout of ytk_page_src (include/yomitoku_b200.h).
struct PageSrc {
    const uint8_t* data;   // pixel (0, 0), channel 0
    long long sh, sw, sc;  // byte strides of a row, a column and a channel
    int H, W;
    int rgb;               // 0: channels B, G, R; 1: R, G, B
    int pad_;
};

// Page i of srcs_dev -> page i of the page table table_dev in dst, as H x W x 3 BGR bytes.  Records on the device,
// checked by the caller; max_pixels: the largest H * W.  One launch on `st`.
int launch_pack_pages(const PageSrc* srcs_dev, const RtSrc* table_dev, int n, long long max_pixels, uint8_t* dst,
                      cudaStream_t st);

}  // namespace ytk
