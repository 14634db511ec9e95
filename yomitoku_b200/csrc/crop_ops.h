// Launcher of the device-side crop extraction (crop_ops.cu; per-pixel arithmetic in crop_math.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "crop_math.h"
#include "resample_math.h"  // RtSrc: the page record of a page table

namespace ytk {

// Page tables: page i of `pages` / `src` / `dst` is table_dev[i], uint8 BGR (records on the device, checked by the
// caller).
//
// geoms_dev: n_crops CropGeom records on the device, crop g on page table_dev[g.page]; scratch / canvases: device
// buffers the records' roi_off / pix_off point into.  Two launches on `st`.
int launch_extract_crops_table(const uint8_t* pages, const RtSrc* table_dev, const CropGeom* geoms_dev, int n_crops,
                               uint8_t* scratch, uint8_t* canvases, cudaStream_t st);
// dst page i = cv2.resize(src page i, None, fx=0.5, fy=0.5, INTER_AREA): dH / dW = cvRound(sH / 2), cvRound(sW / 2)
// (checked by the caller).  max_dst_pixels: the largest dH * dW of the destination pages.
int launch_halve_pages_table(const uint8_t* src, const RtSrc* src_table_dev, int n, uint8_t* dst,
                             const RtSrc* dst_table_dev, long long max_dst_pixels, cudaStream_t st);

}  // namespace ytk
