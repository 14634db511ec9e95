// Launchers of the memory-bound DBNet++ kernels (dbnet_ops.cu).  All return 0 on success.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "resample_math.h"  // RtSrc: the page record of a page table

namespace ytk {

constexpr int kAsfPoolChunks = 64;   // launch_asf: gsum holds n_img * kAsfPoolChunks * 64 floats (partial channel sums)

// BGR u8 pages of any sizes in one buffer: page i is table_dev[i] (whole pages, on the device), all resized to (Hn, Wn)
// by cv2.resize(INTER_AREA) either way: each page gets area resampling when neither of its axes grows, OpenCV's
// bilinear up-scaling otherwise
int launch_preprocess_table(const uint8_t* pages, const RtSrc* table_dev, int n_img, int Hn, int Wn,
                            void* dst_padded_nhwc8, cudaStream_t st);
int launch_pack_nchw_f32(const float* src_nchw, int n_img, int Hn, int Wn, void* dst_padded_nhwc8, cudaStream_t st);
int launch_maxpool(const void* in, void* out, int n_img, int H, int W, int C, cudaStream_t st);
int launch_upsample(const void* src, int n_img, int Hs, int Ws, int C, void* dst, int Hd, int Wd, long long ldd,
                    int coff, int accumulate, cudaStream_t st);
int launch_asf(const void* a, void* fuse, int n_img, int H, int W, const float* w1_dev, const float* w2_dev,
               const float* host_sp3, float host_sp1, const float* host_att, float* gsum, float* gvec, float* gmean,
               float* m, cudaStream_t st);
int launch_op_to_f32(const void* in, float* out, long long n, cudaStream_t st);

}  // namespace ytk
