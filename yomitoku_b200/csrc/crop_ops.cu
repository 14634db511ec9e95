// Device-side crop extraction for the recognizer (SURVEY.md section 8a row R4, section 8f-1): what the reference does
// per text line with OpenCV on 8 host threads (ParseqDataset._preprocess_on, reference src/yomitoku/data/dataset.py:
// 106-123 -> data/functions.py:301-439) as two kernels over ALL crops of ALL pages of a step, reading the pages that
// are already in HBM for the detector and writing the packed canvases the PARSeq patchify kernel consumes - no crop
// pixel crosses PCIe.
//
//   crop_warp_kernel    cv2.warpPerspective (bilinear, 1/32-px fixed point, zero border outside the quad's bounding
//                       box) + the 90-degree rotation of tall crops -> rectified RGB ROI in a scratch buffer
//   crop_canvas_kernel  cv2.resize(INTER_AREA) of the ROI (shrinking only) pasted top-left on a black canvas
//   halve_pages_kernel  one level of the source_downscale pyramid: cv2.resize(page, None, fx=0.5, fy=0.5, INTER_AREA)
//
// The pages are described by a page table (RtSrc records: byte offset and size of each page in one flat buffer, so
// pages of different sizes share a launch).
//
// The arithmetic lives in crop_math.h and is compiled for the host as well (oracle/crop_host.cpp), where the CPU tests
// pin it bit for bit against OpenCV.  This file MUST be compiled with --fmad=false (yomitoku_b200/build.py): OpenCV's
// float / double expressions are not fused.  Both kernels are tiny, HBM/latency-bound byte work (~30 MB per 16-page
// step): one crop per blockIdx.x, blockIdx.y strides over its pixels, the record is staged in shared memory.
#include "crop_ops.h"

#include <climits>

#include "gemm_tc.h"

namespace ytk {

static constexpr int kWarpThreads = 128, kWarpSlices = 4;
static constexpr int kCanvasThreads = 128, kCanvasSlices = 8;

__device__ __forceinline__ void load_geom(CropGeom* sg, const CropGeom* g) {
    static_assert(sizeof(CropGeom) % 8 == 0, "CropGeom is copied as 8-byte words");
    const long long* src = reinterpret_cast<const long long*>(g);
    long long* dst = reinterpret_cast<long long*>(sg);
    for (int i = threadIdx.x; i < (int)(sizeof(CropGeom) / 8); i += blockDim.x) dst[i] = src[i];
    __syncthreads();
}

// crop g reads page table[g.page] of `pages`
__global__ void __launch_bounds__(kWarpThreads) crop_warp_kernel(const uint8_t* __restrict__ pages,
                                                                  const RtSrc* __restrict__ table,
                                                                  const CropGeom* __restrict__ geoms,
                                                                  uint8_t* __restrict__ scratch) {
    __shared__ CropGeom g;
    load_geom(&g, geoms + blockIdx.x);
    const uint8_t* page = pages + table[g.page].page_off;
    const int W = table[g.page].W;
    const int npix = g.w * g.h;
    for (int p = blockIdx.y * blockDim.x + threadIdx.x; p < npix; p += gridDim.y * blockDim.x) {
        const int y = p / g.w;
        warp_store_page(g, page, W, p - y * g.w, y, scratch);
    }
}

__global__ void __launch_bounds__(kCanvasThreads) crop_canvas_kernel(const CropGeom* __restrict__ geoms,
                                                                      const uint8_t* __restrict__ scratch,
                                                                      uint8_t* __restrict__ canvases) {
    __shared__ CropGeom g;
    load_geom(&g, geoms + blockIdx.x);
    const int npix = g.canvas_w * g.canvas_h;
    for (int p = blockIdx.y * blockDim.x + threadIdx.x; p < npix; p += gridDim.y * blockDim.x) {
        const int cy = p / g.canvas_w;
        canvas_store(g, scratch, p - cy * g.canvas_w, cy, canvases);
    }
}

// One page per blockIdx.y: page img of src_table -> page img of dst_table.
__global__ void halve_pages_kernel(const uint8_t* __restrict__ src, const RtSrc* __restrict__ src_table,
                                   uint8_t* __restrict__ dst, const RtSrc* __restrict__ dst_table) {
    const RtSrc a = src_table[blockIdx.y], b = dst_table[blockIdx.y];
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= b.H * b.W) return;
    const int y = idx / b.W;
    halve_pixel(src + a.page_off, a.W, a.H, idx - y * b.W, y, dst + b.page_off + (long long)idx * 3);
}

int launch_halve_pages_table(const uint8_t* src, const RtSrc* src_table_dev, int n, uint8_t* dst,
                             const RtSrc* dst_table_dev, long long max_dst_pixels, cudaStream_t st) {
    if (n <= 0 || max_dst_pixels <= 0) return 0;
    if (n > 65535 || max_dst_pixels > INT_MAX) return 1;
    halve_pages_kernel<<<dim3((unsigned)((max_dst_pixels + 255) / 256), (unsigned)n), 256, 0, st>>>(
        src, src_table_dev, dst, dst_table_dev);
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

int launch_extract_crops_table(const uint8_t* pages, const RtSrc* table_dev, const CropGeom* geoms_dev, int n_crops,
                               uint8_t* scratch, uint8_t* canvases, cudaStream_t st) {
    if (n_crops <= 0) return 0;
    crop_warp_kernel<<<dim3((unsigned)n_crops, kWarpSlices), kWarpThreads, 0, st>>>(pages, table_dev, geoms_dev,
                                                                                    scratch);
    count_launch();
    if (cudaGetLastError() != cudaSuccess) return 1;
    crop_canvas_kernel<<<dim3((unsigned)n_crops, kCanvasSlices), kCanvasThreads, 0, st>>>(geoms_dev, scratch,
                                                                                          canvases);
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

}  // namespace ytk
