// Pages that are already on the device into the page-table buffer every page op reads (ytk_page, include/
// yomitoku_b200.h): what a host page gets from the staging copy and the upload, for a page a decoder or an earlier model
// left in HBM.  Each source page is any strided H x W x 3 uint8 view - a contiguous HWC page, a crop or a step of one,
// the permute(1, 2, 0) of a CHW decode - in BGR or RGB order; the destination is H x W x 3 BGR rows back to back.
//
//   pack_pages_kernel  one page per blockIdx.y, a grid-stride loop over its pixels; three byte loads and three byte
//                      stores per pixel.  A byte copy: the result is exact.
#include "page_ops.h"

#include "gemm_tc.h"

namespace ytk {

static constexpr int kPackThreads = 256, kPackMaxBlocks = 1024;

__global__ void __launch_bounds__(kPackThreads) pack_pages_kernel(const PageSrc* __restrict__ srcs,
                                                                   const RtSrc* __restrict__ table,
                                                                   uint8_t* __restrict__ dst) {
    const PageSrc s = srcs[blockIdx.y];
    uint8_t* out = dst + table[blockIdx.y].page_off;
    const long long total = (long long)s.H * s.W;
    // channel c of the output (B, G, R) is source channel c, or 2 - c for an RGB source
    const long long c0 = s.rgb ? 2 * s.sc : 0, dc = s.rgb ? -s.sc : s.sc;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int y = (int)(idx / s.W), x = (int)(idx - (long long)y * s.W);
        const uint8_t* p = s.data + y * s.sh + x * s.sw + c0;
        const uint8_t b = __ldg(p), g = __ldg(p + dc), r = __ldg(p + 2 * dc);
        uint8_t* o = out + idx * 3;
        o[0] = b;
        o[1] = g;
        o[2] = r;
    }
}

int launch_pack_pages(const PageSrc* srcs_dev, const RtSrc* table_dev, int n, long long max_pixels, uint8_t* dst,
                      cudaStream_t st) {
    if (n <= 0 || max_pixels <= 0) return 0;
    if (n > 65535) return 1;
    const long long b = (max_pixels + kPackThreads - 1) / kPackThreads;
    const unsigned blocks = (unsigned)(b < kPackMaxBlocks ? b : kPackMaxBlocks);
    pack_pages_kernel<<<dim3(blocks, (unsigned)n), kPackThreads, 0, st>>>(srcs_dev, table_dev, dst);
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

}  // namespace ytk
