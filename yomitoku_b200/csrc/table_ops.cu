// Word-to-element assignment of the table semantic parser: for every word of a group, the element (table cell or
// paragraph) that covers the largest share of the word's box, as the reference's TableSemanticParser.aggregate decides
// it (src/yomitoku/table_semantic_parser.py:683-701 with utils/misc.py:35-91):
//
//   * both boxes are truncated toward zero to integers and intersected; a width or height <= 0 is no overlap;
//   * ratio = (integer intersection area) / ((bx2 - bx1) * (by2 - by1)) with b the word's raw fp64 box, IEEE
//     round-to-nearest sub / mul / div with no contraction (the file is also built with --fmad=false);
//   * elements are scanned in order and a candidate replaces the best one only if its ratio is strictly larger,
//     starting from 0, so the first maximum wins and a word without overlap has none;
//   * the result is the element's index, or -1 when there is none or its ratio is below overlap_th.
//
//   assign_best_overlap_kernel  one CTA per (group, 128 words); each thread owns one word.  The group's elements pass
//                               through shared memory in tiles of kTile truncated boxes, so a group may have any
//                               number of elements; a skipped element is staged as an empty box.
#include "table_ops.h"

#include "gemm_tc.h"

namespace ytk {

static constexpr int kTile = 1024;  // elements per shared-memory tile: 16 KB of int4

__global__ void __launch_bounds__(kOverlapThreads) assign_best_overlap_kernel(
    const double4* __restrict__ words, const double4* __restrict__ elems, const uint8_t* __restrict__ skip,
    const OverlapGroup* __restrict__ groups, const OverlapItem* __restrict__ items, double overlap_th,
    int* __restrict__ best, double* __restrict__ ratio) {
    __shared__ int4 tile[kTile];
    const OverlapItem it = items[blockIdx.x];
    const OverlapGroup g = groups[it.group];
    const int w = it.w + (int)threadIdx.x;
    const bool active = w < g.w1;
    int4 wi = make_int4(0, 0, 0, 0);
    double b_area = 1.0;
    if (active) {
        const double4 wb = words[w];
        wi = make_int4(__double2int_rz(wb.x), __double2int_rz(wb.y), __double2int_rz(wb.z), __double2int_rz(wb.w));
        b_area = __dmul_rn(__dsub_rn(wb.z, wb.x), __dsub_rn(wb.w, wb.y));
    }
    int bi = -1;
    double br = 0.0;
    for (int t0 = g.e0; t0 < g.e1; t0 += kTile) {
        const int n = min(kTile, g.e1 - t0);
        __syncthreads();  // the previous tile is no longer read
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const double4 e = elems[t0 + i];
            tile[i] = skip[t0 + i] ? make_int4(1, 1, 0, 0)
                                   : make_int4(__double2int_rz(e.x), __double2int_rz(e.y), __double2int_rz(e.z),
                                               __double2int_rz(e.w));
        }
        __syncthreads();
        if (!active) continue;
        for (int i = 0; i < n; ++i) {
            const int4 e = tile[i];
            const int iw = min(e.z, wi.z) - max(e.x, wi.x);
            const int ih = min(e.w, wi.w) - max(e.y, wi.y);
            if (iw <= 0 || ih <= 0) continue;
            const double r = __ddiv_rn((double)((long long)iw * ih), b_area);
            if (r > br) {
                br = r;
                bi = t0 + i;
            }
        }
    }
    if (active) {
        const long long o = g.out_off + (w - g.w0);
        best[o] = (bi < 0 || br < overlap_th) ? -1 : bi;
        ratio[o] = br;
    }
}

int launch_assign_best_overlap(const double* words, const double* elems, const uint8_t* skip, const OverlapGroup* groups,
                               const OverlapItem* items, int n_items, double overlap_th, int* best, double* ratio,
                               cudaStream_t st) {
    if (n_items <= 0) return 0;
    assign_best_overlap_kernel<<<(unsigned)n_items, kOverlapThreads, 0, st>>>(
        reinterpret_cast<const double4*>(words), reinterpret_cast<const double4*>(elems), skip, groups, items,
        overlap_th, best, ratio);
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

}  // namespace ytk
