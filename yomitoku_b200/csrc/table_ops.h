// Launcher of the word-to-element assignment of the table semantic parser (table_ops.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ytk {

// One assignment group on the device: words [w0, w1) against elements [e0, e1); its results start at out_off.
struct OverlapGroup {
    int w0, w1, e0, e1;
    long long out_off;
    long long pad_;
};

// One CTA of the launch: kOverlapThreads words of group `group` from word w.
struct OverlapItem {
    int group, w;
};

static constexpr int kOverlapThreads = 128;

// words / elems: x1, y1, x2, y2 fp64 per box (|coordinate| < 2^30, checked by the caller); skip: one byte per element,
// non-zero = never a candidate.  groups / items on the device.  One launch of n_items CTAs on `st`.
int launch_assign_best_overlap(const double* words, const double* elems, const uint8_t* skip, const OverlapGroup* groups,
                               const OverlapItem* items, int n_items, double overlap_th, int* best, double* ratio,
                               cudaStream_t st);

}  // namespace ytk
