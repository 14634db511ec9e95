// TEST INFRASTRUCTURE ONLY - host instantiation of yomitoku_b200/csrc/crop_math.h.
//
// The product's device-side crop extraction (csrc/crop_ops.cu) is two thin CUDA kernels around the per-pixel bodies in
// crop_math.h.  This file compiles the very same bodies with g++ (no CUDA) into oracle/_build/libcrop_host.so so that
// tests/test_crop_math.py can pin them, on the CPU and bit for bit, against what the reference executes for row R4:
// cv2.warpPerspective / cv2.rotate / cv2.resize(INTER_AREA) as called by reference
// src/yomitoku/data/functions.py:301-439 (OpenCV 4.13, the version the reference's uv.lock pins).
// Only tests/ loads this library; the product never does (no CPU fallback on the hot path).
//
// Build: g++ -O2 -ffp-contract=off -shared -fPIC oracle/crop_host.cpp -o oracle/_build/libcrop_host.so
//        (oracle/build_crop_host.py, also run by __graft_entry__.build()).
#include "../yomitoku_b200/csrc/crop_math.h"

extern "C" {

int crop_host_geom_size(void) { return (int)sizeof(ytk::CropGeom); }

// Whole row R4 for n crops of same-size pages [n_pages][H0][W0][3]: warp (+ rotation) into scratch, then area resize +
// paste into the canvases.
void crop_host_extract(const uint8_t* pages, int H0, int W0, const ytk::CropGeom* g, int n, uint8_t* scratch,
                       uint8_t* canvases) {
    for (int i = 0; i < n; ++i) {
        const uint8_t* page = pages + (long long)g[i].page * H0 * W0 * 3;
        for (int y = 0; y < g[i].h; ++y)
            for (int x = 0; x < g[i].w; ++x) ytk::warp_store_page(g[i], page, W0, x, y, scratch);
        for (int cy = 0; cy < g[i].canvas_h; ++cy)
            for (int cx = 0; cx < g[i].canvas_w; ++cx) ytk::canvas_store(g[i], scratch, cx, cy, canvases);
    }
}

// cv2.resize(src, (dw, dh), INTER_AREA) alone (shrinking only).
void crop_host_area(const uint8_t* src, int sw, int sh, int dw, int dh, uint8_t* dst) {
    for (int y = 0; y < dh; ++y)
        for (int x = 0; x < dw; ++x) ytk::area_pixel(src, sw, sh, dw, dh, x, y, dst + ((long long)y * dw + x) * 3);
}

// cv2.resize(src, None, fx=0.5, fy=0.5, INTER_AREA): dst is [dh][dw][3] with dw = cvRound(sw / 2), dh = cvRound(sh / 2).
void crop_host_halve(const uint8_t* src, int sw, int sh, int dw, int dh, uint8_t* dst) {
    for (int y = 0; y < dh; ++y)
        for (int x = 0; x < dw; ++x) ytk::halve_pixel(src, sw, sh, x, y, dst + ((long long)y * dw + x) * 3);
}

}  // extern "C"
