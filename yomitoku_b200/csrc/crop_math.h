// Per-pixel arithmetic of the recognizer's crop extraction (SURVEY.md section 8a row R4 / section 8f-1), written ONCE
// for host and device: crop_ops.cu wraps these bodies in CUDA kernels, oracle/crop_host.cpp instantiates the very same
// functions with g++ so that the `-m "not gpu"` tests can pin them bit-for-bit against OpenCV on the CPU.
//
// What is restated (the reference calls OpenCV 4.13 for all of it):
//   * extract_roi_with_perspective  (reference src/yomitoku/data/functions.py:301-333)
//       cv2.warpPerspective(roi, M, (w, h)), INTER_LINEAR, BORDER_CONSTANT(0), 8UC3: OpenCV's WarpPerspectiveInvoker
//       (inverse map in double, evaluated per block of bw0 columns, coordinates rounded to 1/32 px) + remapBilinear's
//       15-bit fixed-point weights ((32-ax)(32-ay)*32 etc., exact, so no table fix-up is ever needed);
//   * rotate_text_image             (functions.py:336-350)   cv2.ROTATE_90_COUNTERCLOCKWISE when h > 2w;
//   * resize_with_padding / resize_with_dynamic_padding (functions.py:379-439)
//       cv2.resize(..., INTER_AREA) for shrinking only: identity copy, the integer-ratio "area fast" path
//       (2x2: (sum+2)>>2, otherwise rint(float(sum) * (1.f/area))) and the general DecimateAlpha path (float32
//       accumulation in OpenCV's tap order, no fused multiply-add), pasted top-left on a black canvas.
// Every floating-point operation below must stay un-fused: crop_ops.cu is compiled with --fmad=false and the host
// harness with -ffp-contract=off.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define YTK_HD __host__ __device__ __forceinline__
#else
#define YTK_HD static inline
#endif

namespace ytk {

// One crop; computed on the host from the quad alone (yomitoku_b200/data.py: crop_geometry).  Same layout as
// ytk_crop_geom in include/yomitoku_b200.h.
struct CropGeom {
    double minv[9];     // inverse of getPerspectiveTransform(quad - origin, [[0,0],[w,0],[w,h],[0,h]]) (cv2.invert)
    long long roi_off;  // byte offset of the rectified (and rotated) ROI in the scratch buffer: [rh2][rw2][3] RGB
    long long pix_off;  // byte offset of the canvas in the packed crop buffer: [canvas_h][canvas_w][3] RGB
    int page;           // page index
    int x0, y0, rw, rh; // bounding-box slice of the quad inside the page (the image warpPerspective sees)
    int w, h;           // size of the rectified ROI before rotation: (int |p0p1|, int |p1p2|)
    int rot;            // bit 0: rotate 90 degrees counter-clockwise after the warp (h > 2w, rotate_text_image);
                        // bit 1: then rotate by 180 degrees (orientation fallback, text_recognizer.py:319-328)
    int cw, ch;         // content size after the area resize (calc_resize_without_padding)
    int canvas_w, canvas_h;
};

YTK_HD int round_half_even_d(double v) {
#ifdef __CUDA_ARCH__
    return __double2int_rn(v);
#else
    return (int)nearbyint(v);  // default rounding mode = to nearest even = cvRound
#endif
}

YTK_HD int round_half_even_f(float v) {
#ifdef __CUDA_ARCH__
    return __float2int_rn(v);
#else
    return (int)nearbyintf(v);
#endif
}

YTK_HD int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// Block width OpenCV evaluates the inverse map in (WarpPerspectiveInvoker: BLOCK_SZ = 32).
YTK_HD int warp_block_width(int w, int h) {
    int bh0 = h < 16 ? h : 16;
    if (bh0 < 1) bh0 = 1;
    int bw0 = 1024 / bh0;
    if (bw0 > w) bw0 = w;
    return bw0 < 1 ? 1 : bw0;
}

// Source coordinate of destination pixel (x, y) in 1/32 px: integer part (ix, iy) and 5-bit fractions (ax, ay).
YTK_HD void warp_coord(const double* M, int x, int y, int bw0, int* ix, int* iy, int* ax, int* ay) {
    const int bx = (x / bw0) * bw0;
    const int x1 = x - bx;
    const double X0 = M[0] * bx + M[1] * y + M[2];
    const double Y0 = M[3] * bx + M[4] * y + M[5];
    const double W0 = M[6] * bx + M[7] * y + M[8];
    double W = W0 + M[6] * x1;
    W = W != 0.0 ? 32.0 / W : 0.0;
    double fX = (X0 + M[0] * x1) * W;
    double fY = (Y0 + M[3] * x1) * W;
    fX = fX < 2147483647.0 ? fX : 2147483647.0;
    fX = fX > -2147483648.0 ? fX : -2147483648.0;
    fY = fY < 2147483647.0 ? fY : 2147483647.0;
    fY = fY > -2147483648.0 ? fY : -2147483648.0;
    const int X = round_half_even_d(fX), Y = round_half_even_d(fY);
    *ix = clampi(X >> 5, -32768, 32767);
    *iy = clampi(Y >> 5, -32768, 32767);
    *ax = X & 31;
    *ay = Y & 31;
}

// Rectified pixel (x, y) of crop g, written at its rotated position into the scratch ROI (RGB order: the reference
// hands ParseqDataset the page as img[:, :, ::-1], data/dataset.py:69).  page: the crop's own BGR page, rows of W0 * 3
// bytes (g.page has already been resolved by the caller).
YTK_HD void warp_store_page(const CropGeom& g, const uint8_t* page, int W0, int x, int y, uint8_t* scratch) {
    int ix, iy, ax, ay;
    warp_coord(g.minv, x, y, warp_block_width(g.w, g.h), &ix, &iy, &ax, &ay);
    const int w00 = (32 - ax) * (32 - ay), w01 = ax * (32 - ay), w10 = (32 - ax) * ay, w11 = ax * ay;
    const uint8_t* base = page + (long long)g.y0 * W0 * 3 + (long long)g.x0 * 3;
    const bool x0ok = ix >= 0 && ix < g.rw, x1ok = ix + 1 >= 0 && ix + 1 < g.rw;
    const bool y0ok = iy >= 0 && iy < g.rh, y1ok = iy + 1 >= 0 && iy + 1 < g.rh;
    const uint8_t* r0 = base + (long long)iy * W0 * 3 + (long long)ix * 3;
    const uint8_t* r1 = r0 + (long long)W0 * 3;
    int v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int p00 = (y0ok && x0ok) ? r0[c] : 0, p01 = (y0ok && x1ok) ? r0[3 + c] : 0;
        const int p10 = (y1ok && x0ok) ? r1[c] : 0, p11 = (y1ok && x1ok) ? r1[3 + c] : 0;
        // 15-bit weights are 32 * (5-bit products): (sum * 32 + 2^14) >> 15 == (sum + 512) >> 10
        v[c] = (p00 * w00 + p01 * w01 + p10 * w10 + p11 * w11 + 512) >> 10;
    }
    int orow, ocol, opitch, orows;
    if (g.rot & 1) {  // ROTATE_90_COUNTERCLOCKWISE: dst (w rows x h cols), dst[i][j] = src[j][w-1-i]
        orow = g.w - 1 - x;
        ocol = y;
        opitch = g.h;
        orows = g.w;
    } else {
        orow = y;
        ocol = x;
        opitch = g.w;
        orows = g.h;
    }
    if (g.rot & 2) {  // ROTATE_180 of that image: dst[i][j] = src[rows-1-i][cols-1-j]
        orow = orows - 1 - orow;
        ocol = opitch - 1 - ocol;
    }
    uint8_t* o = scratch + g.roi_off + ((long long)orow * opitch + ocol) * 3;
    o[0] = (uint8_t)v[2];  // BGR page -> RGB crop
    o[1] = (uint8_t)v[1];
    o[2] = (uint8_t)v[0];
}

// The same for same-size pages: [n][H0][W0][3] BGR, crop g on page g.page.
YTK_HD void warp_store(const CropGeom& g, const uint8_t* pages, int H0, int W0, int x, int y, uint8_t* scratch) {
    warp_store_page(g, pages + (long long)g.page * H0 * W0 * 3, W0, x, y, scratch);
}

// Taps of one destination index along one axis of cv2.resize(INTER_AREA) (computeResizeAreaTab): an optional partial
// left cell, whole cells [s1, s2), an optional partial right cell.
struct AreaTaps {
    int s1, s2;
    bool left, right;
    float a_left, a_mid, a_right;
};

YTK_HD AreaTaps area_taps(int ssize, double scale, int d) {
    AreaTaps t;
    const double fsx1 = d * scale;
    const double fsx2 = fsx1 + scale;
    const double rest = (double)ssize - fsx1;
    const double cell = scale < rest ? scale : rest;
    int sx1 = (int)ceil(fsx1), sx2 = (int)floor(fsx2);
    if (sx2 > ssize - 1) sx2 = ssize - 1;
    if (sx1 > sx2) sx1 = sx2;
    t.s1 = sx1;
    t.s2 = sx2;
    t.left = (double)sx1 - fsx1 > 1e-3;
    t.a_left = (float)(((double)sx1 - fsx1) / cell);
    t.a_mid = (float)(1.0 / cell);
    const double r = fsx2 - (double)sx2;
    t.right = r > 1e-3;
    double m = r < 1.0 ? r : 1.0;
    m = m < cell ? m : cell;
    t.a_right = (float)(m / cell);
    return t;
}

YTK_HD void area_row(const uint8_t* S, const AreaTaps& tx, float* buf) {
    buf[0] = buf[1] = buf[2] = 0.f;
    if (tx.left) {
        const uint8_t* p = S + (long long)(tx.s1 - 1) * 3;
        for (int c = 0; c < 3; ++c) buf[c] = buf[c] + (float)p[c] * tx.a_left;
    }
    for (int sx = tx.s1; sx < tx.s2; ++sx) {
        const uint8_t* p = S + (long long)sx * 3;
        for (int c = 0; c < 3; ++c) buf[c] = buf[c] + (float)p[c] * tx.a_mid;
    }
    if (tx.right) {
        const uint8_t* p = S + (long long)tx.s2 * 3;
        for (int c = 0; c < 3; ++c) buf[c] = buf[c] + (float)p[c] * tx.a_right;
    }
}

YTK_HD uint8_t sat_u8(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// Pixel (dx, dy) of cv2.resize(src [sh][sw][3], (dw, dh), INTER_AREA), dw <= sw, dh <= sh.
YTK_HD void area_pixel(const uint8_t* src, int sw, int sh, int dw, int dh, int dx, int dy, uint8_t* out) {
    if (dw == sw && dh == sh) {
        const uint8_t* p = src + ((long long)dy * sw + dx) * 3;
        out[0] = p[0]; out[1] = p[1]; out[2] = p[2];
        return;
    }
    const double inv_x = (double)dw / sw, inv_y = (double)dh / sh;
    const double scale_x = 1.0 / inv_x, scale_y = 1.0 / inv_y;
    const int isx = round_half_even_d(scale_x), isy = round_half_even_d(scale_y);
    const double eps = 2.220446049250313e-16;
    if (fabs(scale_x - isx) < eps && fabs(scale_y - isy) < eps) {
        int sum[3] = {0, 0, 0};
        for (int j = 0; j < isy; ++j) {
            const uint8_t* p = src + ((long long)(dy * isy + j) * sw + (long long)dx * isx) * 3;
            for (int i = 0; i < isx; ++i, p += 3) {
                sum[0] += p[0]; sum[1] += p[1]; sum[2] += p[2];
            }
        }
        if (isx == 2 && isy == 2) {
            for (int c = 0; c < 3; ++c) out[c] = (uint8_t)((sum[c] + 2) >> 2);
        } else {
            const float sc = 1.f / (float)(isx * isy);
            for (int c = 0; c < 3; ++c) out[c] = sat_u8(round_half_even_f((float)sum[c] * sc));
        }
        return;
    }
    const AreaTaps tx = area_taps(sw, scale_x, dx), ty = area_taps(sh, scale_y, dy);
    float sum[3] = {0.f, 0.f, 0.f}, buf[3];
    bool first = true;
    if (ty.left) {
        area_row(src + (long long)(ty.s1 - 1) * sw * 3, tx, buf);
        for (int c = 0; c < 3; ++c) sum[c] = ty.a_left * buf[c];
        first = false;
    }
    for (int sy = ty.s1; sy < ty.s2; ++sy) {
        area_row(src + (long long)sy * sw * 3, tx, buf);
        for (int c = 0; c < 3; ++c) sum[c] = first ? ty.a_mid * buf[c] : sum[c] + ty.a_mid * buf[c];
        first = false;
    }
    if (ty.right) {
        area_row(src + (long long)ty.s2 * sw * 3, tx, buf);
        for (int c = 0; c < 3; ++c) sum[c] = first ? ty.a_right * buf[c] : sum[c] + ty.a_right * buf[c];
        first = false;
    }
    for (int c = 0; c < 3; ++c) out[c] = sat_u8(round_half_even_f(sum[c]));
}

// Pixel (dx, dy) of cv2.resize(src [sh][sw][3], None, fx=0.5, fy=0.5, INTER_AREA): one level of the source_downscale
// pyramid (reference data/dataset.py:64-86).  dw = cvRound(sw * 0.5), dh = cvRound(sh * 0.5) (round half to even).
// OpenCV's integer-ratio path: full 2x2 cells round half up ((sum + 2) >> 2); the clipped last column / row of an odd
// size averages the pixels that exist, rint((float)sum / count).
YTK_HD void halve_pixel(const uint8_t* src, int sw, int sh, int dx, int dy, uint8_t* out) {
    const int sx0 = 2 * dx, sy0 = 2 * dy;
    if (sy0 + 2 <= sh && dx < sw / 2) {
        const uint8_t* p = src + ((long long)sy0 * sw + sx0) * 3;
        const uint8_t* q = p + (long long)sw * 3;
        for (int c = 0; c < 3; ++c) out[c] = (uint8_t)((p[c] + p[3 + c] + q[c] + q[3 + c] + 2) >> 2);
        return;
    }
    int sum[3] = {0, 0, 0}, count = 0;
    for (int sy = 0; sy < 2 && sy0 + sy < sh; ++sy)
        for (int sx = 0; sx < 2 && sx0 + sx < sw; ++sx) {
            const uint8_t* p = src + ((long long)(sy0 + sy) * sw + sx0 + sx) * 3;
            sum[0] += p[0]; sum[1] += p[1]; sum[2] += p[2];
            ++count;
        }
    for (int c = 0; c < 3; ++c) out[c] = count ? sat_u8(round_half_even_f((float)sum[c] / (float)count)) : (uint8_t)0;
}

// Canvas pixel (cx, cy) of crop g: the resized content top-left, black elsewhere.
YTK_HD void canvas_store(const CropGeom& g, const uint8_t* scratch, int cx, int cy, uint8_t* canvases) {
    uint8_t v[3] = {0, 0, 0};
    if (cx < g.cw && cy < g.ch) {
        const int sw = (g.rot & 1) ? g.h : g.w, sh = (g.rot & 1) ? g.w : g.h;
        area_pixel(scratch + g.roi_off, sw, sh, g.cw, g.ch, cx, cy, v);
    }
    uint8_t* o = canvases + g.pix_off + ((long long)cy * g.canvas_w + cx) * 3;
    o[0] = v[0]; o[1] = v[1]; o[2] = v[2];
}

}  // namespace ytk
