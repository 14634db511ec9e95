// Per-pixel arithmetic of the RT-DETRv2 input resize (csrc/resample_ops.cu), written ONCE for host and device:
// resample_ops.cu wraps these bodies in CUDA kernels, oracle/resample_host.cpp instantiates the very same functions with
// g++ so that the `-m "not gpu"` tests can pin them bit for bit against Pillow on the CPU.
//
// What is restated: Image.fromarray(rgb).resize((S, S), Image.BILINEAR) for an 8-bit RGB image (Pillow's
// ImagingResample: no reducing_gap, box = the whole image), which is what the reference's T.Resize does in front of
// the layout parser, the table structure recognizer and the cell detector:
//   * per axis, coefficients in double (precompute_coeffs): scale = in / out, filterscale = max(scale, 1),
//     support = filterscale, ksize = 2 * ceil(support) + 1, the triangle filter evaluated at
//     (x + xmin - center + 0.5) * (1 / filterscale), normalised by the sum, then rounded to 22 fractional bits
//     (normalize_coeffs_8bpc);
//   * two separable passes, each sample an int32 accumulation 2^21 + sum(u8 * k) clipped to [0, 255] after >> 22; the
//     first pass writes a u8 intermediate that the second reads.  The horizontal pass comes first, except for a tall,
//     narrow input that shrinks vertically (resample_vertical_first: measured against Pillow 12.2, which picks the
//     order by the input's shape).
// Pillow skips the pass of an axis whose size does not change; the coefficients of such an axis are the identity
// ([1, 0] at every index), so running the pass anyway gives the same bytes.
// Every floating-point operation below must stay un-fused: resample_ops.cu is compiled with --fmad=false and
// -ffp-contract=off, the host harness with -ffp-contract=off.
#pragma once
#include <math.h>
#include <stdint.h>

#ifndef YTK_HD
#ifdef __CUDACC__
#define YTK_HD __host__ __device__ __forceinline__
#else
#define YTK_HD static inline
#endif
#endif

namespace ytk {

// One model input: page[y0:y1, x0:x1] of the BGR page at byte page_off (H rows of W * 3 bytes).  Same layout as
// ytk_rtdetr_src in include/yomitoku_b200.h.
struct RtSrc {
    long long page_off;
    int H, W;
    int x0, y0, x1, y1;
};

constexpr int kResampleBits = 22;  // Pillow's PRECISION_BITS for 8-bit images: 32 - 8 - 2

// Taps per output index of an in -> out axis.
YTK_HD int bilinear_ksize(int in, int out) {
    const double scale = (double)in / (double)out;
    const double support = scale < 1.0 ? 1.0 : scale;
    return (int)ceil(support) * 2 + 1;
}

YTK_HD double bilinear_filter(double x) {
    if (x < 0.0) x = -x;
    return x < 1.0 ? 1.0 - x : 0.0;
}

// Coefficient table of an in -> out axis: for output index i, tab[i * (ksize + 2)] = first source index, tab[... + 1]
// = number of taps used, then ksize fixed-point weights (zero beyond the used taps).
YTK_HD void bilinear_coeffs(int in, int out, int* tab) {
    const double scale = (double)in / (double)out;
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = filterscale;
    const int ksize = (int)ceil(support) * 2 + 1;
    const double ss = 1.0 / filterscale;
    for (int i = 0; i < out; ++i) {
        const double center = (i + 0.5) * scale;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in) xmax = in;
        xmax -= xmin;
        double ww = 0.0;
        for (int x = 0; x < xmax; ++x) ww += bilinear_filter((x + xmin - center + 0.5) * ss);
        int* t = tab + (long long)i * (ksize + 2);
        t[0] = xmin;
        t[1] = xmax;
        for (int x = 0; x < ksize; ++x) {
            double k = 0.0;
            if (x < xmax) {
                k = bilinear_filter((x + xmin - center + 0.5) * ss);
                if (ww != 0.0) k /= ww;
            }
            const double f = k * (double)(1 << kResampleBits);
            t[2 + x] = k < 0.0 ? (int)(-0.5 + f) : (int)(0.5 + f);
        }
    }
}

YTK_HD uint8_t resample_clip(int acc) {
    acc >>= kResampleBits;
    return (uint8_t)(acc < 0 ? 0 : (acc > 255 ? 255 : acc));
}

// Pillow 12 runs the vertical pass first for a tall, narrow input that shrinks vertically (more than 100 rows per
// column); otherwise the horizontal pass comes first.  The order changes the bytes: the intermediate is rounded to u8.
YTK_HD bool resample_vertical_first(int cw, int ch, int S) { return ch > S && (long long)ch > 100LL * cw; }

// Pixels of the intermediate: [crop_h][S] after a horizontal first pass, [S][crop_w] after a vertical one.
YTK_HD long long resample_inter_pixels(int cw, int ch, int S) {
    return resample_vertical_first(cw, ch, S) ? (long long)S * cw : (long long)ch * S;
}

// One output sample triple: entry i of a coefficient table (ksize k) applied along a line of 3-byte pixels, `step`
// bytes apart; swap = write the channels in reverse order (BGR page -> RGB).
YTK_HD void resample_taps(const uint8_t* line, long long step, const int* tab, int k, int i, bool swap, uint8_t* out) {
    const int* t = tab + (long long)i * (k + 2);
    const int n = t[1];
    const uint8_t* p = line + (long long)t[0] * step;
    int a0 = 1 << (kResampleBits - 1), a1 = a0, a2 = a0;
    for (int x = 0; x < n; ++x, p += step) {
        const int w = t[2 + x];
        a0 += p[0] * w;
        a1 += p[1] * w;
        a2 += p[2] * w;
    }
    out[0] = resample_clip(swap ? a2 : a0);
    out[1] = resample_clip(a1);
    out[2] = resample_clip(swap ? a0 : a2);
}

// First pass, intermediate pixel (r, c): reads the BGR page, writes RGB into inter.  cx / cy: coefficient tables of
// the crop_w -> S and crop_h -> S axes, kx / ky their ksize.
YTK_HD void resample_first(const uint8_t* pages, const RtSrc& s, const int* cx, int kx, const int* cy, int ky, int S, int r,
                           int c, uint8_t* inter) {
    const int cw = s.x1 - s.x0, ch = s.y1 - s.y0;
    const long long pitch = (long long)s.W * 3;
    const uint8_t* crop = pages + s.page_off + (long long)s.y0 * pitch + (long long)s.x0 * 3;
    if (resample_vertical_first(cw, ch, S))
        resample_taps(crop + (long long)c * 3, pitch, cy, ky, r, true, inter + ((long long)r * cw + c) * 3);
    else
        resample_taps(crop + (long long)r * pitch, 3, cx, kx, c, true, inter + ((long long)r * S + c) * 3);
}

// Second pass, output pixel (oy, ox) from the intermediate.
YTK_HD void resample_second(const uint8_t* inter, int cw, int ch, const int* cx, int kx, const int* cy, int ky, int S,
                            int oy, int ox, uint8_t* v) {
    if (resample_vertical_first(cw, ch, S))
        resample_taps(inter + (long long)oy * cw * 3, 3, cx, kx, ox, false, v);
    else
        resample_taps(inter + (long long)ox * 3, (long long)S * 3, cy, ky, oy, false, v);
}

// ToTensor's u8 -> [0, 1]: torch's u8.float() / 255, an IEEE division (not a multiply by 1/255).
YTK_HD float unit_from_u8(int v) {
#ifdef __CUDA_ARCH__
    return __fdiv_rn((float)v, 255.f);
#else
    return (float)v / 255.f;
#endif
}

}  // namespace ytk
