// Per-pixel arithmetic of the device resize of u8 BGR pages (csrc/resample_ops.cu), written ONCE for host and device:
// resample_ops.cu wraps these bodies in CUDA kernels, oracle/resample_host.cpp instantiates the very same functions with
// g++ so that the `-m "not gpu"` tests can pin them bit for bit against Pillow on the CPU.
//
// What is restated: Image.fromarray(rgb).resize((out_w, out_h), f) for an 8-bit RGB image and f = Image.BILINEAR (the
// reference's T.Resize in front of the layout parser, the table structure recognizer and the cell detector, out_w =
// out_h = S) or Image.LANCZOS (the page images of the searchable PDF).  Pillow's ImagingResample, no reducing_gap, box =
// the whole image:
//   * per axis, coefficients in double (precompute_coeffs): scale = in / out, filterscale = max(scale, 1),
//     support = filter support * filterscale, ksize = 2 * ceil(support) + 1, the filter evaluated at
//     (x + xmin - center + 0.5) * (1 / filterscale), normalised by the sum, then rounded to 22 fractional bits
//     (normalize_coeffs_8bpc).  The tables are built on the host only (libm's sin for LANCZOS, as Pillow calls it);
//   * two separable passes, each sample an int32 accumulation 2^21 + sum(u8 * k) clipped to [0, 255] after >> 22; the
//     first pass writes a u8 intermediate that the second reads.  The horizontal pass comes first, except for a tall,
//     narrow input that shrinks vertically (resample_vertical_first: measured against Pillow 12.2, which picks the
//     order by the input's shape);
//   * as in Pillow, an axis whose size does not change has no pass: one pass reads the page directly, and a source
//     whose size does not change at all is a BGR -> RGB copy.
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

// The filters, numbered as Pillow numbers them (Image.LANCZOS = 1, Image.BILINEAR = 2).
enum ResampleFilter : int { kFilterLanczos = 1, kFilterBilinear = 2 };

YTK_HD bool resample_filter_known(int f) { return f == kFilterLanczos || f == kFilterBilinear; }

YTK_HD double bilinear_filter(double x) {
    if (x < 0.0) x = -x;
    return x < 1.0 ? 1.0 - x : 0.0;
}

YTK_HD double sinc_filter(double x) {
    if (x == 0.0) return 1.0;
    x = x * M_PI;
    return sin(x) / x;
}

// Pillow's truncated sinc: sinc(x) * sinc(x / 3) on [-3, 3).
YTK_HD double lanczos_filter(double x) { return -3.0 <= x && x < 3.0 ? sinc_filter(x) * sinc_filter(x / 3) : 0.0; }

YTK_HD double resample_filter(int f, double x) { return f == kFilterLanczos ? lanczos_filter(x) : bilinear_filter(x); }

YTK_HD double resample_support(int f) { return f == kFilterLanczos ? 3.0 : 1.0; }

// Taps per output index of an in -> out axis.
YTK_HD int resample_ksize(int in, int out, int f) {
    const double scale = (double)in / (double)out;
    const double support = resample_support(f) * (scale < 1.0 ? 1.0 : scale);
    return (int)ceil(support) * 2 + 1;
}

// Coefficient table of an in -> out axis: for output index i, tab[i * (ksize + 2)] = first source index, tab[... + 1]
// = number of taps used, then ksize fixed-point weights (zero beyond the used taps).
YTK_HD void resample_coeffs(int in, int out, int f, int* tab) {
    const double scale = (double)in / (double)out;
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = resample_support(f) * filterscale;
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
        for (int x = 0; x < xmax; ++x) ww += resample_filter(f, (x + xmin - center + 0.5) * ss);
        int* t = tab + (long long)i * (ksize + 2);
        t[0] = xmin;
        t[1] = xmax;
        for (int x = 0; x < ksize; ++x) {
            double k = 0.0;
            if (x < xmax) {
                k = resample_filter(f, (x + xmin - center + 0.5) * ss);
                if (ww != 0.0) k /= ww;
            }
            const double v = k * (double)(1 << kResampleBits);
            t[2 + x] = k < 0.0 ? (int)(-0.5 + v) : (int)(0.5 + v);
        }
    }
}

YTK_HD uint8_t resample_clip(int acc) {
    acc >>= kResampleBits;
    return (uint8_t)(acc < 0 ? 0 : (acc > 255 ? 255 : acc));
}

// Pillow 12 runs the vertical pass first for a tall, narrow input that shrinks vertically (more than 100 rows per
// column); otherwise the horizontal pass comes first.  The order changes the bytes: the intermediate is rounded to u8.
// Measured against Pillow 12.2 on rectangular outputs too: the output width plays no part, and wide, short inputs keep
// the horizontal pass first (tests/test_resample_lanczos_host.py pins both sides of the boundary).
YTK_HD bool resample_vertical_first(int cw, int ch, int oh) { return ch > oh && (long long)ch > 100LL * cw; }

// The passes of a cw x ch -> ow x oh resize: which axes change, and whether the vertical pass comes first.
enum : int { kPassH = 1, kPassV = 2, kPassVFirst = 4 };

YTK_HD int resample_passes(int cw, int ch, int ow, int oh) {
    const int p = (cw != ow ? kPassH : 0) | (ch != oh ? kPassV : 0);
    return p == (kPassH | kPassV) && resample_vertical_first(cw, ch, oh) ? p | kPassVFirst : p;
}

// Columns of the u8 RGB intermediate of a two-pass resize ([ch][ow] after a horizontal first pass, [oh][cw] after a
// vertical one), 0 when there is no intermediate.
YTK_HD int resample_inter_cols(int cw, int ow, int passes) {
    return (passes & (kPassH | kPassV)) != (kPassH | kPassV) ? 0 : (passes & kPassVFirst) ? cw : ow;
}

YTK_HD long long resample_inter_pixels(int cw, int ch, int ow, int oh, int passes) {
    return (passes & (kPassH | kPassV)) != (kPassH | kPassV) ? 0
           : (passes & kPassVFirst)                           ? (long long)oh * cw
                                                              : (long long)ch * ow;
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

// First pass of a two-pass resize, intermediate pixel (r, c): reads the BGR crop (rows `pitch` bytes apart), writes RGB
// into inter ([.][icols]).  cx / cy: coefficient tables of the cw -> ow and ch -> oh axes, kx / ky their ksize.
YTK_HD void resample_first(const uint8_t* crop, long long pitch, int passes, const int* cx, int kx, const int* cy, int ky,
                           int icols, int r, int c, uint8_t* inter) {
    uint8_t* o = inter + ((long long)r * icols + c) * 3;
    if (passes & kPassVFirst)
        resample_taps(crop + (long long)c * 3, pitch, cy, ky, r, true, o);
    else
        resample_taps(crop + (long long)r * pitch, 3, cx, kx, c, true, o);
}

// Output pixel (oy, ox) as RGB: the second pass over the intermediate of a two-pass resize, the only pass over the crop
// of a one-pass resize, or the crop's pixel when no axis changes.
YTK_HD void resample_second(const uint8_t* crop, long long pitch, const uint8_t* inter, int icols, int passes,
                            const int* cx, int kx, const int* cy, int ky, int oy, int ox, uint8_t* v) {
    switch (passes) {
        case kPassH | kPassV | kPassVFirst:
            resample_taps(inter + (long long)oy * icols * 3, 3, cx, kx, ox, false, v);
            break;
        case kPassH | kPassV:
            resample_taps(inter + (long long)ox * 3, (long long)icols * 3, cy, ky, oy, false, v);
            break;
        case kPassH:
            resample_taps(crop + (long long)oy * pitch, 3, cx, kx, ox, true, v);
            break;
        case kPassV:
            resample_taps(crop + (long long)ox * 3, pitch, cy, ky, oy, true, v);
            break;
        default: {
            const uint8_t* p = crop + (long long)oy * pitch + (long long)ox * 3;
            v[0] = p[2];
            v[1] = p[1];
            v[2] = p[0];
        }
    }
}

// The BILINEAR resize to S x S with both passes always run, in the form oracle/resample_host.cpp instantiates for
// tests/test_resample_math.py.  An unchanged axis has the identity table ([1, 0] at every index), so running its pass
// gives the bytes of skipping it, which the device does.
YTK_HD int bilinear_ksize(int in, int out) { return resample_ksize(in, out, kFilterBilinear); }

YTK_HD void bilinear_coeffs(int in, int out, int* tab) { resample_coeffs(in, out, kFilterBilinear, tab); }

YTK_HD int square_passes(int cw, int ch, int S) {
    return kPassH | kPassV | (resample_vertical_first(cw, ch, S) ? kPassVFirst : 0);
}

YTK_HD long long resample_inter_pixels(int cw, int ch, int S) {
    return resample_inter_pixels(cw, ch, S, S, square_passes(cw, ch, S));
}

YTK_HD void resample_first(const uint8_t* pages, const RtSrc& s, const int* cx, int kx, const int* cy, int ky, int S, int r,
                           int c, uint8_t* inter) {
    const int cw = s.x1 - s.x0, ch = s.y1 - s.y0, passes = square_passes(cw, ch, S);
    resample_first(pages + s.page_off + ((long long)s.y0 * s.W + s.x0) * 3, (long long)s.W * 3, passes, cx, kx, cy, ky,
                   resample_inter_cols(cw, S, passes), r, c, inter);
}

YTK_HD void resample_second(const uint8_t* inter, int cw, int ch, const int* cx, int kx, const int* cy, int ky, int S,
                            int oy, int ox, uint8_t* v) {
    const int passes = square_passes(cw, ch, S);
    resample_second(nullptr, 0, inter, resample_inter_cols(cw, S, passes), passes, cx, kx, cy, ky, oy, ox, v);
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
