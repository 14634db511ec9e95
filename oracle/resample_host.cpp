// TEST INFRASTRUCTURE ONLY - host instantiation of yomitoku_b200/csrc/resample_math.h.
//
// The product's device-side input resize of the RT-DETRv2 models (csrc/resample_ops.cu) is two thin CUDA kernels around
// the per-pixel bodies in resample_math.h.  This file compiles the very same bodies with g++ (no CUDA) into
// oracle/_build/libresample_host.so so that tests/test_resample_math.py can pin them, on the CPU and bit for bit,
// against Pillow's Image.resize(..., Image.BILINEAR), which the reference's T.Resize calls.
// Only tests/ loads this library; the product never does (no CPU fallback on the hot path).
//
// Build: g++ -O2 -ffp-contract=off -shared -fPIC oracle/resample_host.cpp -o oracle/_build/libresample_host.so
//        (oracle/build_resample_host.py, also run by __graft_entry__.build()).
#include <vector>

#include "../yomitoku_b200/csrc/resample_math.h"

extern "C" {

int resample_host_src_size(void) { return (int)sizeof(ytk::RtSrc); }

// Both passes for n sources: out = [n][S][S][3] u8 RGB, as ytk_op_resize_bilinear_u8 writes it.
void resample_host_bilinear(const uint8_t* pages, const ytk::RtSrc* srcs, int n, int S, uint8_t* out) {
    for (int i = 0; i < n; ++i) {
        const ytk::RtSrc& s = srcs[i];
        const int cw = s.x1 - s.x0, ch = s.y1 - s.y0;
        const int kx = ytk::bilinear_ksize(cw, S), ky = ytk::bilinear_ksize(ch, S);
        std::vector<int> cx((size_t)S * (kx + 2)), cy((size_t)S * (ky + 2));
        ytk::bilinear_coeffs(cw, S, cx.data());
        ytk::bilinear_coeffs(ch, S, cy.data());
        const int cols = ytk::resample_vertical_first(cw, ch, S) ? cw : S;
        const long long px = ytk::resample_inter_pixels(cw, ch, S);
        std::vector<uint8_t> inter((size_t)px * 3);
        for (long long p = 0; p < px; ++p)
            ytk::resample_first(pages, s, cx.data(), kx, cy.data(), ky, S, (int)(p / cols), (int)(p % cols), inter.data());
        uint8_t* o = out + (long long)i * S * S * 3;
        for (int y = 0; y < S; ++y)
            for (int x = 0; x < S; ++x)
                ytk::resample_second(inter.data(), cw, ch, cx.data(), kx, cy.data(), ky, S, y, x, o + ((long long)y * S + x) * 3);
    }
}

// The 256 values ToTensor makes of a u8 sample (before the device's fp32 -> 16-bit operand conversion).
void resample_host_unit_table(float* out) {
    for (int v = 0; v < 256; ++v) out[v] = ytk::unit_from_u8(v);
}

}  // extern "C"
