// Host instantiation of yomitoku_b200/csrc/resample_math.h for tests/test_resample_lanczos_host.py: the per-pixel bodies
// of the device resize (csrc/resample_ops.cu) compiled with g++ -ffp-contract=off, so that the test pins the LANCZOS
// and rectangular BILINEAR resize bit for bit against Pillow on the CPU.  The test compiles it into a temporary
// directory; the product never loads it.
#include <vector>

#include "../yomitoku_b200/csrc/resample_math.h"

extern "C" {

// The passes resample_ops.cu runs for a cw x ch -> ow x oh resize (kPassH | kPassV | kPassVFirst bits).
int resample_host_passes(int cw, int ch, int ow, int oh) { return ytk::resample_passes(cw, ch, ow, oh); }

// One source resized to ow x oh with filter f (1 = LANCZOS, 2 = BILINEAR): out = [oh][ow][3] u8 RGB.  order < 0: the
// pass order of resample_passes; 0 / 1: horizontal / vertical pass first when both axes change (to show that the other
// order gives other bytes).
void resample_host_resize(const uint8_t* pages, const ytk::RtSrc* s, int ow, int oh, int f, int order, uint8_t* out) {
    const int cw = s->x1 - s->x0, ch = s->y1 - s->y0;
    int passes = ytk::resample_passes(cw, ch, ow, oh);
    if (order >= 0 && (passes & (ytk::kPassH | ytk::kPassV)) == (ytk::kPassH | ytk::kPassV))
        passes = ytk::kPassH | ytk::kPassV | (order ? ytk::kPassVFirst : 0);
    const int kx = ytk::resample_ksize(cw, ow, f), ky = ytk::resample_ksize(ch, oh, f);
    std::vector<int> cx((size_t)ow * (kx + 2)), cy((size_t)oh * (ky + 2));
    ytk::resample_coeffs(cw, ow, f, cx.data());
    ytk::resample_coeffs(ch, oh, f, cy.data());
    const long long pitch = (long long)s->W * 3;
    const uint8_t* crop = pages + s->page_off + (long long)s->y0 * pitch + (long long)s->x0 * 3;
    const int icols = ytk::resample_inter_cols(cw, ow, passes);
    const long long px = ytk::resample_inter_pixels(cw, ch, ow, oh, passes);
    std::vector<uint8_t> inter((size_t)px * 3 + 3);
    for (long long p = 0; p < px; ++p)
        ytk::resample_first(crop, pitch, passes, cx.data(), kx, cy.data(), ky, icols, (int)(p / icols), (int)(p % icols),
                            inter.data());
    for (int y = 0; y < oh; ++y)
        for (int x = 0; x < ow; ++x)
            ytk::resample_second(crop, pitch, inter.data(), icols, passes, cx.data(), kx, cy.data(), ky, y, x,
                                 out + ((long long)y * ow + x) * 3);
}

}  // extern "C"
