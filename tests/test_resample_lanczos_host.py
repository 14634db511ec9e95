"""CPU: the generalised device resize (yomitoku_b200/csrc/resample_math.h: per-source output sizes, a LANCZOS table, no
pass for an unchanged axis) compiled for the host (tests/resample_pages_host.cpp) and pinned BIT FOR BIT against Pillow 12.2
`Image.resize((w, h), LANCZOS)` - what the reference's searchable PDF runs on each page - and BILINEAR on rectangular
outputs; the pass order on both sides of its boundary; and the record checks of the C entry ytk_resize_pages_u8.

The same resize runs on the real kernels in tests/test_gpu_searchable_pdf.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
from PIL import Image

from yomitoku_b200 import _lib, build
from yomitoku_b200.searchable_pdf import BILINEAR, LANCZOS, RESIZE_PAGE_DTYPE, target_size

VP = ctypes.c_void_p
FILTERS = {LANCZOS: Image.LANCZOS, BILINEAR: Image.BILINEAR}


class Src(ctypes.Structure):
    _fields_ = [("page_off", ctypes.c_longlong)] + [(n, ctypes.c_int) for n in ("H", "W", "x0", "y0", "x1", "y1")]


HARNESS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "resample_pages_host.cpp")


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("resample") / "libresample_pages_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", HARNESS,
                    "-o", so], check=True)
    return ctypes.CDLL(so)


def make_page(H, W, seed=0):
    rng = np.random.default_rng(seed)
    page = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    y, x = np.mgrid[0:H, 0:W]
    page[: H // 2] = np.stack([(x * 7 + y) % 256, (y * 5 + 3 * x) % 256, (x * y) % 256], -1)[: H // 2]
    return page


def pil(page_bgr, w, h, f):
    return np.asarray(Image.fromarray(np.ascontiguousarray(page_bgr[:, :, ::-1])).resize((w, h), FILTERS[f]))


def host(lib, page, w, h, f, order=-1):
    H, W = page.shape[:2]
    out = np.zeros((h, w, 3), np.uint8)
    lib.resample_host_resize(page.ctypes.data_as(VP), ctypes.byref(Src(0, H, W, 0, 0, W, H)), w, h, f, order,
                             out.ctypes.data_as(VP))
    return out


def _preset_cases():
    out = []
    for H, W in ((3508, 2480), (1600, 1200)):
        for q in ("middle", "low"):
            out.append(((H, W), target_size(W, H, q)))
    return out


# (H, W) -> (w, h): the presets of A4 at 300 dpi and of 1200 x 1600, odd sizes, scales near 1 and near 0.3, 1-pixel
# outputs, one axis growing while the other shrinks, unchanged axes
SHAPES = _preset_cases() + [
    ((333, 517), (511, 331)), ((1001, 999), (997, 1003)), ((400, 300), (121, 91)), ((97, 1003), (31, 301)),
    ((50, 60), (1, 1)), ((50, 60), (60, 1)), ((50, 60), (1, 50)), ((1, 1), (7, 5)), ((120, 80), (240, 30)),
    ((80, 120), (40, 300)), ((300, 200), (200, 150)), ((300, 200), (130, 300)), ((300, 200), (200, 300)),
    ((17, 23), (17, 23)), ((2, 900), (450, 1))]


@pytest.mark.parametrize("shape,size", SHAPES)
def test_lanczos_equals_pillow(host_lib, shape, size):
    page = make_page(*shape)
    np.testing.assert_array_equal(host(host_lib, page, *size, LANCZOS), pil(page, *size, LANCZOS))


@pytest.mark.parametrize("shape,size", [((333, 517), (511, 331)), ((97, 1003), (31, 301)), ((120, 80), (240, 30)),
                                        ((300, 200), (130, 300)), ((50, 60), (1, 1)), ((1600, 1200), (640, 480))])
def test_bilinear_rectangular_equals_pillow(host_lib, shape, size):
    page = make_page(*shape, seed=1)
    np.testing.assert_array_equal(host(host_lib, page, *size, BILINEAR), pil(page, *size, BILINEAR))


# tall-narrow pages around 100 rows per column, with outputs that grow or shrink the width, and wide-short pages (which
# keep the horizontal pass first): (H, W, w, h, vertical pass first)
ORDER_CASES = [(701, 7, 3, 300, True), (700, 7, 3, 300, False), (701, 7, 50, 300, True), (700, 7, 50, 300, False),
               (1001, 10, 500, 999, True), (1000, 10, 500, 999, False), (2001, 20, 1, 30, True),
               (2001, 20, 15, 2001, False), (2001, 20, 15, 2002, False), (7, 701, 300, 3, False),
               (10, 1001, 999, 5, False), (300, 2, 1, 299, True), (199, 2, 1, 100, False)]


@pytest.mark.parametrize("H,W,w,h,vfirst", ORDER_CASES)
@pytest.mark.parametrize("f", [LANCZOS, BILINEAR])
def test_pass_order_equals_pillow(host_lib, H, W, w, h, vfirst, f):
    """The rule picks the order Pillow takes; where both axes change, the other order gives other bytes."""
    page = make_page(H, W, seed=3)
    passes = host_lib.resample_host_passes(W, H, w, h)
    assert bool(passes & 4) == vfirst
    ref = pil(page, w, h, f)
    np.testing.assert_array_equal(host(host_lib, page, w, h, f), ref)
    if passes & 3 == 3:
        assert not np.array_equal(host(host_lib, page, w, h, f, order=0 if vfirst else 1), ref)


def test_square_rule_is_unchanged(host_lib):
    """For out_w == out_h == S the rule is the one the RT-DETRv2 resize was measured with: ch > S and ch > 100 cw."""
    for cw, ch, S in [(7, 701, 640), (7, 700, 640), (10, 1001, 640), (3, 961, 960), (3, 900, 960), (100, 10001, 64),
                      (1000, 5, 64), (10, 2000, 1500), (1, 640, 640), (1, 641, 640)]:
        want = ch > S and ch > 100 * cw
        assert bool(host_lib.resample_host_passes(cw, ch, S, S) & 4) == want, (cw, ch, S)


def test_unchanged_page_is_a_channel_swap(host_lib):
    page = make_page(31, 17)
    assert host_lib.resample_host_passes(17, 31, 17, 31) == 0
    np.testing.assert_array_equal(host(host_lib, page, 17, 31, LANCZOS), page[:, :, ::-1])


def test_target_size_is_the_reference_expression():
    for W, H in [(2480, 3508), (1200, 1600), (3508, 2480), (2000, 10), (1999, 2001), (4001, 1)]:
        for q, m in (("middle", 2000), ("low", 1500)):
            if max(W, H) > m:
                s = m / max(W, H)
                want = (int(W * s), int(H * s))
            else:
                want = (W, H)
            if min(want) < 1:
                with pytest.raises(ValueError):
                    target_size(W, H, q)
            else:
                assert target_size(W, H, q) == want
        assert target_size(W, H, "high") == (W, H)
    assert target_size(2480, 3508, "middle") == (1413, 2000)
    with pytest.raises(ValueError):
        target_size(10, 10, "best")


# ---------------------------------------------------------------------------------------- ytk_resize_pages_u8 checks
P = 0x10000  # stand-in device pointer: never dereferenced on the refusal paths


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.lib()


def _recs(*rows):
    r = np.zeros(len(rows), RESIZE_PAGE_DTYPE)
    for i, row in enumerate(rows):
        r[i] = row
    return r


GOOD = [(0, 100, 80, 40, 50, 0), (100 * 80 * 3, 60, 90, 90, 60, 40 * 50 * 3)]
PAGES_BYTES = 100 * 80 * 3 + 60 * 90 * 3
OUT_BYTES = 40 * 50 * 3 + 90 * 60 * 3


@pytest.mark.parametrize("rows,filt,pages_bytes,out_bytes,fragment", [
    ([(0, 100, 80, 40, 50, 0), (100 * 80 * 3 + 1, 60, 90, 90, 60, 6000)], LANCZOS, PAGES_BYTES, OUT_BYTES,
     b"source 1 (page at 24001, 60x90"),
    ([(-3, 100, 80, 40, 50, 0)], LANCZOS, PAGES_BYTES, OUT_BYTES, b"source 0 (page at -3"),
    ([(0, 0, 80, 40, 50, 0)], LANCZOS, PAGES_BYTES, OUT_BYTES, b"source 0 (page at 0, 0x80"),
    ([(0, 100, 80, 0, 50, 0)], LANCZOS, PAGES_BYTES, OUT_BYTES, b"output size 0x50"),
    ([(0, 100, 80, 40, -1, 0)], LANCZOS, PAGES_BYTES, OUT_BYTES, b"output size 40x-1"),
    ([(0, 100, 80, 40, 50, 1)], LANCZOS, PAGES_BYTES, 6000, b"page 0: output of 6000 bytes at 1 lies outside"),
    ([(0, 100, 80, 40, 50, -6)], LANCZOS, PAGES_BYTES, OUT_BYTES, b"at -6 lies outside"),
    ([GOOD[0], (100 * 80 * 3, 60, 90, 90, 60, 5999)], LANCZOS, PAGES_BYTES, OUT_BYTES,
     b"the outputs of pages 0 and 1 overlap"),
    ([GOOD[1], GOOD[0], (0, 100, 80, 1, 1, 40 * 50 * 3 + 90 * 60 * 3 - 3)], LANCZOS, PAGES_BYTES, OUT_BYTES,
     b"the outputs of pages 0 and 2 overlap"),
    (GOOD, 3, PAGES_BYTES, OUT_BYTES, b"unknown filter 3"),
    (GOOD, 0, PAGES_BYTES, OUT_BYTES, b"unknown filter 0"),
])
def test_resize_pages_refusals(lib, rows, filt, pages_bytes, out_bytes, fragment):
    recs = _recs(*rows)
    before = lib.ytk_launch_count()
    st = lib.ytk_resize_pages_u8(P, pages_bytes, recs.ctypes.data, len(recs), filt, P, 1 << 30, P, out_bytes, None)
    assert st != 0
    msg = lib.ytk_last_error()
    assert fragment in msg, msg
    assert lib.ytk_launch_count() == before


def test_resize_pages_argument_refusals(lib):
    recs = _recs(*GOOD)
    for args, fragment in [((None, PAGES_BYTES, recs.ctypes.data, 2, LANCZOS, P, 1 << 30, P, OUT_BYTES),
                            b"null argument"),
                           ((P, PAGES_BYTES, recs.ctypes.data, 0, LANCZOS, P, 1 << 30, P, OUT_BYTES), b"0 pages"),
                           ((P, PAGES_BYTES, recs.ctypes.data, 2, LANCZOS, P, 16, P, OUT_BYTES),
                            b"scratch_dev holds 16 bytes")]:
        assert lib.ytk_resize_pages_u8(*args, None) != 0
        assert fragment in lib.ytk_last_error(), lib.ytk_last_error()
    assert lib.ytk_resize_pages_scratch_bytes(recs.ctypes.data, 2, LANCZOS) > 0
    assert lib.ytk_resize_pages_scratch_bytes(recs.ctypes.data, 2, 7) == -1
    # an unchanged page needs no coefficient table and no intermediate: plans only
    same = _recs((0, 100, 80, 80, 100, 0))
    assert lib.ytk_resize_pages_scratch_bytes(same.ctypes.data, 1, LANCZOS) == 96
