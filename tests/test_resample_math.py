"""CPU: the arithmetic of the RT-DETRv2 input resize (yomitoku_b200/csrc/resample_math.h, the bodies of the two CUDA
kernels in csrc/resample_ops.cu) compiled for the host (oracle/resample_host.cpp) and pinned BIT FOR BIT against
Pillow's Image.resize(..., Image.BILINEAR) - what the reference's T.Resize runs in front of the layout parser, the table
structure recognizer and the cell detector - plus the u8 -> [0, 1] table, the records `rtdetr_sources` makes of the
modules' boxes, and the C record layout.

The same resize runs on the real kernels in tests/test_gpu_rtdetr_u8.py."""
import ctypes

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import build_resample_host
from yomitoku_b200 import _lib
from yomitoku_b200.layout_parser import RTDETR_SRC_DTYPE, rtdetr_sources

# (H, W) -> S: shrinking, growing, both at once, an unchanged axis, extreme aspect ratios, sizes next to S, a 1 x 1
# page and inputs already S x S (Pillow copies them)
CASES = [((1600, 1200), 640), ((1200, 1600), 640), ((37, 523), 960), ((700, 900), 960), ((2000, 3000), 960),
         ((640, 300), 640), ((300, 640), 640), ((5, 7), 640), ((9000, 120), 640), ((961, 959), 960),
         ((1283, 1777), 640), ((1, 1), 640), ((640, 640), 640), ((960, 960), 960)]


@pytest.fixture(scope="module")
def host_lib():
    lib = ctypes.CDLL(build_resample_host.build())
    lib.resample_host_src_size.restype = ctypes.c_int
    return lib


def make_page(H, W, kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    if kind == "gradient":
        y, x = np.mgrid[0:H, 0:W]
        return np.stack([(x * 7 + y) % 256, (y * 5 + 3 * x) % 256, (x * y) % 256], -1).astype(np.uint8)
    return np.full((H, W, 3), (17, 200, 255), np.uint8)


def pil_resize(page_bgr, rect, S):
    x0, y0, x1, y1 = rect
    rgb = np.ascontiguousarray(page_bgr[y0:y1, x0:x1, ::-1])
    return np.asarray(Image.fromarray(rgb).resize((S, S), Image.BILINEAR))


def host_resize(lib, pages, rects, S):
    """pages: BGR arrays; rects: (page index, (x0, y0, x1, y1)).  Returns [n, S, S, 3] RGB from the host build."""
    buf = np.concatenate([p.reshape(-1) for p in pages])
    recs, _ = rtdetr_sources([p.shape for p in pages], rects)
    out = np.full((len(rects), S, S, 3), 77, np.uint8)
    vp = ctypes.c_void_p
    lib.resample_host_bilinear(buf.ctypes.data_as(vp), recs.ctypes.data_as(vp), len(recs), S, out.ctypes.data_as(vp))
    return out


@pytest.mark.parametrize("shape,S", CASES)
@pytest.mark.parametrize("kind", ["random", "gradient", "constant"])
def test_host_resize_equals_pillow(host_lib, shape, S, kind):
    H, W = shape
    page = make_page(H, W, kind)
    got = host_resize(host_lib, [page], [(0, (0, 0, W, H))], S)[0]
    np.testing.assert_array_equal(got, pil_resize(page, (0, 0, W, H), S))


@pytest.mark.parametrize("shape,S", [((701, 7), 640), ((700, 7), 640), ((1001, 10), 640), ((1000, 10), 640),
                                     ((961, 3), 960), ((900, 3), 960), ((1600, 3), 640), ((10001, 100), 64),
                                     ((5, 1000), 64), ((2000, 10), 1500)])
def test_host_resize_pass_order_equals_pillow(host_lib, shape, S):
    """Tall narrow inputs on both sides of the shape at which Pillow runs the vertical pass first."""
    H, W = shape
    page = make_page(H, W, "random", 3)
    got = host_resize(host_lib, [page], [(0, (0, 0, W, H))], S)[0]
    np.testing.assert_array_equal(got, pil_resize(page, (0, 0, W, H), S))


def test_host_resize_of_rectangles_equals_pillow_on_crops(host_lib):
    """Several rectangles of pages of different sizes in one call: each equals Pillow on the numpy crop."""
    pages = [make_page(1200, 900, "random", 1), make_page(700, 1500, "gradient", 2)]
    rects = [(0, (0, 0, 900, 1200)), (0, (13, 40, 611, 1040)), (1, (1000, 5, 1500, 37)), (1, (3, 2, 4, 700)),
             (0, (850, 1190, 900, 1200)), (0, (450, 0, 453, 1200)), (1, (700, 0, 705, 700)), (0, (0, 100, 9, 1100))]
    for S in (640, 960):
        got = host_resize(host_lib, pages, rects, S)
        for i, (p, r) in enumerate(rects):
            np.testing.assert_array_equal(got[i], pil_resize(pages[p], r, S), err_msg="rect %d at %d" % (i, S))


def test_unit_table_equals_torch_to_tensor(host_lib):
    table = np.zeros(256, np.float32)
    host_lib.resample_host_unit_table(table.ctypes.data_as(ctypes.c_void_p))
    ref = torch.arange(256, dtype=torch.uint8).float() / 255
    assert np.array_equal(table.view(np.uint32), ref.numpy().view(np.uint32))
    # the device converts with round-to-nearest-even, as torch's .half() does
    assert np.array_equal(table.astype(np.float16).view(np.uint16), ref.half().numpy().view(np.uint16))


def test_record_layout(host_lib):
    assert ctypes.sizeof(_lib.YtkRtdetrSrc) == 32
    assert host_lib.resample_host_src_size() == 32
    assert RTDETR_SRC_DTYPE.itemsize == 32


def test_rtdetr_sources_follow_numpy_slicing():
    pages = [np.zeros((100, 80, 3), np.uint8), np.zeros((50, 200, 3), np.uint8)]
    shapes = [p.shape for p in pages]
    boxes = [(0, (0, 0, 80, 100)),                # the whole page
             (0, (10, 20, 30, 40)),               # inside
             (1, (150, 10, 400, 90)),             # overhanging right and bottom: clamped
             (1, (5.9, 3.2, 17.7, 49.99)),        # float coordinates: int() truncates
             (0, (-0.5, 0, 10, 10))]              # int(-0.5) == 0: not negative
    recs, sizes = rtdetr_sources(shapes, boxes)
    offs = [0, 100 * 80 * 3]
    for rec, size, (p, box) in zip(recs, sizes, boxes):
        x1, y1, x2, y2 = (int(v) for v in box)
        crop = pages[p][y1:y2, x1:x2]
        assert size == crop.shape[:2]
        assert (rec["page_off"], rec["H"], rec["W"]) == (offs[p], pages[p].shape[0], pages[p].shape[1])
        assert (rec["x0"], rec["y0"]) == (x1, y1)
        assert (rec["y1"] - rec["y0"], rec["x1"] - rec["x0"]) == crop.shape[:2]
    for bad in [(0, (-3, 0, 10, 10)), (0, (0, -1, 10, 10)), (0, (5, 5, 5, 9)), (0, (90, 0, 120, 10)),
                (1, (0, 60, 10, 70)), (1, (10, 10, 3, 20))]:
        assert rtdetr_sources(shapes, [(0, (1, 1, 2, 2)), bad]) is None, bad
