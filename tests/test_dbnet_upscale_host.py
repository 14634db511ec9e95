"""CPU: the detector's resize for pages that grow to the detector input, and the refusals of the op-level
pre-processing entry on such pages.

OpenCV's cv2.resize(INTER_AREA) uses its area tables only when no axis grows.  When some axis grows it resamples BOTH
axes bilinearly with "area-mode" coefficients; per axis, for destination index d, source size s, destination size n:

    inv = n / s;  scale = 1 / inv;  sx = floor(d * scale)
    f = fp32((d + 1) - (sx + 1) * inv);  f = 0 if f <= 0 else f - floor(f)
    if sx >= s - 1: sx, f = s - 1, 0
    value = S[sx] (1 - f) + S[sx + 1] f        (fp32 weights; horizontal pass per row, then vertical)

`up_matrix` restates these tables in float64 as a sparse [n, s] matrix; applied to both axes it is the reference of
preprocess_kernel<AreaUpSampler> (tests/test_gpu_dbnet_upscale.py).  Here it is checked against cv2 itself, and the
trap is pinned: scale = s / n instead of 1 / (n / s) floors to the neighbouring pixel wherever d * s / n is an integer
that 1 / (n / s) rounds below, which on 300x420 -> 640x512 and 700x900 -> 700x1000 moves values by up to 255."""
import ctypes
import math

import cv2
import numpy as np
import pytest
import scipy.sparse as sp

from test_op_entries_host import preprocess_table
from yomitoku_b200 import _lib, build
from yomitoku_b200.data import shortest_edge_size

# (page, detector input): the detector sizes of common small pages, then explicit sizes - an exact 2x, ratio exactly
# 1 on one axis, the two shapes where s / n and 1 / (n / s) floor apart, and two mixed cases (one axis grows, the
# other shrinks: OpenCV samples the shrinking axis bilinearly too)
DETECTOR_SHAPES = [(300, 420), (720, 1280), (827, 1169), (1000, 1000), (1100, 1500), (600, 1500), (1279, 1599),
                   (33, 50), (1, 1), (640, 640), (20, 3000)]
TRAPS = [((300, 420), (640, 512)), ((700, 900), (700, 1000))]
SHAPES = [(hw, shortest_edge_size(*hw, 1280, 1600)) for hw in DETECTOR_SHAPES] + TRAPS + [((100, 800), (96, 1600))]
SHAPE_IDS = ["%dx%d-%dx%d" % (h, w, hn, wn) for (h, w), (hn, wn) in SHAPES]


def up_matrix(ssize, dsize, variant=None):
    """float64 [dsize, ssize] weights of cv2.resize(INTER_AREA) along one axis when some axis grows.  Wrong variants:
    's_over_n' (scale = ssize / dsize), 'linear' (INTER_LINEAR: half-pixel centres)."""
    inv = dsize / ssize
    scale = ssize / dsize if variant == "s_over_n" else 1.0 / inv
    rows, cols, vals = [], [], []
    for d in range(dsize):
        if variant == "linear":
            fx = np.float32((d + 0.5) * scale - 0.5)
            s = math.floor(fx)
            f = np.float32(fx - s)
        else:
            s = math.floor(d * scale)
            f = np.float32((d + 1) - (s + 1) * inv)
            f = np.float32(0) if f <= 0 else np.float32(f - math.floor(f))
        if s < 0:
            s, f = 0, np.float32(0)
        if s >= ssize - 1:
            s, f = ssize - 1, np.float32(0)
        rows.append(d)
        cols.append(s)
        vals.append(float(np.float32(1) - f))
        if f != 0:
            rows.append(d)
            cols.append(s + 1)
            vals.append(float(f))
    return sp.csr_matrix((vals, (rows, cols)), shape=(dsize, ssize))


def up_resize(page, Hn, Wn, variant=None):
    """float64 [Hn, Wn, 3] on the 0..255 scale"""
    Ry, Rx = up_matrix(page.shape[0], Hn, variant), up_matrix(page.shape[1], Wn, variant)
    x = page.astype(np.float64)
    return np.stack([(Rx @ (Ry @ x[:, :, c]).T).T for c in range(3)], -1)


def same_tables(H0, W0, Hn, Wn, variant):
    """True if the variant's tables equal OpenCV's on both axes (then no page can tell them apart)."""
    return all((up_matrix(s, d, variant) != up_matrix(s, d)).nnz == 0 for s, d in ((H0, Hn), (W0, Wn)))


def _random_page(H0, W0):
    return np.random.default_rng(H0 * 31 + W0).integers(0, 256, (H0, W0, 3), dtype=np.uint8)


@pytest.mark.parametrize("hw,size", SHAPES, ids=SHAPE_IDS)
def test_restatement_equals_cv2(hw, size):
    (H0, W0), (Hn, Wn) = hw, size
    assert Hn > H0 or Wn > W0                      # every case is one OpenCV up-scales
    page = _random_page(H0, W0)
    cvr = cv2.resize(page.astype(np.float32), (Wn, Hn), interpolation=cv2.INTER_AREA)
    d = np.abs(up_resize(page, Hn, Wn) - cvr).max()
    print("[upscale] %dx%d -> %dx%d: |float64 tables - cv2| max %.3g" % (H0, W0, Hn, Wn, d))
    assert d <= 1e-4, d


@pytest.mark.parametrize("hw,size", TRAPS, ids=["%dx%d-%dx%d" % (h, w, hn, wn) for (h, w), (hn, wn) in TRAPS])
def test_s_over_n_scale_misses_cv2(hw, size):
    (H0, W0), (Hn, Wn) = hw, size
    page = _random_page(H0, W0)
    cvr = cv2.resize(page.astype(np.float32), (Wn, Hn), interpolation=cv2.INTER_AREA)
    d = np.abs(up_resize(page, Hn, Wn, "s_over_n") - cvr).max()
    print("[upscale] %dx%d -> %dx%d: scale = s / n is off by %.0f" % (H0, W0, Hn, Wn, d))
    assert d >= 100, d


# ======================================================================================================== op entry
P = 0x10000          # 16-byte aligned stand-in for a device pointer: never dereferenced on a refusal


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.lib()


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(src=None), b"ytk_op_dbnet_preprocess_table_u8: null argument"), (dict(canvas=None), b"null argument"),
    (dict(n=0), b"0 page records"), (dict(n=65536), b"65536 page records"), (dict(table=False), b"page records"),
    (dict(H0=0), b"page 0 (at 0, 0x1200"), (dict(W0=-1), b"page 0 (at 0, 900x-1"),
    (dict(Hn=0), b"non-positive input size 0x1600"), (dict(Wn=-32), b"non-positive input size 1184x-32"),
    (dict(canvas=P + 8), b"canvas_dev must be 16-byte aligned"),
])
def test_preprocess_table_up_refusals(lib, kwargs, fragment):
    """The pre-processing entry on pages that grow to the detector input (900x1200 -> 1184x1600)."""
    before = lib.ytk_launch_count()
    status = preprocess_table(lib, **dict(dict(H0=900, W0=1200), **kwargs))
    assert status != 0
    msg = lib.ytk_last_error()
    assert fragment in msg, msg
    assert lib.ytk_launch_count() == before
