"""GPU: op-level parity of the DBNet detector's own kernels through the C ABI against float64 references on the operands
the kernel reads (fp16-rounded activations and packed weights, fp32 where the kernel reads fp32).  u = 2^-24 is the fp32
unit roundoff; rounding a value y to fp16 costs at most 2^-11 |y| + 2^-25.

  pre-processing  ytk_op_dbnet_preprocess_u8 (preprocess_kernel) vs OpenCV's INTER_AREA tables (computeResizeAreaTab
                  with its 1e-3 sliver rule) applied in float64 as two separable matrices, / 255, mean / std by position.
                  The device value must be fp16(r) for some r within e of the reference: equal to fp16(reference)
                  except where the reference lies within e of a rounding boundary of fp16.  e = 2 ((nx + ny + 4) u / 0.224
                  + 2 u (|ref| + 3)): the kernel sums at most nx x ny taps in two fp32 passes (weights rounded to fp32,
                  values <= 255, weights summing to <= 1) and divides by std >= 0.224 in double with fp32 mean / std.
                  The reference itself equals cv2.resize(page.astype(float32), INTER_AREA) within 1e-4 on the 0..255 scale.
  stem            ytk_op_dbnet_stem_f16 (stem plan of gemm_tc_kernel) vs F.conv2d(stride 2, padding 3) + bias, ReLU:
                  |d| <= 2^-11 |ref| + 2^-25 + 2 * 148 u (sum |x| |w| + |b|): fp16 output rounding plus fp32 accumulation
                  of 147 products and the bias (the K = 448 GEMM's padding products are exact zeros), at 2 u per add
                  for the tensor cores' accumulation.
  max-pool        ytk_op_maxpool3x3s2_f16 (maxpool3x3s2_kernel) is bitwise equal to max_pool2d(3, 2, 1).
  upsampling      ytk_op_upsample_bilinear_f16 (upsample_bilinear_kernel) vs float64 bilinear with PyTorch's source index
                  (d + 0.5) s - 0.5 clamped at 0: |d| <= 2^-11 |want| + 2^-25 + (16 max(Hs, Ws) + 8) u max|src|
                  (+ 2 u |dst| when accumulating).  The kernel forms the source coordinate in fp32 (about 4 max(Hs, Ws)
                  u of error per axis), which moves the result by at most that times the difference of two neighbours
                  (2 max|src|) per axis; the fp32 blend adds a few u max|src|; the fp16 sum rounds once.
  scale fusion    ytk_op_asf_f16 (asf_pool / asf_gate / asf_cmean / asf_apply) vs ScaleChannelSpatialAttention in float64,
                  checked at the channel gate g, the channel-mean map m and the rescaled fuse; m and fuse against the
                  device's own fp32 gate, which their kernels read.  The bounds propagate first-order fp32 error through
                  the formula, and allow twice that: a sum of L terms costs L u sum |terms|; a sigmoid scales an
                  argument error e by its largest slope within e of the argument, S(x, e); __expf / expf cost
                  (2 + 1.16 |x|) ulp of e^x, i.e. E(x) = (2 + 1.16 |x|) 2^-25 + 2 u after the sigmoid:
                    e_mean  = L u mean|a|, L = ceil(ceil(HW / 64) / 32) + 32 + 64 + 1 (lane, pixel-lane, chunk sums)
                    e_g     = S e_gl + E(gl), e_gl = |W2| (|W1| e_mean + 65 u |W1| |mean|) + 17 u |W2| |hid|
                    e_m     = 12 u mean_c|a| + 65 u mean_c g + 2 u |m|
                    e_score = S e_part + E(part), e_part = |att| (e_s + 2 u |z|) + 64 u |att| |z|,
                              e_s = S e_sarg + E(sarg), e_sarg = |sp1| |sp3| (e_m + 9 u |m|)
                  fuse: |d| <= 2 |fuse| e_score + 2^-11 |want| + 2^-25.  A common offset of 100 on `a` stresses the
                  fp32 sums; there the spatial branch and the scores saturate, so the wrong spatial kernel and the
                  swapped groups are checked on the other cases.
  fused head      ytk_op_dbnet_head_f32 (EPI_CONVT_FINAL epilogue of gemm_tc_kernel) vs float64
                  relu(conv_transpose2d(x, w1) + b1), then sigmoid(conv_transpose2d(., w2) + b2), the intermediate
                  unrounded as in the epilogue: |d| <= 2 (S e_logit + E(logit)) + u, e_logit = |w2| e_h + 128 u |w2| |h|,
                  e_h = 130 u (|x| |w1| + |b1|) (64 products and the bias at 2 u per add).

Every output buffer is larger than the output and filled with NaN or 7.0; whatever lies outside the output must come
back unchanged.  Every group also checks a plausible wrong variant of its reference - mean / std applied to true RGB and
area weights renormalised to sum 1 (the sliver rule ignored); a one-pixel shift of the stem, its kh / kw swapped, R and B
swapped; a zero-padded max-pool; align_corners=True; the channel mean without sigmoid(g), a flipped spatial kernel,
score group i applied to group 3 - i; either 2x2 sub-block of the head transposed and its first ReLU left out - which the
kernel must miss by at least 10x the tolerance, or fail its equality check.
"""
import ctypes
import math

import cv2
import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn.functional as F

from oracle import pipeline as opipe
from oracle import weights
from yomitoku_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENT = 7.0          # sentinel of output elements the kernel must not write
U = 2.0 ** -24      # fp32 unit roundoff
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _ratio(got, want, tol):
    """max |got - want| / tol over the elements (<= 1: inside the tolerance)."""
    return ((got - want).abs() / tol).max().item()


def _E(x):
    """error of a sigmoid evaluated through __expf / expf in fp32: (2 + 1.16 |x|) ulp of e^x, / 4, plus the add and
    the division"""
    return (2 + 1.16 * x.abs()) * 2.0 ** -25 + 2 * U


def _dsig(x, e):
    """max of sigmoid' over [x - e, x + e]: how far an argument error e can move a sigmoid"""
    s = torch.sigmoid((x.abs() - e).clamp(min=0))
    return s * (1 - s)


def _fp(t):
    return ctypes.c_void_p(t.data_ptr())


# ======================================================================================================== pre-processing
def _area_matrix(ssize, dsize, renormalise=False):
    """float64 [dsize, ssize]: OpenCV's computeResizeAreaTab for scale = ssize / dsize >= 1 as a sparse matrix.  A
    partial source cell is dropped when it covers 1e-3 or less, so a row of weights may sum to slightly less than 1;
    renormalise=True is the wrong variant that rescales every row to sum 1."""
    scale = ssize / dsize
    rows, cols, vals = [], [], []
    for d in range(dsize):
        fs1 = d * scale
        fs2 = fs1 + scale
        cell = min(scale, ssize - fs1)
        s1, s2 = math.ceil(fs1), math.floor(fs2)
        s2 = min(s2, ssize - 1)
        s1 = min(s1, s2)
        taps = []
        if s1 - fs1 > 1e-3:
            taps.append((s1 - 1, (s1 - fs1) / cell))
        taps += [(s, 1.0 / cell) for s in range(s1, s2)]
        if fs2 - s2 > 1e-3:
            taps.append((s2, min(min(fs2 - s2, 1.0), cell) / cell))
        tot = sum(w for _, w in taps) if renormalise else 1.0
        for s, w in taps:
            rows.append(d)
            cols.append(s)
            vals.append(w / tot)
    return sp.csr_matrix((vals, (rows, cols)), shape=(dsize, ssize))


def _area_resize(page, Hn, Wn, renormalise=False):
    """float64 [Hn, Wn, 3] on the 0..255 scale"""
    Ry, Rx = _area_matrix(page.shape[0], Hn, renormalise), _area_matrix(page.shape[1], Wn, renormalise)
    x = page.astype(np.float64)
    return np.stack([(Rx @ (Ry @ x[:, :, c]).T).T for c in range(3)], -1)


def _normalise(v, true_rgb=False):
    """B,G,R planes / 255 with the RGB mean / std applied by position (the reference's double flip); true_rgb is the
    wrong variant that applies them to the channels they were measured on."""
    idx = [2, 1, 0] if true_rgb else [0, 1, 2]
    return np.stack([(v[..., c] / 255.0 - MEAN[idx[c]]) / STD[idx[c]] for c in range(3)], -1)


def _page(kind, H, W, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    if kind == "bright":
        return np.full((H, W, 3), 255, dtype=np.uint8)
    yy, xx = np.mgrid[0:H, 0:W]
    base = (xx * 255.0 / W + yy * 96.0 / H)
    return np.stack([(base + 40 * c) % 256 for c in range(3)], -1).astype(np.uint8)


def _fp16_match(got, ref, e):
    """got is fp16(r) for some r within e of ref: fp16(ref - e) <= got <= fp16(ref + e) (rounding is monotonic).  Away
    from the rounding midpoints both ends round alike and only got == fp16(ref) passes.  Returns (ok mask, count of
    values other than fp16(ref))."""
    lo, hi = (ref - e).astype(np.float16), (ref + e).astype(np.float16)
    ok = (got >= lo) & (got <= hi)
    return ok, int((ok & (got != ref.astype(np.float16))).sum())


PREP_PAGES = [(1200, 1600), (2560, 3200), (1755, 2481), (3508, 2480), (1300, 1301), (4000, 900), (1280, 1600),
              (1281, 1601)]
# (page size, input size or None for detector_input_size, contents: one page each)
PREP_CASES = [(hw, None, ("random",)) for hw in PREP_PAGES[:4]] + [
    ((1300, 1301), None, ("random", "gradient", "bright")),   # 1301 -> 1280: sliver rows on both axes
    ((4000, 900), None, ("gradient",)),                        # the 1600 limit binds: 1600 x 352
    ((1280, 1600), None, ("random",)),                         # ratio exactly 1 on both axes
    ((1281, 1601), None, ("bright", "random", "gradient")),    # 1601 -> 1568
    ((1755, 2481), None, ("bright",)),                         # 2481 -> 1600
    ((1300, 1600), (1280, 1600), ("gradient", "bright")),      # ratio exactly 1 on one axis
    ((2560, 3200), None, ("gradient", "bright", "random")),    # integer ratio 2
]


@pytest.mark.parametrize("hw,size,kinds", PREP_CASES, ids=["%dx%d-%s" % (h, w, "-".join(k)) for (h, w), _, k in
                                                         PREP_CASES])
def test_preprocess_vs_float64(hw, size, kinds):
    H0, W0 = hw
    Hn, Wn = size if size else opipe.detector_input_size(H0, W0)
    n = len(kinds)
    pages = np.stack([_page(k, H0, W0, seed=H0 * 7 + W0 + i) for i, k in enumerate(kinds)])
    # one canvas more than the call writes, everything NaN: the border ring and channels 3..7 must come back 0
    canvas = torch.full((n + 1, Hn + 6, Wn + 8, 8), float("nan"), dtype=torch.float16, device=DEV)
    src = torch.from_numpy(pages).to(DEV)
    _lib.check(_lib.lib().ytk_op_dbnet_preprocess_u8(_fp(src), n, H0, W0, Hn, Wn, _fp(canvas), None))
    torch.cuda.synchronize()
    out = canvas.cpu().numpy()
    assert np.isnan(out[n]).all()                                 # nothing past the n canvases
    inner = np.zeros(out.shape[:3], dtype=bool)
    inner[:, 3:3 + Hn, 3:3 + Wn] = True
    assert (out[:n][~inner[:n]] == 0).all()                       # exactly zero border ring
    assert (out[:n, :, :, 3:] == 0).all()                         # exactly zero channels 3..7
    got = out[:n, 3:3 + Hn, 3:3 + Wn, :3]
    nx = math.ceil(W0 / Wn) + 1
    ny = math.ceil(H0 / Hn) + 1
    n_nb, worst_cv, r_rgb, sliver_miss, sliver_rows = 0, 0.0, float("inf"), 0, 0
    for i in range(n):
        area = _area_resize(pages[i], Hn, Wn)
        cvr = cv2.resize(pages[i].astype(np.float32), (Wn, Hn), interpolation=cv2.INTER_AREA)
        worst_cv = max(worst_cv, float(np.abs(area - cvr).max()))
        assert np.abs(area - cvr).max() <= 1e-4                   # the reference is the reference project's op
        ref = _normalise(area)
        e = 2 * ((nx + ny + 4) * U / 0.224 + 2 * U * (np.abs(ref) + 3))
        ok, nb = _fp16_match(got[i], ref, e)
        n_nb += nb
        assert ok.all(), (i, kinds[i], int((~ok).sum()), np.argwhere(~ok)[:5])
        tol = 2.0 ** -11 * np.abs(ref) + e
        wrong = _normalise(area, true_rgb=True)
        r_rgb = min(r_rgb, float((np.abs(got[i] - wrong) / tol).max()))
        if kinds[i] == "bright":
            ren = _normalise(_area_resize(pages[i], Hn, Wn, renormalise=True)).astype(np.float16)
            sliver_rows += int((ren != ref.astype(np.float16)).sum())    # values where the variant rounds apart
            sliver_miss += int((got[i] != ren).sum())
    print("[preprocess] %dx%d -> %dx%d n %d: fp16(ref) exact except %d values next to a midpoint; reference vs cv2 %.2g; "
          "mean/std on true RGB %.0f x tol; renormalised weights: %d fp16 values differ from the reference, the kernel "
          "misses %d" % (H0, W0, Hn, Wn, n, n_nb, worst_cv, r_rgb, sliver_rows, sliver_miss))
    assert r_rgb >= 10.0, r_rgb
    if sliver_rows:
        assert sliver_miss > 0                                    # the sliver rule is what the kernel does


# ======================================================================================================== stem
def _stem_case(n, Hn, Wn, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, 3, Hn, Wn, generator=g) * 1.2).half()
    w = torch.randn(64, 3, 7, 7, generator=g) * 0.1
    b = torch.randn(64, generator=g) * 0.2
    return x, w, b


def _stem_ref(x64, w64, b64, variant=None):
    if variant == "shift":                                        # the canvas read one pixel up-left
        return F.relu(F.conv2d(F.pad(x64, (2, 4, 2, 4)), w64, b64, stride=2))
    if variant == "kh_kw":
        w64 = w64.transpose(2, 3)
    if variant == "rb":
        x64 = x64.flip(1)
    return F.relu(F.conv2d(x64, w64, b64, stride=2, padding=3))


STEM_SHAPES = [(32, 32), (32, 1600), (1600, 32), (96, 160), (1184, 1600)]


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("Hn,Wn", STEM_SHAPES)
def test_stem_vs_float64(Hn, Wn, n):
    x, w, b = _stem_case(n, Hn, Wn, seed=Hn * 3 + Wn + n)
    canvas = torch.zeros(n, Hn + 6, Wn + 8, 8, dtype=torch.float16)
    canvas[:, 3:3 + Hn, 3:3 + Wn, :3] = x.permute(0, 2, 3, 1)
    cd = canvas.to(DEV)
    Ho, Wo = Hn // 2, Wn // 2
    out = torch.full((n * Ho * Wo * 64 + 4096,), SENT, dtype=torch.float16, device=DEV)
    _lib.check(_lib.lib().ytk_op_dbnet_stem_f16(_fp(cd), n, Hn, Wn, _fp(w), _fp(b), _fp(out), None))
    torch.cuda.synchronize()
    out = out.cpu()
    assert (out[n * Ho * Wo * 64:] == SENT).all()
    got = out[:n * Ho * Wo * 64].reshape(n, Ho, Wo, 64).permute(0, 3, 1, 2).double().to(DEV)
    x64, w64, b64 = x.double().to(DEV), w.half().double().to(DEV), b.double().to(DEV)
    want = _stem_ref(x64, w64, b64)
    mag = F.conv2d(x64.abs(), w64.abs(), b64.abs(), stride=2, padding=3)
    tol = 2.0 ** -11 * want.abs() + 2.0 ** -25 + 2 * 148 * U * mag
    r = _ratio(got, want, tol)
    misses = {v: _ratio(got, _stem_ref(x64, w64, b64, v), tol) for v in ("shift", "kh_kw", "rb")}
    print("[stem] %dx%d n %d: worst |d| / tol %.3f; wrong variants: %s" % (
        Hn, Wn, n, r, ", ".join("%s %.0f x tol" % kv for kv in misses.items())))
    assert r <= 1.0, r
    for v, m in misses.items():
        assert m >= 10.0, (v, m)


# ======================================================================================================== max-pool
POOL_CASES = [(1, 7, 9, 8), (2, 8, 10, 64), (3, 33, 32, 8), (2, 296, 400, 64), (1, 320, 320, 64), (2, 480, 480, 64)]


@pytest.mark.parametrize("negative", [False, True], ids=["mixed", "negative"])
@pytest.mark.parametrize("n,H,W,C", POOL_CASES)
def test_maxpool_bitwise(n, H, W, C, negative):
    g = torch.Generator().manual_seed(H * W + C + n)
    x = torch.randn(n, H, W, C, generator=g) * 3
    if negative:
        x = -(x.abs() + 0.01)                   # all negative: a zero-padded max-pool returns 0 along the border
    x = x.half().to(DEV)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    out = torch.full((n * Ho * Wo * C + 1024,), SENT, dtype=torch.float16, device=DEV)
    _lib.check(_lib.lib().ytk_op_maxpool3x3s2_f16(_fp(x), n, H, W, C, _fp(out), None))
    torch.cuda.synchronize()
    assert (out[n * Ho * Wo * C:] == SENT).all()
    got = out[:n * Ho * Wo * C].reshape(n, Ho, Wo, C)
    xc = x.permute(0, 3, 1, 2).float()
    want = F.max_pool2d(xc, 3, 2, 1).half().permute(0, 2, 3, 1)
    assert torch.equal(got, want)
    zero_pad = F.max_pool2d(F.pad(xc, (1, 1, 1, 1)), 3, 2, 0).half().permute(0, 2, 3, 1)
    if negative:
        assert not torch.equal(got, zero_pad)


# ======================================================================================================== upsampling
def _bilinear_matrix(s, d, align_corners=False):
    """float64 [d, s] interpolation weights along one axis"""
    m = torch.zeros(d, s, dtype=torch.float64)
    for i in range(d):
        if align_corners:
            f = i * (s - 1) / (d - 1) if d > 1 else 0.0
        else:
            f = max((i + 0.5) * s / d - 0.5, 0.0)
        y0 = min(int(math.floor(f)), s - 1)
        y1 = min(y0 + 1, s - 1)
        l = f - y0
        m[i, y0] += 1 - l
        m[i, y1] += l
    return m


def _bilinear(src, Hd, Wd, align_corners=False):
    """src [n, Hs, Ws, C] -> float64 [n, Hd, Wd, C]"""
    Ay = _bilinear_matrix(src.shape[1], Hd, align_corners).to(src.device)
    Ax = _bilinear_matrix(src.shape[2], Wd, align_corners).to(src.device)
    return torch.einsum("yh,nhwc,xw->nyxc", Ay, src.double(), Ax)


# (n, Hs, Ws, C, Hd, Wd, ldd, coff, accumulate): the engine's top-down sums (x2 into C = 256) and the concat of
# p2 / p3 / p4 (x2 at coff 128, x4 at 64 and 0 of a 256-channel buffer), then non-integer ratios
UP_CASES = [(2, 37, 50, 256, 74, 100, 256, 0, 1), (1, 74, 100, 256, 148, 200, 256, 0, 1),
            (2, 74, 100, 64, 148, 200, 256, 128, 0), (2, 37, 50, 64, 148, 200, 256, 64, 0),
            (1, 37, 50, 64, 148, 200, 256, 0, 0), (3, 37, 50, 64, 96, 128, 256, 64, 0),
            (2, 50, 37, 32, 77, 64, 48, 8, 1), (1, 13, 17, 8, 40, 41, 8, 0, 0), (2, 40, 41, 16, 29, 23, 40, 24, 1)]


@pytest.mark.parametrize("n,Hs,Ws,C,Hd,Wd,ldd,coff,acc", UP_CASES)
def test_upsample_vs_float64(n, Hs, Ws, C, Hd, Wd, ldd, coff, acc):
    g = torch.Generator().manual_seed(Hs * Ws + Hd + coff + acc)
    src = (torch.randn(n, Hs, Ws, C, generator=g) * 2).half().to(DEV)
    dst = torch.full((n + 1, Hd, Wd, ldd), SENT, dtype=torch.float16, device=DEV)
    old = (torch.randn(n, Hd, Wd, C, generator=g) * 2).half().to(DEV)
    if acc:
        dst[:n, :, :, coff:coff + C] = old
    _lib.check(_lib.lib().ytk_op_upsample_bilinear_f16(_fp(src), n, Hs, Ws, C, _fp(dst), Hd, Wd, ldd, coff, acc, None))
    torch.cuda.synchronize()
    assert (dst[n] == SENT).all()                                 # nothing past the n images
    assert (dst[:n, :, :, :coff] == SENT).all() and (dst[:n, :, :, coff + C:] == SENT).all()
    got = dst[:n, :, :, coff:coff + C].double()
    base = old.double() if acc else 0.0
    want = base + _bilinear(src, Hd, Wd)
    smax = src.abs().max().double()
    tol = 2.0 ** -11 * want.abs() + 2.0 ** -25 + (16 * max(Hs, Ws) + 8) * U * smax
    if acc:
        tol = tol + 2 * U * old.double().abs()
    r = _ratio(got, want, tol)
    r_ac = _ratio(got, base + _bilinear(src, Hd, Wd, align_corners=True), tol)
    print("[upsample] n %d %dx%d -> %dx%d C %d at %d of %d, %s: worst |d| / tol %.3f; align_corners=True %.0f x tol"
          % (n, Hs, Ws, Hd, Wd, C, coff, ldd, "accumulate" if acc else "write", r, r_ac))
    assert r <= 1.0, r
    assert r_ac >= 10.0, r_ac


# ======================================================================================================== scale fusion
def _asf_weights(g):
    # the spatial kernel leans positive so that relu(conv m) is mostly active and its orientation matters
    return dict(w1=torch.randn(16, 64, generator=g) * 0.25, w2=torch.randn(64, 16, generator=g) * 0.4,
                sp3=torch.randn(9, generator=g) * 0.5 + 0.3, sp1=float(torch.randn(1, generator=g).abs() * 2 + 1),
                att=torch.randn(4, 64, generator=g) * 0.2)


def _asf_ref(a, fuse, wt, variant=None, gate=None):
    """float64 ScaleChannelSpatialAttention after its conv and the per-group rescale of fuse = [p4, p3, p2, p1].
    a [n, H, W, 64], fuse [n, H, W, 256] -> (g [n, 64], m [n, H, W], fuse out, error bounds e_g, e_m, e_score).
    gate: the device's fp32 gate, which the channel-mean and rescale kernels read; m and fuse are then computed from
    it (and their bounds leave out the gate's own error).
    Wrong variants: 'no_g' (m without sigmoid(g)), 'flip' (3x3 spatial kernel flipped), 'swap' (score i on group 3-i)."""
    a = a.double()
    n, H, W, _ = a.shape
    w1, w2, att = wt["w1"].double().to(a.device), wt["w2"].double().to(a.device), wt["att"].double().to(a.device)
    sp3 = wt["sp3"].double().to(a.device).reshape(1, 1, 3, 3)
    sp1 = wt["sp1"]
    HW = H * W
    L = math.ceil(math.ceil(HW / 64) / 32) + 32 + 64 + 1
    mean = a.mean((1, 2))                                                       # AdaptiveAvgPool2d(1)
    hid = F.relu(mean @ w1.T)
    gl = hid @ w2.T
    g = torch.sigmoid(gl)
    e_mean = L * U * a.abs().mean((1, 2))
    e_hid = e_mean @ w1.abs().T + 65 * U * (mean.abs() @ w1.abs().T)
    e_gl = e_hid @ w2.abs().T + 17 * U * (hid.abs() @ w2.abs().T)
    e_g = 2 * (_dsig(gl, e_gl) * e_gl + _E(gl))
    if gate is not None:
        g, e_gd = gate.double(), torch.zeros_like(e_g)
    else:
        e_gd = e_g
    m = a.mean(-1) + (0 if variant == "no_g" else g.mean(-1)[:, None, None])
    k = sp3.flip(2, 3) if variant == "flip" else sp3
    conv = F.conv2d(m[:, None], k, padding=1)[:, 0]
    sarg = sp1 * F.relu(conv)
    s = torch.sigmoid(sarg)
    z = s[..., None] + a + g[:, None, None, :]
    part = z @ att.T                                                            # [n, H, W, 4]
    score = torch.sigmoid(part)
    if variant == "swap":
        score = score.flip(-1)
    out = fuse.double() * score.repeat_interleave(64, -1)
    # first-order fp32 error bounds (module docstring)
    e_m = 2 * (12 * U * a.abs().mean(-1) + e_gd.mean(-1)[:, None, None] + 65 * U * g.mean(-1)[:, None, None] +
               2 * U * m.abs())
    e_conv = sp3.abs().sum() * (e_m.amax((1, 2)) + 9 * U * m.abs().amax((1, 2)))[:, None, None]
    e_sarg = abs(sp1) * e_conv
    e_s = _dsig(sarg, e_sarg) * e_sarg + _E(sarg)
    e_z = e_s[..., None] + e_gd[:, None, None, :] + 2 * U * z.abs()
    e_part = e_z @ att.abs().T + 64 * U * (z.abs() @ att.abs().T)
    e_score = 2 * (_dsig(part, e_part) * e_part + _E(part))
    return g, m, out, e_g, e_m, e_score


# (n, H, W, offset of a): HW = 1, 63, 65 against the 64 pooling chunks and 32 pixel lanes, and the engine's size
ASF_CASES = [(1, 1, 1, 0.0), (2, 7, 9, 0.0), (3, 5, 13, 0.0), (4, 1, 65, 0.0), (2, 296, 400, 0.0), (1, 296, 400, 100.0),
             (3, 5, 13, 100.0)]


@pytest.mark.parametrize("n,H,W,offset", ASF_CASES)
def test_asf_vs_float64(n, H, W, offset):
    g = torch.Generator().manual_seed(n * 1000 + H * W + int(offset))
    wt = _asf_weights(g)
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    ramp = (torch.sin(0.9 * xx) + torch.cos(0.6 * yy)).float()[None, :, :, None]   # asymmetric spatial pattern
    a = (torch.randn(n, H, W, 64, generator=g) + ramp + offset).half().to(DEV)
    fuse = (torch.randn(n, H, W, 256, generator=g) * 2).half()
    fbuf = torch.full((n * H * W * 256 + 1024,), SENT, dtype=torch.float16, device=DEV)
    fbuf[:n * H * W * 256] = fuse.reshape(-1).to(DEV)
    gvec = torch.full((n + 1, 64), float("nan"), device=DEV)
    mbuf = torch.full((n * H * W + 64,), float("nan"), device=DEV)
    w1d, w2d = wt["w1"].to(DEV).contiguous(), wt["w2"].to(DEV).contiguous()
    sp3h, atth = wt["sp3"].contiguous(), wt["att"].contiguous()
    _lib.check(_lib.lib().ytk_op_asf_f16(_fp(a), _fp(fbuf), n, H, W, _fp(w1d), _fp(w2d), _fp(sp3h), wt["sp1"], _fp(atth),
                                         _fp(gvec), _fp(mbuf), None))
    torch.cuda.synchronize()
    assert torch.isnan(gvec[n]).all() and torch.isnan(mbuf[n * H * W:]).all()
    assert (fbuf[n * H * W * 256:] == SENT).all()
    got_g, got_m = gvec[:n].double(), mbuf[:n * H * W].reshape(n, H, W).double()
    got_f = fbuf[:n * H * W * 256].reshape(n, H, W, 256).double()
    want_g, _, _, e_g, _, _ = _asf_ref(a, fuse.to(DEV), wt)
    _, want_m, want_f, _, e_m, e_score = _asf_ref(a, fuse.to(DEV), wt, gate=got_g)
    tol_f = 2 * fuse.to(DEV).double().abs() * e_score.repeat_interleave(64, -1) + 2.0 ** -11 * want_f.abs() + 2.0 ** -25
    r_g, r_m, r_f = _ratio(got_g, want_g, e_g), _ratio(got_m, want_m, e_m), _ratio(got_f, want_f, tol_f)
    r_nog = _ratio(got_m, _asf_ref(a, fuse.to(DEV), wt, "no_g", gate=got_g)[1], e_m)
    misses = {"no sigmoid(g) in m": r_nog}
    if offset == 0:
        # with the offset the scores saturate to 0 / 1 and a wrong variant may land on the same values
        misses["groups swapped"] = _ratio(got_f, _asf_ref(a, fuse.to(DEV), wt, "swap", gate=got_g)[2], tol_f)
        if H * W > 1:
            flip = _asf_ref(a, fuse.to(DEV), wt, "flip", gate=got_g)[2]
            misses["spatial kernel flipped"] = _ratio(got_f, flip, tol_f)
    print("[asf] n %d %dx%d offset %g: worst |d| / tol gate %.3f, channel mean %.3f, fuse %.3f; wrong variants: %s"
          % (n, H, W, offset, r_g, r_m, r_f, ", ".join("%s %.0f x tol" % kv for kv in misses.items())))
    assert r_g <= 1.0 and r_m <= 1.0 and r_f <= 1.0, (r_g, r_m, r_f)
    for v, m in misses.items():
        assert m >= 10.0, (v, m)


# ======================================================================================================== fused head
def _head_ref(x64, w1, b1, w2, b2, variant=None):
    """float64 head on x [n, 64, H, W] -> (prob [n, 4H, 4W], error bound).  Wrong variants: 't1' / 't2' (the 2x2
    sub-block of the first / second transposed conv transposed), 'no_relu'."""
    if variant == "t1":
        w1 = w1.transpose(2, 3)
    if variant == "t2":
        w2 = w2.transpose(2, 3)
    pre = F.conv_transpose2d(x64, w1, b1, stride=2)
    h = pre if variant == "no_relu" else F.relu(pre)
    logit = F.conv_transpose2d(h, w2, b2, stride=2)
    prob = torch.sigmoid(logit)[:, 0]
    e_h = 130 * U * (F.conv_transpose2d(x64.abs(), w1.abs(), b1.abs(), stride=2))
    e_logit = F.conv_transpose2d(e_h, w2.abs(), stride=2) + 128 * U * F.conv_transpose2d(h.abs(), w2.abs(), stride=2)
    tol = 2 * (_dsig(logit, e_logit) * e_logit + _E(logit))[:, 0] + U
    return prob, tol


HEAD_SHAPES = [(8, 8), (8, 400), (400, 8), (37, 50), (296, 400)]


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("H,W", HEAD_SHAPES)
def test_head_vs_float64(H, W, n):
    g = torch.Generator().manual_seed(H * W + n)
    x = (torch.randn(n, H, W, 64, generator=g).abs() * 1.5).half().to(DEV)    # the output of a ReLU
    w1 = torch.randn(64, 64, 2, 2, generator=g) * 0.15
    b1 = torch.randn(64, generator=g) * 0.2
    w2 = torch.randn(64, 1, 2, 2, generator=g) * 0.3
    b2 = float(torch.randn(1, generator=g)[0] * 0.3)
    npx = n * 16 * H * W
    prob = torch.full((npx + 4096,), float("nan"), device=DEV)
    _lib.check(_lib.lib().ytk_op_dbnet_head_f32(_fp(x), n, H, W, _fp(w1), _fp(b1), _fp(w2), b2, _fp(prob), None))
    torch.cuda.synchronize()
    assert torch.isnan(prob[npx:]).all()                          # nothing past n * 4H * 4W
    got = prob[:npx].reshape(n, 4 * H, 4 * W).double()
    assert torch.isfinite(got).all()                              # ... and all of it written
    x64 = x.permute(0, 3, 1, 2).double()
    args = (w1.half().double().to(DEV), b1.double().to(DEV), w2.double().to(DEV),
            torch.tensor([b2], dtype=torch.float32).double().to(DEV))
    want, tol = _head_ref(x64, *args)
    r = _ratio(got, want, tol)
    misses = {v: _ratio(got, _head_ref(x64, *args, variant=v)[0], tol) for v in ("t1", "t2", "no_relu")}
    print("[head] %dx%d n %d: max|d| %.3g, worst |d| / tol %.3f; wrong variants: %s" % (
        H, W, n, (got - want).abs().max().item(), r, ", ".join("%s %.0f x tol" % kv for kv in misses.items())))
    assert r <= 1.0, r
    for v, m in misses.items():
        assert m >= 10.0, (v, m)


# ======================================================================================================== engine wiring
def _debug(model, n, H, W, name):
    L = _lib.lib()
    shape = (ctypes.c_int * 4)()
    cap = n * H * W * 64 + 16
    buf = torch.empty(cap, dtype=torch.float32)
    _lib.check(L.ytk_dbnet_debug_tensor(model._ensure(), n, H, W, name.encode(), buf.data_ptr(), cap, shape))
    n_, h_, w_, c_ = list(shape)
    return buf[: n_ * h_ * w_ * c_].reshape(n_, h_, w_, c_)


def test_engine_passes_the_op_arguments():
    """The engine's max-pool and channel-mean map at 1184 x 1600, n = 2, against the same checks on its own
    intermediates: the arguments it passes are the ones the op-level cases cover."""
    from yomitoku_b200 import TextDetector
    d = TextDetector(from_pretrained=False, device="cuda")
    sd = weights.make_dbnet_state_dict(seed=3)
    d.model.load_state_dict(sd)
    H, W = 1184, 1600
    x = torch.randn(2, 3, H, W, generator=torch.Generator().manual_seed(5))
    d.model(x)
    stem = _debug(d.model, 2, H, W, "stem").to(DEV)
    pool = _debug(d.model, 2, H, W, "pool").to(DEV)
    want = F.max_pool2d(stem.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert torch.equal(pool, want)
    a = _debug(d.model, 2, H, W, "asf_a").to(DEV)
    m = _debug(d.model, 2, H, W, "asf_m")[..., 0].to(DEV).double()
    e = "decoder.concat_attention.enhanced_attention."
    wt = dict(w1=sd[e + "channel_wise.1.weight"].reshape(16, 64), w2=sd[e + "channel_wise.3.weight"].reshape(64, 16),
              sp3=sd[e + "spatial_wise.0.weight"].reshape(9), sp1=float(sd[e + "spatial_wise.2.weight"].reshape(-1)[0]),
              att=sd[e + "attention_wise.0.weight"].reshape(4, 64))
    _, want_m, _, _, e_m, _ = _asf_ref(a, torch.zeros(2, H // 4, W // 4, 256, device=DEV), wt)
    r = _ratio(m, want_m, e_m)
    print("[engine] pool == max_pool2d(stem); asf_m worst |d| / tol %.3f" % r)
    assert r <= 1.0, r
