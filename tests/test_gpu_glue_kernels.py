"""GPU: op-level parity of the RT-DETRv2 engine's small kernels and of PARSeq's patch input through the C ABI, against
float64, torch or exact integer references on the operands the kernel reads (fp16 values where it reads fp16), and the
engine's wiring of those kernels checked in place through its debug tensors.

  avgpool2        ytk_op_rt_avgpool2_f16 (avgpool2_kernel)
                  magnitudes within 2^12 of each other (the fp16 exponents of four inputs differ by at most 11): the
                  four-term fp32 sum and the * 0.25 are exact, so the output is the fp16 round-to-nearest-even of the
                  float64 mean, bit for bit; any magnitudes: within one fp16 ulp of the float64 mean plus the error of
                  a three-addition fp32 sum, 3 * 2^-24 * mean(|x|) (it matters only where the four values cancel)
  upsample        ytk_op_rt_upsample_nearest2_f16 (upsample_nearest2_kernel): bit copy of repeat_interleave, every
                  column outside [coff, coff + C) untouched
  add             ytk_op_rt_add_f16 (add_f16_kernel): bit for bit (a.float() + b.float()).half(), or with the fp32
                  table (a.float() + table[row % period]).half(); and within one fp16 ulp of float64
  mask_invalid    ytk_op_rt_mask_invalid_f32: the listed anchors' rows of every image equal the bias, every other row is
                  bit-unchanged
  enc_scores      ytk_op_rt_enc_scores_f32: exactly max(logits[rt_anchor_row(img, a), :C])
  gather_queries  ytk_op_rt_gather_queries_f32: tgt, tgt16 = tgt.half() and anchor_sel (with +inf) exactly
  ref_update      ytk_op_rt_ref_update_f32 vs float64 sigmoid(delta + base), base = anchor or inverse_sigmoid(ref):
                  |d| <= s (1 - s) (|t| 2^-24 + e_base + 2^-21) + 2^-22 s, s the float64 result, t = delta + base;
                  e_base = 0 with anchors, 2^-22 (1 + |base|) + 4e-8 in the refinement
  qpos_l0         ytk_op_rt_qpos_l0_f32 vs float64 relu(W r + b): |d| <= ulp16(|y| + E) / 2 + E, E = 6 * 2^-24 *
                  (|b| + sum |w_i r_i|); clearly negative pre-activations (y < -E) give exactly 0
  patchify        ytk_op_patchify_u8 / _f32 (patchify_u8_kernel, patchify_f32_kernel): A bit for bit equal to the
                  torch fp32 restatement of ToTensor + Normalize(0.5, 0.5), then .half() (u8), or to the pixels' .half()
                  (f32); -1 right of the stored width, zero K padding, x rows = pos_embed cropped as oracle/parseq.py
                  crops it, token rows outside every crop untouched - all exact

The ref_update bound: the library is built without --use_fast_math, so expf is within 2 ulp and logf within 1 ulp
(CUDA C Programming Guide, mathematical functions), and the fp32 division is correctly rounded.  The refinement base
log(max(x, 1e-5) / max(1 - x, 1e-5)) carries the rounding of 1 - x and of the division (2^-24 relative each), logf's
ulp of the result (2^-23 |base|) and the fp32 value of the clamp 1e-5 (relative 2.5e-8).  The sum t = delta + base
rounds once (2^-24 |t|); sigmoid turns a relative error r of exp(-t) into s (1 - s) r, and 1 + e and the division each
add 2^-24 s.  The bound doubles each of those terms.

The qpos_l0 term E: a bias plus a four-term dot product in fp32 (with or without fused multiply-adds) is within
5 * 2^-24 * (|b| + sum |w_i r_i|) of the exact value; rounding that to fp16 adds at most half an fp16 ulp.  Its worst
ratio sits near 1 for any correct kernel: the fp16 rounding alone can take the whole half ulp, and E is small.

Every comparator is also given a plausible wrong result computed on the host - h and w swapped, a level boundary
shifted by one, the token pairing of the position table transposed, the clamp in inverse_sigmoid removed, a delta stride
of 4, the ref components paired with the wrong weights, pos_embed taken from the cropped grid width instead of the full
one, the padding value 0 - and must reject it.

The in-situ checks run one layout forward at 640 with n = 3 and one cell-detector forward at 960 with n = 2 (seeded
weights, enc_output.proj given a nonzero bias so that the masked rows are visible) and require the relations between
the engine's debug tensors that its wiring of these kernels implies: the packed input, the FPN up-sampling halves of
cat4 / cat3, fpn4 = t2 + x2 of the first FPN block, aifi.q = proj5 + pos (every image), the bias rows of the invalid
anchors, the encoder scores through the level-major row order, anchor_sel = anchors[topk] and pred_logits =
logits[:, :C].  aifi.q is compared with the float64 sum within one fp16 ulp plus 2^-21 (1 + g), g the
grid side: the engine's fp32 table and oracle.rtdetr.sincos_2d evaluate powf, the product y * omega and sin / cos
separately, each within an fp32 ulp or two, so their arguments (up to g) and values may differ by that much."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import parseq as OP
from oracle import rtdetr as R
from yomitoku_b200 import _lib
from yomitoku_b200.config import LayoutParserRTDETRv2V2Config, TableCellParserRTDETRv2Config, to_config
from yomitoku_b200.models import RTDETRv2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D = 256
SQ640 = [(80, 80), (40, 40), (20, 20)]
SQ960 = [(120, 120), (60, 60), (30, 30)]
RAGGED = [(12, 20), (6, 10), (3, 5), (2, 3)]         # four non-square levels


def L():
    return _lib.lib()


def _bits(t):
    return t.contiguous().view(torch.int16)


def _ulp16(v):
    """fp16 ulp at |v| (float64 tensor), the subnormal spacing below 2^-14."""
    _, e = torch.frexp(v.abs().double().clamp(min=2.0 ** -14))
    return torch.ldexp(torch.ones_like(v, dtype=torch.float64), e - 11)


def _ratio(got, want, tol):
    return ((got.double() - want.double()).abs() / tol).max().item()


def _report(name, worst):
    print("%-40s worst |d| / bound = %.3g" % (name, worst))


def _rand_f16(shape, g, lo=-6, hi=6):
    """fp16 values with magnitudes in [2^lo, 2^hi) (log-uniform) and random signs."""
    mag = torch.exp2(torch.rand(shape, generator=g, dtype=torch.float64) * (hi - lo) + lo)
    sign = torch.randint(0, 2, shape, generator=g).double() * 2 - 1
    return (mag * sign).half()


# ======================================================================================================== avgpool2
def _pool_ref(x):
    """float64 mean of each 2x2 cell of NHWC x, summed in the kernel's order."""
    x = x.double()
    return (x[:, 0::2, 0::2] + x[:, 0::2, 1::2] + x[:, 1::2, 0::2] + x[:, 1::2, 1::2]) / 4


def _avgpool(x):
    n, H, W, C = x.shape
    out = torch.full((n, H // 2, W // 2, C), float("nan"), dtype=torch.float16, device=DEV)
    _lib.check(L().ytk_op_rt_avgpool2_f16(x.data_ptr(), n, H, W, C, out.data_ptr(), None))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("n,H,W,C", [
    (1, 160, 160, 256), (3, 80, 80, 512), (1, 40, 40, 1024),           # the three pooled shortcuts at 640
    (1, 240, 240, 256), (3, 120, 120, 512), (8, 60, 60, 1024),         # and at 960
    (3, 6, 10, 8), (8, 10, 6, 16), (1, 2, 2, 8), (3, 2, 2, 24),        # non-square; 45, 240, 1 and 9 threads
])
def test_avgpool2_vs_float64(n, H, W, C):
    g = torch.Generator().manual_seed(n * 1000 + H + W + C)
    x = _rand_f16((n, H, W, C), g, -6, 5.9).to(DEV)                  # |x| in [2^-6, 2^5.9]: ratio below 2^12
    got = _avgpool(x)
    mean = _pool_ref(x)
    # exact sum: one rounding of the float64 mean (exactly representable in fp32) to fp16
    assert torch.equal(_bits(got), _bits(mean.half()))
    # h and w swapped: the same bytes pooled as an (n, W, H, C) image
    if H != W:
        wrong = _pool_ref(x.reshape(n, W, H, C)).half().reshape(n, H // 2, W // 2, C)
        assert not torch.equal(_bits(got), _bits(wrong))
    # magnitudes from 2^-20 to 2^15: inexact sums, one fp16 ulp plus the fp32 sum's error where the four cancel
    wide = _rand_f16((n, H, W, C), g, -20, 15).to(DEV)
    got = _avgpool(wide)
    mean = _pool_ref(wide)
    worst = _ratio(got, mean, _ulp16(mean) + 3 * 2.0 ** -24 * _pool_ref(wide.abs()))
    _report("avgpool2 %dx%dx%dx%d wide range" % (n, H, W, C), worst)
    assert worst <= 1.0


# ======================================================================================================== upsample
def _nearest2(x):
    return x.repeat_interleave(2, 1).repeat_interleave(2, 2)


@pytest.mark.parametrize("n,Hs,Ws,C", [(1, 20, 20, D), (3, 40, 40, D), (2, 30, 30, D), (1, 60, 60, D), (3, 3, 5, 8),
                                        (2, 7, 4, 24)])
@pytest.mark.parametrize("first_half", [True, False])
def test_upsample_nearest2_bitwise(n, Hs, Ws, C, first_half):
    g = torch.Generator().manual_seed(Hs * 7 + Ws + C + n)
    # the engine reads the lateral output from the second half of a [.., 2D] PAN buffer (l5 = pcat5 + D) and writes the
    # first half of a [.., 2D] FPN buffer; every 16-bit pattern is moved, NaN and infinity included
    srcbuf = torch.randint(-32768, 32768, (n, Hs, Ws, 2 * C), generator=g, dtype=torch.int16).to(DEV)
    src = srcbuf.view(torch.float16)
    coff = 0 if first_half else C
    sent = torch.full((n, 2 * Hs, 2 * Ws, 2 * C), 0x5A5A, dtype=torch.int16, device=DEV)
    dst = sent.clone()
    _lib.check(L().ytk_op_rt_upsample_nearest2_f16(src.data_ptr() + C * 2, 2 * C, n, Hs, Ws, C, dst.data_ptr(), 2 * C,
                                                   coff, None))
    torch.cuda.synchronize()
    want = sent.clone()
    want[..., coff:coff + C] = _nearest2(srcbuf[..., C:])
    assert torch.equal(dst, want)
    if Hs != Ws:                                                   # h and w swapped
        wrong = sent.clone()
        wrong[..., coff:coff + C] = _nearest2(srcbuf[..., C:].reshape(n, Ws, Hs, C)).reshape(n, 2 * Hs, 2 * Ws, C)
        assert not torch.equal(dst, wrong)


# ======================================================================================================== add
def _add(a, b=None, table=None, period=1):
    rows, C = a.shape
    out = torch.full_like(a, float("nan"))
    _lib.check(L().ytk_op_rt_add_f16(a.data_ptr(), None if b is None else b.data_ptr(),
                                     None if table is None else table.data_ptr(), C, period, out.data_ptr(), rows, None))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("rows,C", [(3 * 1600, D), (8 * 300, D), (2 * 1500 + 5, D), (45, 8), (1, 8)])
def test_add_f16_bitwise(rows, C):
    g = torch.Generator().manual_seed(rows + C)
    a = _rand_f16((rows, C), g, -20, 14).to(DEV)
    b = _rand_f16((rows, C), g, -20, 14).to(DEV)
    got = _add(a, b)
    assert torch.equal(_bits(got), _bits((a.float() + b.float()).half()))
    exact = a.double() + b.double()
    worst = _ratio(got, exact, _ulp16(exact))
    _report("add f16 %dx%d" % (rows, C), worst)
    assert worst <= 1.0


def _swap_grid(period):
    """token r = y * g + x -> x * g + y: the transposed token pairing of the square AIFI grid"""
    gs = int(round(math.sqrt(period)))
    r = torch.arange(period)
    return (r % gs) * gs + r // gs


@pytest.mark.parametrize("n,period", [(1, 400), (3, 400), (8, 400), (1, 900), (2, 900), (8, 900), (3, 401)])
def test_add_table_bitwise(n, period):
    g = torch.Generator().manual_seed(n * 31 + period)
    rows = n * period if period % 100 == 0 else n * 400 + 17        # 3 x 400 + 17 rows: 401 does not divide them
    a = _rand_f16((rows, D), g, -12, 6).to(DEV)
    table = (torch.randn(period, D, generator=g) * 2).to(DEV)
    got = _add(a, table=table, period=period)
    ridx = torch.arange(rows, device=DEV) % period
    assert torch.equal(_bits(got), _bits((a.float() + table[ridx]).half()))
    exact = a.double() + table.double()[ridx]
    worst = _ratio(got, exact, _ulp16(exact))
    _report("add table n=%d period=%d" % (n, period), worst)
    assert worst <= 1.0
    if period % 100 == 0:                                           # the transposed token pairing
        wrong = (a.float() + table[_swap_grid(period).to(DEV)[ridx]]).half()
        assert not torch.equal(_bits(got), _bits(wrong))


# ======================================================================================================== level-major rows
def _levels(shapes):
    arr = lambda v: (ctypes.c_int * len(v))(*v)
    return arr([h for h, _ in shapes]), arr([w for _, w in shapes]), len(shapes)


def _offsets(shapes):
    off = [0]
    for h, w in shapes:
        off.append(off[-1] + h * w)
    return off


def anchor_row(shapes, n, img, a, shift=False):
    """rt_anchor_row (csrc/rtdetr_ops.h) over tensors: level l of image img holds rows off[l] * n + img * h * w + ...
    shift=True: the level boundary shifted by one (an anchor equal to off[l] stays in level l - 1)."""
    off = torch.tensor(_offsets(shapes), dtype=torch.int64, device=a.device)
    hw = torch.tensor([h * w for h, w in shapes], dtype=torch.int64, device=a.device)
    lvl = torch.zeros_like(a)
    for k in range(1, len(shapes)):
        lvl += (a > off[k]) if shift else (a >= off[k])
    return off[lvl] * n + img * hw[lvl] + (a - off[lvl])


def _edge_anchors(shapes):
    """first and last anchor of every level"""
    off = _offsets(shapes)
    return sorted({v for l in range(len(shapes)) for v in (off[l], off[l + 1] - 1)})


def _invalid_lists():
    """(shapes, anchors): the border anchors of the engine's two sizes, and random lists with every level's ends"""
    out = []
    for size, shapes in ((640, SQ640), (960, SQ960)):
        _, valid = R.generate_anchors(R.RTDETRSpec(img_size=[size, size]))
        out.append((shapes, torch.nonzero(~valid.reshape(-1)).reshape(-1).tolist()))
    g = torch.Generator().manual_seed(5)
    for shapes in (SQ640, RAGGED):
        total = _offsets(shapes)[-1]
        pick = torch.randperm(total, generator=g)[:total // 7].tolist()
        out.append((shapes, sorted(set(pick) | set(_edge_anchors(shapes)))))
    return out


@pytest.mark.parametrize("case", range(4))
@pytest.mark.parametrize("n", [1, 3, 8])
def test_mask_invalid_exact(case, n):
    shapes, invalid = _invalid_lists()[case]
    total = _offsets(shapes)[-1]
    g = torch.Generator().manual_seed(case * 10 + n)
    x0 = torch.randn(total * n, D, generator=g).to(DEV)
    bias = torch.randn(D, generator=g).to(DEV)
    inv = torch.tensor(invalid, dtype=torch.int32, device=DEV)
    x = x0.clone()
    h, w, nl = _levels(shapes)
    _lib.check(L().ytk_op_rt_mask_invalid_f32(x.data_ptr(), D, bias.data_ptr(), inv.data_ptr(), len(invalid), h, w, nl,
                                              n, None))
    torch.cuda.synchronize()

    def expected(shift):
        e = x0.clone()
        a = inv.long().repeat(n)
        img = torch.arange(n, device=DEV).repeat_interleave(len(invalid))
        e[anchor_row(shapes, n, img, a, shift)] = bias
        return e

    assert torch.equal(x, expected(False))
    # with one image the level-major order is the raster order; the border lists are closed under the shifted mapping
    # (the first anchor of a level and the first of the next image's level are both border anchors)
    if n > 1 and case >= 2:
        assert not torch.equal(x, expected(True))


@pytest.mark.parametrize("shapes", [SQ640, SQ960, RAGGED], ids=["640", "960", "ragged"])
@pytest.mark.parametrize("n", [1, 2, 8])
@pytest.mark.parametrize("C", [1, 3, 6])
def test_enc_scores_exact(shapes, n, C):
    total = _offsets(shapes)[-1]
    g = torch.Generator().manual_seed(total + n * 3 + C)
    # 16 levels of score (long runs of tied maxima) and columns C..7 above every real one, which must be ignored
    logits = (torch.randint(0, 16, (total * n, 8), generator=g) * 0.25 - 2.0).float()
    logits[:, C:] = 100.0 + torch.rand(total * n, 8 - C, generator=g)
    logits = logits.to(DEV)
    scores = torch.full((n, total), float("nan"), device=DEV)
    h, w, nl = _levels(shapes)
    _lib.check(L().ytk_op_rt_enc_scores_f32(logits.data_ptr(), 8, C, h, w, nl, n, scores.data_ptr(), None))
    torch.cuda.synchronize()
    rowmax = logits[:, :C].max(1).values
    a = torch.arange(total, device=DEV).repeat(n)
    img = torch.arange(n, device=DEV).repeat_interleave(total)
    assert torch.equal(scores.reshape(-1), rowmax[anchor_row(shapes, n, img, a)])
    if n > 1:
        assert not torch.equal(scores.reshape(-1), rowmax[anchor_row(shapes, n, img, a, shift=True)])


def _anchors(shapes):
    """[total, 4] anchors: the model's own (with +inf at the border) for the square sizes, else random with +inf rows"""
    for size, sq in ((640, SQ640), (960, SQ960)):
        if shapes == sq:
            return R.generate_anchors(R.RTDETRSpec(img_size=[size, size]))[0].reshape(-1, 4)
    total = _offsets(shapes)[-1]
    a = torch.randn(total, 4, generator=torch.Generator().manual_seed(2))
    a[::5] = float("inf")
    return a


@pytest.mark.parametrize("shapes,K", [(SQ640, 300), (SQ960, 1500), (RAGGED, 300)], ids=["640", "960", "ragged"])
@pytest.mark.parametrize("n", [1, 3, 8])
def test_gather_queries_exact(shapes, K, n):
    total = _offsets(shapes)[-1]
    g = torch.Generator().manual_seed(total + n)
    om = (torch.randn(total * n, D, generator=g) * torch.exp2(torch.randint(-10, 10, (total * n, 1), generator=g))).to(DEV)
    anchors = _anchors(shapes).to(DEV)
    idx = torch.stack([torch.randperm(total, generator=g)[:K] for _ in range(n)])
    edges = torch.tensor(_edge_anchors(shapes))
    idx[:, :len(edges)] = edges                                      # every image takes the ends of every level
    idx[-1, -len(edges):] = edges.flip(0)
    idx = idx.int().to(DEV)
    tgt = torch.full((n * K, D), float("nan"), device=DEV)
    tgt16 = torch.full((n * K, D), float("nan"), dtype=torch.float16, device=DEV)
    asel = torch.full((n * K, 4), float("nan"), device=DEV)
    h, w, nl = _levels(shapes)
    _lib.check(L().ytk_op_rt_gather_queries_f32(om.data_ptr(), D, idx.data_ptr(), K, h, w, nl, n, tgt.data_ptr(),
                                                tgt16.data_ptr(), anchors.data_ptr(), asel.data_ptr(), None))
    torch.cuda.synchronize()
    a = idx.reshape(-1).long()
    img = torch.arange(n, device=DEV).repeat_interleave(K)
    rows = anchor_row(shapes, n, img, a)
    assert torch.equal(tgt, om[rows])
    assert torch.equal(_bits(tgt16), _bits(om[rows].half()))
    assert torch.equal(asel, anchors[a])
    assert torch.isinf(asel).any()
    if n > 1:
        assert not torch.equal(tgt, om[anchor_row(shapes, n, img, a, shift=True)])


# ======================================================================================================== ref_update
def _inverse_sigmoid64(ref, clamp=True):
    x = ref.double().clip(0.0, 1.0)
    return torch.log(x.clip(min=1e-5) / (1 - x).clip(min=1e-5)) if clamp else torch.log(x / (1 - x))


def _ref_update(delta, asel, ref):
    out = ref.clone()
    _lib.check(L().ytk_op_rt_ref_update_f32(delta.data_ptr(), delta.shape[1], None if asel is None else asel.data_ptr(),
                                            out.data_ptr(), ref.shape[0], None))
    torch.cuda.synchronize()
    return out


def _ref_tol(t, s, e_base):
    return s * (1 - s) * (t.abs() * 2.0 ** -24 + e_base + 2.0 ** -21) + 2.0 ** -22 * s + 1e-300


@pytest.mark.parametrize("n", [8 * 300, 2 * 1500])
def test_ref_update_vs_float64(n):
    g = torch.Generator().manual_seed(n)
    # delta [n, 8]: the first 4 columns are read; columns 4..7 are huge, so a stride taken as 4 cannot pass
    delta = torch.cat([(torch.rand(n, 4, generator=g) * 2 - 1) * 30, torch.full((n, 4), 1e30)], 1)
    f = np.float32
    edges = [0.0, 1e-7, np.nextafter(f(1e-5), f(0)), f(1e-5), np.nextafter(f(1e-5), f(1)), 0.5,
             np.nextafter(f(1 - 1e-5), f(0)), f(1 - 1e-5), np.nextafter(f(1 - 1e-5), f(1)), np.nextafter(f(1), f(0)),
             1.0, -0.25, 1.5]
    ref = torch.rand(n, 4, generator=g)
    e = torch.tensor(np.array(edges, np.float32))
    ref.view(-1)[:len(e) * 9].copy_(e.repeat_interleave(9))          # every edge value in every box column
    delta[:len(e) * 3, :4] = (torch.rand(len(e) * 3, 4, generator=g) * 2 - 1) * 3
    anchor = torch.randn(n, 4, generator=g) * 3
    anchor[::7, 1] = float("inf")
    delta, ref, anchor = delta.to(DEV), ref.to(DEV), anchor.to(DEV)
    d = delta[:, :4].double()
    for base_kind in ("anchor", "refine"):
        if base_kind == "anchor":
            got = _ref_update(delta, anchor, ref)
            base, e_base = anchor.double(), 0.0
        else:
            got = _ref_update(delta, None, ref)
            base = _inverse_sigmoid64(ref)
            e_base = 2.0 ** -22 + 2.0 ** -22 * base.abs() + 4e-8
        t = d + base
        s = torch.sigmoid(t)
        assert bool(((got >= 0) & (got <= 1)).all())
        fin = torch.isfinite(t)                                       # +inf anchors only: exactly 1
        assert bool((got[~fin] == 1.0).all())
        assert bool((~fin).any()) == (base_kind == "anchor")
        tol = _ref_tol(t[fin], s[fin], e_base if base_kind == "anchor" else e_base[fin])
        worst = _ratio(got[fin], s[fin], tol)
        _report("ref_update %s n=%d" % (base_kind, n), worst)
        assert worst <= 1.0
        if base_kind == "refine":
            # the clamp removed: ref 0 / 1 become -inf / +inf before the sigmoid
            wrong = torch.sigmoid(d + _inverse_sigmoid64(ref, clamp=False))
            assert _ratio(got[fin], wrong[fin].nan_to_num(0.5), tol) > 1.0
        # delta read with a stride of 4
        wrong = torch.sigmoid(delta.reshape(-1)[:n * 4].reshape(n, 4).double() + base)
        assert _ratio(got[fin], wrong[fin], tol) > 1.0


# ======================================================================================================== qpos_l0
@pytest.mark.parametrize("rows", [8 * 300, 2 * 1500])
def test_qpos_l0_vs_float64(rows):
    H1 = 512
    g = torch.Generator().manual_seed(rows)
    ref = torch.rand(rows, 4, generator=g)
    ref[:64] = torch.randint(0, 2, (64, 4), generator=g).float()   # saturated boxes: components exactly 0 or 1
    W = torch.randn(H1, 4, generator=g) * 0.5
    b = torch.randn(H1, generator=g) * 0.02
    ref, W, b = ref.to(DEV), W.to(DEV), b.to(DEV)
    out = torch.full((rows, H1), float("nan"), dtype=torch.float16, device=DEV)
    _lib.check(L().ytk_op_rt_qpos_l0_f32(ref.data_ptr(), W.data_ptr(), b.data_ptr(), H1, out.data_ptr(), rows, None))
    torch.cuda.synchronize()
    y = ref.double() @ W.double().T + b.double()
    E = 6 * 2.0 ** -24 * ((ref.double().abs() @ W.double().abs().T) + b.double().abs())
    want = y.clamp(min=0)
    tol = 0.5 * _ulp16(want + E) + E
    worst = _ratio(out, want, tol)
    _report("qpos_l0 rows=%d" % rows, worst)
    assert worst <= 1.0
    neg = y < -E
    assert bool(neg.any()) and bool((out[neg] == 0).all())
    # the box components paired with the wrong weights (x, y, w, h against columns x, y, h, w)
    wrong = (ref[:, [0, 1, 3, 2]].double() @ W.double().T + b.double()).clamp(min=0)
    assert _ratio(out, wrong, tol) > 1.0


# ======================================================================================================== patchify
PATCH = {"large-v4_1": OP.SPECS["parseq-large-v4_1"], "tiny-dynw-v4": OP.SPECS["parseq-tiny-dynw-v4"],
         "tiny": OP.SPECS["parseq-tiny"], "small": OP.SPECS["parseq-small"]}
A_SENT, X_SENT = 0x3E3E, 7.0


def _kpad(ph, pw):
    return (3 * ph * pw + 63) // 64 * 64


def _patches(img, ph, pw):
    """(3, 32, wp) -> (gh * gw, 3 * ph * pw) in token order (gy major) and K order (c, py, px): the flattened conv weight"""
    c, H, Wd = img.shape
    return img.reshape(c, H // ph, ph, Wd // pw, pw).permute(1, 3, 0, 2, 4).reshape((H // ph) * (Wd // pw), c * ph * pw)


def _pos_rows(pos, spec, gh, gw, cropped=True):
    """oracle/parseq.py:87: pos_embed [gh * full_gw, D] as (gh, full_gw) cropped to (gh, gw); cropped=False is the wrong
    reading with the cropped grid width as the row pitch"""
    full_gw = spec.grid[1]
    Dm = pos.shape[1]
    if cropped:
        return pos.reshape(gh, full_gw, Dm)[:, :gw].reshape(gh * gw, Dm)
    return pos[:gh * gw]


def _crop_widths(ncrops, pw, g):
    base = [1, pw - 1, pw, pw + 1, 2 * pw - 1, 3 * pw + 5, 37, 200, 799]
    ws = [base[i % len(base)] for i in range(ncrops)]
    ws = [max(1, min(w, 800)) for w in ws]
    perm = torch.randperm(ncrops, generator=g).tolist()
    return [ws[i] for i in perm]


@pytest.mark.parametrize("model", list(PATCH))
@pytest.mark.parametrize("ncrops", [1, 7, 64])
def test_patchify_u8_exact(model, ncrops):
    spec = PATCH[model]
    ph, pw = spec.patch
    gh, full_gw = spec.grid
    img_w = full_gw * pw
    Kpad, K, Dm = _kpad(ph, pw), 3 * ph * pw, spec.embed_dim
    g = torch.Generator().manual_seed(ncrops * 13 + ph * 5 + pw)
    widths = [min(w, img_w) for w in _crop_widths(ncrops, pw, g)]
    # mini-batches of up to 5 crops padded to the group's widest crop (the reference's _collate); a gap of 3 token
    # rows after every crop and at the end that the kernel must not write
    descs, canvases, pix, tok = [], [], 0, 2
    for i0 in range(0, ncrops, 5):
        grp = widths[i0:i0 + 5]
        wp = (max(grp) + pw - 1) // pw * pw
        for w in grp:
            ntok = gh * (wp // pw)
            canvases.append(torch.randint(0, 256, (32, w, 3), generator=g, dtype=torch.uint8))
            descs.append((pix, w, wp, tok, ntok, i0 // 5))
            pix += 32 * w * 3
            tok += ntok + 3
    T = tok + 3
    crops = torch.cat([c.reshape(-1) for c in canvases]).to(DEV)
    drec = (_lib.YtkCrop * ncrops)(*[_lib.YtkCrop(*d) for d in descs])
    ddev = torch.frombuffer(bytearray(bytes(drec)), dtype=torch.uint8).to(DEV)
    pos = torch.randn(gh * full_gw, Dm, generator=g).to(DEV)
    A = torch.full((T, Kpad), A_SENT, dtype=torch.int16, device=DEV)
    x = torch.full((T, Dm), X_SENT, device=DEV)
    _lib.check(L().ytk_op_patchify_u8(crops.data_ptr(), ddev.data_ptr(), ncrops, ph, pw, Kpad, pos.data_ptr(), full_gw,
                                      Dm, A.data_ptr(), x.data_ptr(), None))
    torch.cuda.synchronize()

    def expected(pad_value=-1.0, cropped=True):
        eA = torch.full((T, Kpad), A_SENT, dtype=torch.int16, device=DEV)
        ex = torch.full((T, Dm), X_SENT, device=DEV)
        for (p, w, wp, t0, ntok, _), c in zip(descs, canvases):
            norm = (c.to(DEV).permute(2, 0, 1).float().div(255) - 0.5) / 0.5   # ToTensor + Normalize(0.5, 0.5)
            img = torch.full((3, 32, wp), pad_value, device=DEV)
            img[:, :, :w] = norm
            rowsA = torch.zeros((ntok, Kpad), dtype=torch.float16, device=DEV)
            rowsA[:, :K] = _patches(img, ph, pw).half()
            eA[t0:t0 + ntok] = _bits(rowsA)
            ex[t0:t0 + ntok] = _pos_rows(pos, spec, gh, wp // pw, cropped)
        return eA, ex

    eA, ex = expected()
    assert torch.equal(A, eA)
    assert torch.equal(x, ex)
    for _, _, _, t0, ntok, _ in descs:                               # zero K padding, -1 right of the canvas
        assert bool((A[t0:t0 + ntok, K:] == 0).all())
    assert bool((A.view(torch.float16) == -1).any())
    if any(w < wp for _, w, wp, *_ in descs):                        # padding value 0 instead of -1
        assert not torch.equal(A, expected(pad_value=0.0)[0])
    if any(wp // pw < full_gw and gh > 1 for _, _, wp, *_ in descs):  # pos_embed rows with the cropped grid pitch
        assert not torch.equal(x, expected(cropped=False)[1])


@pytest.mark.parametrize("model", list(PATCH))
@pytest.mark.parametrize("B,gw", [(1, 1), (5, 10), (2, None)])
def test_patchify_f32_exact(model, B, gw):
    spec = PATCH[model]
    ph, pw = spec.patch
    gh, full_gw = spec.grid
    gw = full_gw if gw is None else gw
    W = gw * pw
    Kpad, K, Dm = _kpad(ph, pw), 3 * ph * pw, spec.embed_dim
    g = torch.Generator().manual_seed(B * 17 + gw + ph)
    # normalised pixels, plus values that fp16 must round (random fp32 mantissas) and a few large ones
    images = torch.rand(B, 3, 32, W, generator=g) * 2 - 1
    images.view(-1)[::97] *= 3000.0
    images = images.to(DEV)
    pos = torch.randn(gh * full_gw, Dm, generator=g).to(DEV)
    ntok = gh * gw
    A = torch.full((B * ntok, Kpad), A_SENT, dtype=torch.int16, device=DEV)
    x = torch.full((B * ntok, Dm), X_SENT, device=DEV)
    _lib.check(L().ytk_op_patchify_f32(images.data_ptr(), B, W, ph, pw, Kpad, pos.data_ptr(), full_gw, Dm,
                                       A.data_ptr(), x.data_ptr(), None))
    torch.cuda.synchronize()
    eA = torch.zeros((B * ntok, Kpad), dtype=torch.float16, device=DEV)
    eA[:, :K] = torch.cat([_patches(images[b], ph, pw) for b in range(B)]).half()
    assert torch.equal(A, _bits(eA))
    assert torch.equal(x, _pos_rows(pos, spec, gh, gw).repeat(B, 1))
    if gw < full_gw and gh > 1:
        assert not torch.equal(x, _pos_rows(pos, spec, gh, gw, cropped=False).repeat(B, 1))


# ======================================================================================================== in situ
def _engine(cfg, spec, seed, n):
    sd = R.make_state_dict(spec, seed=seed)
    # a nonzero enc_output.proj bias: the masked rows of the invalid anchors must show it
    sd["decoder.enc_output.proj.bias"] = 0.1 * torch.randn(D, generator=torch.Generator().manual_seed(seed))
    m = RTDETRv2(cfg=to_config(cfg()))
    m.load_state_dict(sd)
    m = m.to("cuda")
    S = spec.img_size[0]
    x = torch.rand(n, 3, S, S, generator=torch.Generator().manual_seed(seed + 1))
    out = m(x.to(DEV))
    torch.cuda.synchronize()
    return dict(m=m, sd=sd, spec=spec, n=n, x=x, out={k: v.cpu() for k, v in out.items()})


@pytest.fixture(scope="module")
def layout640():
    return _engine(LayoutParserRTDETRv2V2Config, R.SPECS["layout"], 21, 3)


@pytest.fixture(scope="module")
def cell960():
    return _engine(TableCellParserRTDETRv2Config, R.RTDETRSpec(num_classes=6, num_queries=1500, img_size=[960, 960]),
                   22, 2)


@pytest.fixture(params=["layout640", "cell960"])
def run(request):
    return request.getfixturevalue(request.param)


def _dbg(run, name):
    """debug tensor of the run's batch size as fp32 (the packed inputs outgrow RTDETRv2.debug_tensor's buffer)"""
    h, n, shape = run["m"]._ensure(), run["n"], (ctypes.c_int * 4)()
    L().ytk_rtdetr_debug_tensor(h, n, name.encode(), None, 0, shape)      # refused for capacity 0, after the shape
    buf = torch.empty(math.prod(shape), dtype=torch.float32)
    _lib.check(L().ytk_rtdetr_debug_tensor(h, n, name.encode(), buf.data_ptr(), buf.numel(), shape))
    return buf.reshape(list(shape))


def test_engine_input_and_fpn_wiring(run):
    n = run["n"]
    inp = _dbg(run, "input")
    assert torch.equal(inp[..., :3], run["x"].permute(0, 2, 3, 1).half().float())
    assert bool((inp[..., 3:] == 0).all())
    cat4, cat3, pcat4, pcat5 = (_dbg(run, k) for k in ("cat4", "cat3", "pcat4", "pcat5"))
    assert torch.equal(cat4[..., :D], _nearest2(pcat5[..., D:]))
    assert torch.equal(cat3[..., :D], _nearest2(pcat4[..., D:]))
    assert not torch.equal(cat4[..., :D], _nearest2(pcat5[..., :D]))          # the other half of the PAN buffer
    fpn4 = _dbg(run, "fpn4")
    assert torch.equal(fpn4, (_dbg(run, "fpn0.t2") + _dbg(run, "fpn0.x2")).half().float())
    assert fpn4.shape[0] == n


def test_engine_aifi_position_embedding(run):
    spec, n = run["spec"], run["n"]
    g5 = spec.img_size[0] // 32
    proj5 = _dbg(run, "proj5").reshape(n, g5 * g5, D).double()
    q = _dbg(run, "aifi.q").reshape(n, g5 * g5, D)
    pos = R.sincos_2d(g5, g5, D, spec.pe_temperature)[0].double()           # row r pairs with token r (raster order)
    exact = proj5 + pos
    tol = _ulp16(exact) + 2.0 ** -21 * (1 + g5)
    worst = _ratio(q, exact, tol)
    _report("aifi.q %d images at %d" % (n, spec.img_size[0]), worst)
    assert worst <= 1.0
    wrong = proj5 + pos[_swap_grid(g5 * g5)]
    assert _ratio(q, wrong, tol) > 1.0


def test_engine_encoder_selection_wiring(run):
    spec, n, sd = run["spec"], run["n"], run["sd"]
    S = spec.img_size[0]
    shapes = [(S // s, S // s) for s in spec.strides]
    total = _offsets(shapes)[-1]
    C, K = spec.num_classes, spec.num_queries
    a = torch.arange(total).repeat(n)
    img = torch.arange(n).repeat_interleave(total)
    rows = anchor_row(shapes, n, img, a)
    # the invalid anchors' rows of enc_output.proj hold its bias, in every image
    y = _dbg(run, "enc.y").reshape(total * n, D)
    invalid = ~sd["decoder.valid_mask"].reshape(-1)
    inv_rows = rows.reshape(n, total)[:, invalid].reshape(-1)
    assert invalid.any() and torch.equal(y[inv_rows], sd["decoder.enc_output.proj.bias"].expand(len(inv_rows), D))
    # encoder scores: class max of the logits through the level-major row order
    logits = _dbg(run, "enc.logits").reshape(total * n, 8)
    scores = _dbg(run, "enc.scores").reshape(n * total)
    assert torch.equal(scores, logits[:, :C].max(1).values[rows])
    assert not torch.equal(scores, logits[:, :C].max(1).values[anchor_row(shapes, n, img, a, shift=True)])
    # the decoder starts from the anchors of the selected queries
    topk = _dbg(run, "topk").view(torch.int32).reshape(n * K).long()
    anchors = sd["decoder.anchors"].reshape(total, 4)
    assert torch.equal(_dbg(run, "anchor_sel").reshape(n * K, 4), anchors[topk])
    # the returned logits are the first C columns of the last score head
    last = _dbg(run, "logits").reshape(n * K, 8)
    assert torch.equal(run["out"]["pred_logits"].reshape(n * K, C), last[:, :C])
