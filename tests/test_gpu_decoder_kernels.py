"""GPU: op-level parity of three decoder kernels through the C ABI against float64 references on the same operands the
kernel reads (fp16-rounded values, fp32 offsets / boxes / rows):

  deformable attention   ytk_op_deform_attn_f16 (deform_attn_kernel) vs oracle.rtdetr.deformable_attention
                         |d| <= 2^-10 max|v| + 2^-11 |ref|: fp16 output rounding plus fp32 coordinate and sum error
  LayerNorm              ytk_op_layernorm_f32 (layernorm_kernel)
                         fp32 output |d| <= 1e-5 (1 + |y|) + e |gamma| (1 + |xhat|), e = 2^-20 |mean| rstd;
                         fp16 output: that plus one fp16 rounding of y (2^-11 |y| + 2^-25)
  single-query attention ytk_op_single_query_attn_f16 (single_query_attn_kernel, both modes)
                         |d| <= 2e-3 max|v|: fp16 output rounding (2^-11 |o|) plus the approximate __expf

The LayerNorm term e: fp32 arithmetic cannot place a row's mean closer than a few units in the last place of |mean|
(the kernel sums up to 1024 values in a lane-then-butterfly tree and divides once: worst case about 4 ulp), and
y = (x - mean) rstd gamma + beta carries that error times rstd.  A row with mean 1e3 and standard deviation 1e-2 has
ulp(mean) = 2^-14 and rstd = 100, so the output error is of order 1e-2 whatever the algorithm; 2^-20 |mean| (about
16 ulp) bounds it with margin.  On ordinary rows (|mean| rstd of order 1) e is below 1e-6 and 1e-5 (1 + |y|) rules.
The term is kept small enough that a one-pass fp32 variance, which loses the variance of those rows to cancellation,
still misses by more than 10x.
The fp16 check sits close to its bound by construction: rounding the exact y to fp16 alone can take the whole
2^-11 |y| (a value just above a power of two), so its worst ratio is near 1 for any correct kernel; the fp32 output of
the same call, and the equality of the fp16 output with the fp32 output rounded once, carry the tight check.

Every group also checks a plausible wrong variant of its reference - the sampling grid of align_corners=True, image 1
reading image 0's coarsest level, statistics over the padded width, eps 1e-6 instead of 1e-5, a one-pass fp32
variance E[x^2] - mean^2 on the mean-1e3 rows (which the widened LayerNorm bound must still catch), the last key dropped -
and requires the kernel to miss it by at least 10x the tolerance: a bound that loose would not catch the mistake.
"""
import ctypes

import pytest
import torch

from oracle import rtdetr as ort
from yomitoku_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENT = 7.0          # sentinel of output rows / columns the kernel must not write


def _ratio(got, want, tol):
    """max |got - want| / tol over the elements (<= 1: inside the tolerance)."""
    return ((got - want).abs() / tol).max().item()


# ======================================================================================================== deformable
SPEC = ort.RTDETRSpec()                   # 8 heads of 32 channels, 3 levels x 4 points, offset_scale 0.5
HEADS, HD = SPEC.heads, SPEC.hidden // SPEC.heads
NP = sum(SPEC.num_points)
N_OW = HEADS * NP * 3                     # offsets (x, y per point) then logits, as the engine's sampling-offset GEMM
LAYERS, LAYER = 6, 3                      # value holds the 6 decoder layers' projections side by side; read layer 3
LDOUT = HEADS * HD + 8                    # 8 sentinel columns right of the output
LAYOUT = [(80, 80), (40, 40), (20, 20)]
CELL = [(120, 120), (60, 60), (30, 30)]


def _point_sizes(shapes):
    """(NP, 2) float64: (w, h) of each point's level."""
    return torch.tensor([[w, h] for (h, w), p in zip(shapes, SPEC.num_points) for _ in range(p)], dtype=torch.float64)


def _adversarial_rows(shapes, g):
    """(ref [4], offsets [HEADS, NP, 2], logits [HEADS, NP], far) rows at the edges where grid sampling goes wrong."""
    wh = _point_sizes(shapes)
    rows = []

    def add(ref, off=None, logits=None, far=False):
        off = torch.randn(HEADS, NP, 2, generator=g, dtype=torch.float64) * 2 if off is None else off
        logits = torch.randn(HEADS, NP, generator=g, dtype=torch.float64) if logits is None else logits
        rows.append((torch.tensor(ref, dtype=torch.float32), off.float(), logits.float(), far))

    def unit_box_at(loc):
        """offsets that put the points of a unit box at the centre on `loc`: loc = 0.5 + off * (1/4) * 1 * 0.5"""
        return (loc - 0.5) * 8.0

    # boxes of size 0: every point samples the box centre, here exactly the image's corners and edges
    for ref in ([0, 0, 0, 0], [1, 1, 0, 0], [0, 1, 0, 0], [1, 0.5, 0, 0]):
        add(ref)
    # a unit box: offsets -4 / +4 land exactly on 0 / 1, mixed over heads, points and axes
    edge = torch.randint(0, 2, (HEADS, NP, 2), generator=g).double()
    add([0.5, 0.5, 1, 1], off=unit_box_at(edge))
    # pixel centres (i + 0.5) / size of each point's level: one tap carries (almost) all the weight
    for _ in range(2):
        idx = torch.floor(torch.rand(HEADS, NP, 2, generator=g, dtype=torch.float64) * wh)
        add([0.5, 0.5, 1, 1], off=unit_box_at((idx + 0.5) / wh))
    # less than one pixel outside the border (partial zero padding), on every side and in the corners
    for frac in (0.2, 0.5, 0.8, 0.99):
        side = torch.randint(0, 2, (HEADS, NP, 2), generator=g).double()
        loc = torch.where(side > 0, 1.0 + frac / wh, -frac / wh)
        add([0.5, 0.5, 1, 1], off=unit_box_at(loc))
    # far outside: the output is exactly 0
    sign = torch.randint(0, 2, (HEADS, NP, 2), generator=g).double() * 2 - 1
    add([0.5, 0.5, 1, 1], off=sign * 100.0, far=True)
    add([-3.0, 0.5, 0, 0], far=True)
    add([0.5, 4.0, 0, 0], far=True)
    # attention logits all equal, and spread over about 1e3 (the softmax is one-hot in float64)
    add([0.4, 0.6, 0.3, 0.2], logits=torch.zeros(HEADS, NP, dtype=torch.float64))
    add([0.4, 0.6, 0.3, 0.2], logits=torch.full((HEADS, NP), 7.5, dtype=torch.float64))
    spread = torch.stack([torch.linspace(-500, 500, NP, dtype=torch.float64)[torch.randperm(NP, generator=g)]
                          for _ in range(HEADS)])
    add([0.4, 0.6, 0.3, 0.2], logits=spread)
    add([0.5, 0.5, 1, 1], off=unit_box_at(torch.zeros(HEADS, NP, 2, dtype=torch.float64)), logits=spread)
    return rows


def _deform_inputs(shapes, K, n, seed):
    g = torch.Generator().manual_seed(seed)
    total = sum(h * w for h, w in shapes)
    rows = n * K
    value = torch.randn(total * n, HEADS * HD, generator=g).half()        # level-major, image-major inside a level
    ref = torch.cat([torch.rand(rows, 2, generator=g) * 0.9 + 0.05, torch.rand(rows, 2, generator=g) * 0.6 + 0.02], 1)
    ow = torch.cat([torch.randn(rows, HEADS * NP * 2, generator=g) * 2, torch.randn(rows, HEADS * NP, generator=g) * 2], 1)
    adv = _adversarial_rows(shapes, g)
    far = []
    # the adversarial rows go to the first queries of image 0 and the last queries of the last image
    for k, (r, off, logits, is_far) in enumerate(adv):
        for row in (k, rows - 1 - k):
            ref[row] = r
            ow[row, :HEADS * NP * 2] = off.reshape(-1)
            ow[row, HEADS * NP * 2:] = logits.reshape(-1)
            if is_far:
                far.append(row)
    return ow, ref, value, far


def _per_image(value, shapes, n):
    """level-major [total * n, 256] -> (n, total, HEADS, HD): level l of image i at rows off_l * n + i * h_l * w_l"""
    parts, off = [], 0
    for h, w in shapes:
        parts.append(value[off * n:(off + h * w) * n].reshape(n, h * w, HEADS * HD))
        off += h * w
    return torch.cat(parts, 1).reshape(n, off, HEADS, HD)


def _deform_ref(ow, ref, value, shapes, n, K, align_corners=False, swap_last_level=False):
    """float64 deformable attention: sampling locations and softmax as oracle.rtdetr.ms_deform_attn, sampling by
    oracle.rtdetr.deformable_attention.  Wrong variants: align_corners=True (pixel = loc * (size - 1), expressed as
    the equivalent align_corners=False location), and images 0 / 1 reading each other's coarsest level."""
    o, r = ow.double(), ref.double()
    off = o[:, :HEADS * NP * 2].reshape(n, K, HEADS, NP, 2)
    wts = torch.softmax(o[:, HEADS * NP * 2:].reshape(n, K, HEADS, NP), -1)
    scale = torch.tensor([1.0 / p for p in SPEC.num_points for _ in range(p)], dtype=torch.float64).unsqueeze(-1)
    rr = r.reshape(n, K, 1, 1, 4)
    loc = rr[..., :2] + off * scale * rr[..., 2:] * SPEC.offset_scale
    if align_corners:
        size = _point_sizes(shapes)
        loc = (loc * (size - 1) + 0.5) / size
    v = _per_image(value.double(), shapes, n)
    if swap_last_level:
        last = slice(sum(h * w for h, w in shapes[:-1]), None)
        v[0, last], v[1, last] = v[1, last].clone(), v[0, last].clone()
    return ort.deformable_attention(SPEC, v, shapes, loc, wts).reshape(n * K, HEADS * HD)


def _deform_kernel(ow, ref, value, shapes, n, K):
    L = _lib.lib()
    total = sum(h * w for h, w in shapes)
    vbuf = torch.full((total * n, LAYERS * HEADS * HD), float("nan"), dtype=torch.float16, device=DEV)
    vbuf[:, LAYER * HEADS * HD:(LAYER + 1) * HEADS * HD] = value.to(DEV)
    ow_d, ref_d = ow.to(DEV).contiguous(), ref.to(DEV).contiguous()
    out = torch.full((n * K, LDOUT), SENT, dtype=torch.float16, device=DEV)
    arr = lambda v: (ctypes.c_int * len(v))(*v)
    _lib.check(L.ytk_op_deform_attn_f16(_lib.ptr(ow_d), N_OW, _lib.ptr(ref_d), _lib.ptr(vbuf), LAYERS * HEADS * HD,
                                        LAYER * HEADS * HD, arr([h for h, _ in shapes]), arr([w for _, w in shapes]),
                                        arr(SPEC.num_points), len(shapes), n, K, HEADS, HD, SPEC.offset_scale,
                                        _lib.ptr(out), LDOUT, None))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("shapes,K,n", [(LAYOUT, 300, 1), (LAYOUT, 300, 3), (CELL, 1500, 2)],
                         ids=["layout-n1", "layout-n3", "cell-n2"])
def test_deform_attn_vs_float64(shapes, K, n):
    ow, ref, value, far = _deform_inputs(shapes, K, n, seed=K + n)
    out = _deform_kernel(ow, ref, value, shapes, n, K)
    assert (out[:, HEADS * HD:] == SENT).all()                   # nothing right of the 256 output columns
    got = out[:, :HEADS * HD].double()
    assert torch.isfinite(got).all()                             # no other layer's (NaN) columns were read
    want = _deform_ref(ow, ref, value, shapes, n, K)
    tol = 2.0 ** -10 * value.abs().max().double() + 2.0 ** -11 * want.abs()
    r = _ratio(got, want, tol)
    n_adv = len(_adversarial_rows(shapes, torch.Generator().manual_seed(0)))
    adv = list(range(n_adv)) + list(range(n * K - n_adv, n * K))
    r_adv = _ratio(got[adv], want[adv], tol[adv])
    print("[deform] %s K %d n %d: max|d| %.3g (max|v| %.3g), worst |d| / tol %.3f (adversarial rows %.3f)"
          % ("x".join(str(h) for h, _ in shapes), K, n, (got - want).abs().max().item(), value.abs().max().item(), r,
             r_adv))
    assert r <= 1.0, r
    assert (want[far] == 0).all() and (got[far] == 0).all()
    r_ac = _ratio(got, _deform_ref(ow, ref, value, shapes, n, K, align_corners=True), tol)
    print("[deform]   wrong variants: align_corners=True %.1f x tol" % r_ac)
    assert r_ac >= 10.0, r_ac
    if n >= 2:
        r_sw = _ratio(got, _deform_ref(ow, ref, value, shapes, n, K, swap_last_level=True), tol)
        print("[deform]   wrong variants: images 0 / 1 swap their coarsest level %.1f x tol" % r_sw)
        assert r_sw >= 10.0, r_sw


# ======================================================================================================== LayerNorm
EPS = 1e-5


def _ln_rows(M, D, d_real, g):
    """fp32 rows [M + 1, D] (the last row is outside the call), zero padding right of d_real.  Row kinds by row % 5:
    ordinary, mean 1e3 / std 1e-2 (cancellation), constant 0.5 (exact fp32 sums), near-constant (std 1e-3: eps
    matters), wide (std 100)."""
    x = torch.zeros(M + 1, D, dtype=torch.float64)
    z = torch.randn(M + 1, d_real, generator=g, dtype=torch.float64)
    kind = torch.arange(M + 1) % 5
    scale = torch.rand(M + 1, 1, generator=g, dtype=torch.float64) * 2.5 + 0.5
    shift = torch.randn(M + 1, 1, generator=g, dtype=torch.float64)
    x[:, :d_real] = torch.where((kind == 0)[:, None], z * scale + shift, x[:, :d_real])
    x[:, :d_real] = torch.where((kind == 1)[:, None], 1e3 + 1e-2 * z, x[:, :d_real])
    x[:, :d_real] = torch.where((kind == 2)[:, None], torch.full_like(z, 0.5), x[:, :d_real])
    x[:, :d_real] = torch.where((kind == 3)[:, None], 0.5 + 1e-3 * z, x[:, :d_real])
    x[:, :d_real] = torch.where((kind == 4)[:, None], 100.0 * z, x[:, :d_real])
    return x.float(), kind[:M]


def _ln_ref(x, d_real, gamma, beta, eps=EPS, stats_width=None):
    """float64 LayerNorm of fp32 rows; stats_width = D is the wrong variant that averages over the padding too."""
    x = x.double()
    n = d_real if stats_width is None else stats_width
    mean = x[:, :n].mean(1, keepdim=True)
    var = ((x[:, :n] - mean) ** 2).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    xhat = torch.zeros_like(x)
    xhat[:, :d_real] = (x[:, :d_real] - mean) * rstd
    y = xhat * gamma.double() + beta.double()
    tol = 1e-5 * (1 + y.abs()) + 2.0 ** -20 * mean.abs() * rstd * gamma.double().abs() * (1 + xhat.abs())
    return y, tol


def _ln_one_pass_f32(x, d_real, gamma, beta, eps=EPS):
    """The wrong variant for cancellation: fp32 one-pass variance E[x^2] - mean^2 (clamped at 0, as such code does)."""
    xr = x[:, :d_real].float()
    mean = xr.sum(1, keepdim=True) / d_real
    var = ((xr * xr).sum(1, keepdim=True) / d_real - mean * mean).clamp(min=0.0)
    y = torch.zeros(x.shape, dtype=torch.float64)
    y[:, :d_real] = ((xr - mean) * torch.rsqrt(var + eps) * gamma[:d_real] + beta[:d_real]).double()
    return y


def _ln_kernel(x, M, D, d_real, gamma, beta, f16, f32, addvec=None, period=1, row0_dev=None, row0=0, writeback=0,
               eps=EPS):
    L = _lib.lib()
    xd = x.to(DEV).contiguous()
    o16 = torch.full((M + 1, D), SENT, dtype=torch.float16, device=DEV) if f16 else None
    o32 = torch.full((M + 1, D), SENT, dtype=torch.float32, device=DEV) if f32 else None
    r0 = torch.tensor([row0_dev], dtype=torch.int32, device=DEV) if row0_dev is not None else None
    _lib.check(L.ytk_op_layernorm_f32(_lib.ptr(xd), M, D, d_real, _lib.ptr(gamma), _lib.ptr(beta), eps, _lib.ptr(o16),
                                      _lib.ptr(o32), _lib.ptr(addvec), period, _lib.ptr(r0), row0, writeback, None))
    torch.cuda.synchronize()
    return xd.cpu(), None if o16 is None else o16.cpu(), None if o32 is None else o32.cpu()


@pytest.mark.parametrize("M", [1, 7, 8, 9, 900, 4097])
@pytest.mark.parametrize("D,d_real", [(256, 256), (384, 368), (512, 512), (768, 768), (1024, 1024)])
def test_layernorm_vs_float64(D, d_real, M):
    g = torch.Generator().manual_seed(D * 10007 + M)
    x, kind = _ln_rows(M, D, d_real, g)
    gamma = torch.zeros(D)
    beta = torch.zeros(D)
    gamma[:d_real] = 1.0 + 0.3 * torch.randn(d_real, generator=g)
    beta[:d_real] = 0.3 * torch.randn(d_real, generator=g)
    table = torch.zeros(5, D)
    table[:, :d_real] = 0.5 * torch.randn(5, d_real, generator=g)
    gd, bd, td = gamma.to(DEV), beta.to(DEV), table.to(DEV)
    worst32 = worst16 = 0.0
    # (outputs, addvec period, first table row from the device / as a value, writeback)
    runs = [("f32", 0, None, 0, 0), ("f16", 0, None, 0, 0), ("both", 0, None, 0, 0), ("both", 3, None, 2, 0),
            ("both", 3, 2, 0, 1), ("f16", 1, 1, 0, 1)]
    for outs, period, row0_dev, row0, wb in runs:
        if period:
            r0 = row0_dev if row0_dev is not None else row0
            xin = x.clone()
            xin[:M] = x[:M] + table[(torch.arange(M) % period) + r0]   # fp32 adds, as the kernel's
        else:
            xin = x
        xo, o16, o32 = _ln_kernel(x, M, D, d_real, gd, bd, outs != "f32", outs != "f16", td if period else None,
                                  max(period, 1), row0_dev, row0, wb)
        assert torch.equal(xo, xin if wb else x)                     # writeback stores exactly x + addvec, else x stays
        y, tol = _ln_ref(xin[:M], d_real, gamma, beta)
        if o32 is not None:
            assert (o32[M] == SENT).all()
            assert (o32[:M, d_real:] == 0).all()
            r = _ratio(o32[:M].double(), y, tol)
            worst32 = max(worst32, r)
            assert r <= 1.0, (outs, period, row0_dev, row0, wb, r)
        if o16 is not None:
            assert (o16[M] == SENT).all()
            assert (o16[:M, d_real:] == 0).all()
            r = _ratio(o16[:M].double(), y, tol + 2.0 ** -11 * y.abs() + 2.0 ** -25)
            worst16 = max(worst16, r)
            assert r <= 1.0, (outs, period, row0_dev, row0, wb, r)
        if o16 is not None and o32 is not None:
            assert torch.equal(o16[:M], o32[:M].half())              # one y, rounded once
        if not period:
            const = kind == 2                                        # constant rows: x - mean is exactly 0
            if o32 is not None:
                assert (o32[:M][const] == beta).all()
            if o16 is not None:
                assert (o16[:M][const] == beta.half()).all()
        if outs == "f32" and not period:
            if d_real < D:
                y_w, _ = _ln_ref(x[:M], d_real, gamma, beta, stats_width=D)
                r_w = _ratio(o32[:M].double(), y_w, tol)
                print("[layernorm]   wrong variant: statistics over D %.1f x tol" % r_w)
                assert r_w >= 10.0, r_w
            near = kind == 3
            if near.any():
                y_e, _ = _ln_ref(x[:M], d_real, gamma, beta, eps=1e-6)
                r_e = _ratio(o32[:M][near].double(), y_e[near], tol[near])
                print("[layernorm]   wrong variant: eps 1e-6 on near-constant rows %.1f x tol" % r_e)
                assert r_e >= 10.0, r_e
            far_mean = kind == 1
            if far_mean.any():
                y_1 = _ln_one_pass_f32(x[:M], d_real, gamma, beta)[far_mean]
                r_1 = _ratio(o32[:M][far_mean].double(), y_1, tol[far_mean])
                print("[layernorm]   wrong variant: one-pass fp32 variance on mean-1e3 rows %.1f x tol" % r_1)
                assert r_1 >= 10.0, r_1
    print("[layernorm] D %d d_real %d M %d: worst |d| / tol fp32 %.3f, fp16 %.3f" % (D, d_real, M, worst32, worst16))


# ======================================================================================================== AR attention
# (head dim, heads): every LPK / CPL / NSUB instantiation of single_query_attn_kernel (hd 32: 4 lanes per key, 8 key
# subsets; hd 48 = padded parseq-tiny: 2 lanes, 16 subsets; hd 64 / 96: 4 lanes, 2 / 3 chunks each), and head counts
# that leave B * heads odd, so the last CTA has idle warps
SQA_CFGS = [(32, 8), (48, 8), (64, 12), (96, 8), (48, 7), (32, 5)]


def _sqa_ref(q, k, v, heads, drop_last=False):
    """float64 softmax attention of one query row per row of a batch: q (R, D), k / v (R, nk, D) -> (R, D)."""
    q, k, v = q.double(), k.double(), v.double()
    if drop_last:
        k, v = k[:, :-1], v[:, :-1]
    R, nk, D = k.shape
    hd = D // heads
    s = torch.einsum("rjhd,rhd->rhj", k.reshape(R, nk, heads, hd), q.reshape(R, heads, hd)) / hd ** 0.5
    return torch.einsum("rhj,rjhd->rhd", torch.softmax(s, -1), v.reshape(R, nk, heads, hd)).reshape(R, D)


def _sqa_kernel(mode, q, kv, B, S, D, heads, step=None, crops=None):
    L = _lib.lib()
    out = torch.full((B + 3, D), SENT, dtype=torch.float16, device=DEV)
    step_dev = torch.tensor([step], dtype=torch.int32, device=DEV) if step is not None else None
    _lib.check(L.ytk_op_single_query_attn_f16(mode, _lib.ptr(q), _lib.ptr(kv), B, S, D, heads, _lib.ptr(step_dev), crops,
                                              _lib.ptr(out), None))
    torch.cuda.synchronize()
    out = out.cpu()
    assert (out[B:] == SENT).all()                                   # rows outside B are not written
    return out[:B].double()


@pytest.mark.parametrize("hd,heads", SQA_CFGS)
def test_single_query_self_attn_vs_float64(hd, heads):
    """mode 0: AR step i, query q[i] against keys 0..i of each row's cache; steps at and around every key-subset
    boundary.  Cache positions after the step hold NaN: they must not be read."""
    S, B = 26, 13
    D = hd * heads
    g = torch.Generator().manual_seed(hd * 100 + heads)
    worst, drop = 0.0, float("inf")
    for qscale in (1.0, 6.0):                                       # 6: scores spread over about +-30
        q = (torch.randn(S, D, generator=g) * qscale).half()
        ckv = torch.randn(B, S, 2 * D, generator=g).half()
        vmax = ckv[:, :, D:].abs().max().double()
        for step in (0, 1, 7, 8, 9, 15, 16, 17, S - 1):
            cache = ckv.clone()
            cache[:, step + 1:] = float("nan")
            got = _sqa_kernel(0, q.to(DEV), cache.to(DEV), B, S, D, heads, step=step)
            k, v = ckv[:, :step + 1, :D], ckv[:, :step + 1, D:]
            qi = q[step].expand(B, D)
            want = _sqa_ref(qi, k, v, heads)
            r = (got - want).abs().max().item() / (2e-3 * vmax.item())
            worst = max(worst, r)
            assert r <= 1.0, (qscale, step, r)
            if step >= 1:
                r_d = (got - _sqa_ref(qi, k, v, heads, drop_last=True)).abs().max().item() / (2e-3 * vmax.item())
                drop = min(drop, r_d)
                assert r_d >= 10.0, (qscale, step, r_d)
    print("[sq-attn self] hd %d heads %d: worst |d| / tol %.3f; last key dropped: smallest miss over the steps %.0f x tol"
          % (hd, heads, worst, drop))


@pytest.mark.parametrize("hd,heads", SQA_CFGS)
def test_single_query_cross_attn_vs_float64(hd, heads):
    """mode 1: each row's query against its crop's encoder memory, ragged lengths up to the engine's 800 tokens in one
    call.  Three NaN rows separate the crops: a read past ntok shows.

    The dropped-last-key check takes the largest miss over the crops of a call, so the short crops decide it: on the
    799- and 800-token crops the last key weighs about 1/800 and dropping it stays inside 2e-3 max|v|.  Reads past the
    end of a long crop are caught by the NaN rows instead; mode 0 runs the check at every step."""
    ntoks = [1, 7, 8, 16, 17, 100, 799, 800, 33, 5, 250]
    B, D, gap = len(ntoks), hd * heads, 3
    g = torch.Generator().manual_seed(hd * 100 + heads + 1)
    crops = (_lib.YtkCrop * B)()
    offs, T = [], gap
    for i, n in enumerate(ntoks):
        offs.append(T)
        crops[i] = _lib.YtkCrop(0, 0, 0, T, n, 0)
        T += n + gap
    worst = 0.0
    for qscale in (1.0, 6.0):
        q = (torch.randn(B, D, generator=g) * qscale).half()
        mem = torch.full((T, 2 * D), float("nan")).half()
        for o, n in zip(offs, ntoks):
            mem[o:o + n] = torch.randn(n, 2 * D, generator=g).half()
        vmax = max(mem[o:o + n, D:].abs().max().item() for o, n in zip(offs, ntoks))
        got = _sqa_kernel(1, q.to(DEV), mem.to(DEV), B, 0, D, heads, crops=crops)
        r_drop = 0.0
        for i, (o, n) in enumerate(zip(offs, ntoks)):
            k, v = mem[o:o + n, :D][None], mem[o:o + n, D:][None]
            want = _sqa_ref(q[i:i + 1], k, v, heads)
            r = (got[i:i + 1] - want).abs().max().item() / (2e-3 * vmax)
            worst = max(worst, r)
            assert r <= 1.0, (qscale, n, r)
            if n >= 2:
                r_drop = max(r_drop, (got[i:i + 1] - _sqa_ref(q[i:i + 1], k, v, heads, drop_last=True)).abs().max().item()
                             / (2e-3 * vmax))
        print("[sq-attn cross] hd %d heads %d qscale %g: last key dropped %.0f x tol" % (hd, heads, qscale, r_drop))
        assert r_drop >= 10.0, r_drop
    print("[sq-attn cross] hd %d heads %d: worst |d| / tol %.3f" % (hd, heads, worst))
