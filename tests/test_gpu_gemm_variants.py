"""GPU: every gemm_tc_kernel instance the plans pick, element by element against float64.

The kernel is gemm_tc_kernel<BLOCK_N, OUT_F32, RESID, MODE, DIRECT>; finish_plan picks the instance from the shape and
the number of SMs.  Each case here reaches its instance by shape alone and reads which one ran from the YTK_GEMM_DUMP
record of its own profiling window (block_n, out_f32, resid, mode, act, epi = 1 TMA / 0 staged, bw_log2).

Reference: A W^T + bias + residual in float64 on the device, from the exact 16-bit operands the kernel reads, then the
exact activation (erf GELU, 1 / (1 + e^-x), x / (1 + e^-x)).  Bound, per element:

    |got - ref| <= L_act e_pre + e_act + u_out (|ref| + L_act e_pre + e_act) + a_out

  e_pre = gamma_{K} S + 2^-23 (S + |bias| + |resid|),   S = sum_k |a_k w_k| (float64),   gamma_n = n u / (1 - n u)
        with u = 2^-23.  A product of two fp16 operands has at most 22 significant bits, so it is exact in fp32.  The
        tensor core adds the K products into the fp32 accumulator; each addition is assumed correct to one unit in the
        last place of a 24-bit significand, as truncation (not rounding to nearest) gives, relative to the larger of the
        running sum and the addend, both at most S.  At most K such additions give gamma_K S.  The bias and residual
        additions are IEEE fp32 additions (2^-24 of a result no larger than S + |bias| + |resid|, two of them).
  L_act = the largest |derivative| of the activation: 1 (none, ReLU), 1.13 (GELU, 1.1289 at x = sqrt 2), 0.25
        (sigmoid), 1.1 (SiLU, 1.0998 at x = 2.40).
  e_act = the error of the activation as evaluated in fp32: GELU: 5e-7 (gelu_fast's documented maximum) + 2^-24 |ref|
        (its final fma).  Sigmoid and SiLU: __expf(-x) is within 2 + floor(1.173 |x|) units of 2^-23 relative (CUDA
        programming guide, intrinsic functions), which reaches 1 / (1 + E) scaled by E / (1 + E) = 1 - s; the addition
        1 + E adds 2^-24 and __fdividef 2 units of 2^-23, so relative to |ref|: 2^-23 ((1 - s)(2 + 1.173 |x|) + 3).
  u_out = 2^-11 (fp16 output, rounded to nearest) or 2^-24 (fp32); a_out = 2^-25 for fp16 (half the subnormal spacing).

fp16 outputs also pass a sharper test: the conversion is monotone, so the stored value lies between the fp16 values
nearest to ref - e and ref + e (e = L_act e_pre + e_act).  Away from a rounding midpoint that is exactly the fp16 value
nearest to ref.

Around every output the test keeps guards filled with a NaN bit pattern and compares them bitwise afterwards: at least
129 rows past the last row, the columns from Cout to the pitch and, where a case writes at a column offset (a concat
half), the columns before it.  A, W, bias and the residual (unless it is the output) must be bitwise unchanged.

Wrong variants of the reference (a dropped K block, a shifted bias column, a residual row off by one, tanh-GELU,
sigmoid for SiLU, truncated fp16 output) must miss the bound by at least 10x on some element: the bound is tight
enough to see each of them."""
import csv
import os

import pytest
import torch
import torch.nn.functional as F

from yomitoku_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

U23, U24, U11 = 2.0 ** -23, 2.0 ** -24, 2.0 ** -11
LIP = {0: 1.0, 1: 1.0, 2: 1.13, 3: 0.25, 4: 1.1}
GELU_ERR = 5e-7
GUARD_ROWS = 129
NAN16, NAN32 = 0x7E5A, 0x7FA5A5A5          # quiet NaNs with a payload no kernel computes
ACT_NAMES = {0: "none", 1: "relu", 2: "gelu", 3: "sigmoid", 4: "silu"}

_DUMP = {}          # path of the dump file of the current profiling window
_RESULTS = {}       # case -> per-act results (a case runs once per process)
_CHECKED = set()    # (block_n, out_f32, resid, mode, act, epi) of every launch checked against float64
_RATIOS = {}        # group -> largest error / bound


@pytest.fixture(scope="module", autouse=True)
def _dump_path(tmp_path_factory):
    _DUMP["path"] = str(tmp_path_factory.mktemp("gemm_dump") / "dump.csv")
    yield
    for group, r in sorted(_RATIOS.items()):
        print("[gemm variants] %-34s max error / bound %.3g" % (group, r))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _launches(fn):
    """Runs fn inside a gemm profiling window and returns the dump records of the launches it made."""
    L = _lib.lib()
    path = _DUMP["path"]
    if os.path.exists(path):
        os.remove(path)
    old = os.environ.get("YTK_GEMM_DUMP")
    os.environ["YTK_GEMM_DUMP"] = path           # read by every ytk_gemm_profile_end
    try:
        L.ytk_gemm_profile_begin()
        try:
            fn()
        finally:
            _lib.check(L.ytk_gemm_profile_end(None, None, None))
    finally:
        if old is None:
            del os.environ["YTK_GEMM_DUMP"]
        else:
            os.environ["YTK_GEMM_DUMP"] = old
    if not os.path.exists(path):
        return []
    with open(path) as f:
        rows = [r for r in csv.DictReader(l for l in f if not l.startswith("pixels") or "cout" in l)
                if r["pixels"] != "pixels"]
    return [{k: (float(v) if k in ("flops", "ms") else int(v)) for k, v in r.items()} for r in rows]


def _instance(r):
    return (r["block_n"], r["out_f32"], r["resid"], r["mode"], r["act"], r["epi"])


# ------------------------------------------------------------------------------------------------ reference and bound
def _act(x, act):
    if act == 1:
        return x.clamp(min=0)
    if act == 2:
        return 0.5 * x * (1 + torch.erf(x / 2 ** 0.5))
    if act == 3:
        return torch.sigmoid(x)
    if act == 4:
        return x * torch.sigmoid(x)
    return x


def _inner(pre, e_pre, act, y):
    """Error of the fp32 value before the output rounding: L_act e_pre + e_act."""
    if act == 2:
        e_act = GELU_ERR + U24 * y.abs()
    elif act in (3, 4):
        s = torch.sigmoid(pre)
        e_act = y.abs() * U23 * ((1 - s) * (2 + 1.173 * (pre.abs() + e_pre)) + 3)
    else:
        e_act = 0.0
    return LIP[act] * e_pre + e_act


def _fp16_grid(t, mode):
    """float64 -> the fp16 value rounded to nearest-even ("rn") or toward zero ("rz"), exactly, as float64."""
    _, e = torch.frexp(t)                                      # t = m 2^e, 0.5 <= |m| < 1
    ulp = torch.ldexp(torch.ones_like(t), (e - 11).clamp(min=-24))
    q = t / ulp
    return (torch.round(q) if mode == "rn" else torch.trunc(q)) * ulp


def _ratio(got, y, inner, of32):
    """Largest |got - ref| / bound (NaN if any output is NaN)."""
    u = U24 if of32 else U11
    bound = inner + u * (y.abs() + inner) + (0.0 if of32 else 2.0 ** -25)
    return ((got - y).abs() / bound).max().item()


def _rounding_ratio(got, y, inner, mode="rn"):
    """fp16 outputs: |got - R(ref)| over the spread of R over [ref - inner, ref + inner] (R = the rounding) + inner."""
    inner = inner * (1 + 1e-9) + 1e-300
    r = _fp16_grid(y, mode)
    spread = torch.maximum((_fp16_grid(y + inner, mode) - r).abs(), (_fp16_grid(y - inner, mode) - r).abs())
    return ((got - r).abs() / (spread + inner)).max().item()


def _e_pre(K, S, extra):
    return K * U23 / (1 - K * U23) * S + U23 * (S + extra)


def _assert_close(tag, group, K, pre, S, extra, act, got, of32):
    y = _act(pre, act)
    inner = _inner(pre, _e_pre(K, S, extra), act, y)
    r = _ratio(got, y, inner, of32)
    _RATIOS[group] = max(_RATIOS.get(group, 0.0), r)
    assert r <= 1.0, "%s act %s: error / bound %.3g" % (tag, ACT_NAMES[act], r)
    if not of32:
        rr = _rounding_ratio(got, y, inner)
        assert rr <= 1.0, "%s act %s: fp16 output is not the rounded reference (%.3g)" % (tag, ACT_NAMES[act], rr)


# ------------------------------------------------------------------------------------------------ buffers and guards
def _guarded(rows, ld, f32):
    t = torch.empty((rows + GUARD_ROWS, ld), device=DEV, dtype=torch.float32 if f32 else torch.float16)
    t.view(torch.int32 if f32 else torch.int16).fill_(NAN32 if f32 else NAN16)
    return t


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _check_guards(tag, buf, before, rows, coff, n):
    """Everything of buf outside rows [0, rows) x columns [coff, coff + n) holds its old bits."""
    keep = torch.ones(buf.shape, dtype=torch.bool, device=DEV)
    keep[:rows, coff:coff + n] = False
    changed = (_bits(buf) != _bits(before)) & keep
    if changed.any():
        r, c = changed.nonzero()[0].tolist()
        raise AssertionError("%s: guard element (%d, %d) was written (output rows %d, columns [%d, %d))"
                             % (tag, r, c, rows, coff, coff + n))


def _up(x, a):
    return (x + a - 1) // a * a


# ------------------------------------------------------------------------------------------------ linear cases
def _linear_case(M, K, N, of32, resid=0, acts=(0,), lda=None, coff=0, ldc=None, ldr=None, bias=True, in_place=False,
                 a_scale=0.5, b_scale=1.0, seed=0):
    """Runs ytk_op_linear_f16 once per activation on one operand set; returns the float64 reference terms and, per
    activation, the output and the dump records of its launch.  Guards and operands are checked here."""
    key = ("linear", M, K, N, of32, resid, tuple(acts), lda, coff, ldc, ldr, bias, in_place, a_scale, b_scale, seed)
    if key in _RESULTS:
        return _RESULTS[key]
    L = _lib.lib()
    g = torch.Generator(device=DEV).manual_seed(seed * 7919 + M + 31 * N + K)
    lda = lda or K
    es = 4 if of32 else 2
    ldc = ldc or (coff + _up(N, 16 // es) + 16 // es)              # sentinel columns past Cout
    A = (torch.randn(M, lda, generator=g, device=DEV) * a_scale).half()
    W = (torch.randn(N, K, generator=g, device=DEV) / K ** 0.5).half()
    b = (torch.randn(N, generator=g, device=DEV) * b_scale) if bias else None
    R = None
    rf32 = 1 if resid == 2 else 0
    if in_place:
        assert resid == (2 if of32 else 1)
        ldr = ldc
        R_vals = torch.randn(M, N, generator=g, device=DEV).to(torch.float32 if of32 else torch.float16)
    elif resid:
        res = 4 if resid == 2 else 2
        ldr = ldr or (_up(N, 16 // res) + 2 * (16 // res))
        R = torch.randn(M, ldr, generator=g, device=DEV).to(torch.float32 if resid == 2 else torch.float16)
        R_vals = R[:, :N]
    a64 = A[:, :K].double()
    w64 = W.double()
    pre = a64 @ w64.t()
    S = a64.abs() @ w64.abs().t()
    extra = torch.zeros_like(pre)
    if b is not None:
        pre = pre + b.double()
        extra = extra + b.double().abs()
    if resid:
        r64 = R_vals.double()
        pre = pre + r64
        extra = extra + r64.abs()
    snap = [t.clone() for t in (A, W, b, R) if t is not None]
    out = {}
    for act in acts:
        buf = _guarded(M, ldc, of32)
        if in_place:
            buf[:M, coff:coff + N] = R_vals
        before = buf.clone()
        optr = buf.data_ptr() + coff * es
        rptr = optr if in_place else _lib.ptr(R)
        recs = _launches(lambda: _lib.check(L.ytk_op_linear_f16(
            _lib.ptr(A), lda, M, K, _lib.ptr(W), N, _lib.ptr(b), rptr, rf32, ldr or 0, optr, 1 if of32 else 0, ldc, act,
            None)))
        torch.cuda.synchronize()
        tag = "linear M %d K %d N %d out %s resid %d act %d" % (M, K, N, "f32" if of32 else "f16", resid, act)
        _check_guards(tag, buf, before, M, coff, N)
        out[act] = (buf[:M, coff:coff + N].double(), recs)
    for t, s in zip([t for t in (A, W, b, R) if t is not None], snap):
        assert torch.equal(_bits(t) if t.dtype != torch.float32 else t.view(torch.int32),
                           _bits(s) if s.dtype != torch.float32 else s.view(torch.int32)), "an operand changed"
    res = dict(K=K, pre=pre, S=S, extra=extra, out=out, A=A, W=W, b=b, R_vals=R_vals if resid else None, of32=of32)
    _RESULTS[key] = res
    return res


def _check_linear(group, res, tag, expect=None, mode=0):
    for act, (got, recs) in res["out"].items():
        assert len(recs) == 1, recs
        r = recs[0]
        if expect is not None:
            got_inst = (r["block_n"], r["out_f32"], r["resid"], r["epi"])
            assert got_inst == expect, "%s act %d reached %s, not %s" % (tag, act, got_inst, expect)
        _assert_close(tag, group, res["K"], res["pre"], res["S"], res["extra"], act, got, res["of32"])
        _CHECKED.add(_instance(r))


def _instance_cases():
    """The 30 EPI_NORMAL instances (block_n, out_f32, resid, epi) and a shape that reaches each.  N tile: Cout <= 64 ->
    64, <= 128 -> 128, 264 / 250 -> 256 (pick_block_n), kept only with at least one tile per SM (the shrink rule).
    Staged path for matching types: Cout x element size not a multiple of 16 bytes."""
    big = 128 * _sms() + 77                                       # one more M tile than SMs
    shapes = {64: (300, {1: 40, 0: 42}), 128: (big, {1: 120, 0: 122}), 256: (big, {1: 264, 0: 250})}
    cases = []
    i = 0
    for bn in (64, 128, 256):
        M, ncols = shapes[bn]
        for of32 in (0, 1):
            for resid in (0, 1, 2):
                matching = resid == 0 or (resid == 2) == (of32 == 1)
                for epi in ((1, 0) if matching else (0,)):
                    K = (64, 128, 192)[i % 3]
                    coff = (0, 16 // (4 if of32 else 2))[i % 2]
                    cases.append(((bn, of32, resid, epi), dict(M=M, K=K, N=ncols[epi], of32=of32, resid=resid,
                                                               coff=coff, seed=i)))
                    i += 1
    return cases


def _instance_ids():
    return ["bn%d-%s-r%d-%s" % (bn, "f32" if of32 else "f16", r, "tma" if epi else "staged")
            for bn in (64, 128, 256) for of32 in (0, 1) for r in (0, 1, 2)
            for epi in ((1, 0) if (r == 0 or (r == 2) == (of32 == 1)) else (0,))]


@pytest.mark.parametrize("idx", range(30), ids=_instance_ids())
def test_linear_instance_all_activations(idx):
    inst, kw = _instance_cases()[idx]
    res = _linear_case(acts=(0, 1, 2, 3, 4), **kw)
    _check_linear("linear %s / %s" % ("f32" if inst[1] else "f16", "tma" if inst[3] else "staged"), res,
                  "instance %s" % (inst,), expect=inst)


def test_every_linear_instance_reached():
    reached = set()
    for inst, kw in _instance_cases():
        for _, recs in _linear_case(acts=(0, 1, 2, 3, 4), **kw)["out"].values():
            reached |= {(r["block_n"], r["out_f32"], r["resid"], r["epi"]) for r in recs}
    want = {inst for inst, _ in _instance_cases()}
    assert len(want) == 30
    missing = sorted(want - reached)
    assert not missing, "instances (block_n, out_f32, resid, epi) never launched: %s" % missing


# M = 1 / 127 / 129, a ragged M with several tiles per CTA, K = 64, lda > K, no bias, in-place residuals
EDGE_LINEAR = [
    dict(M=1, K=64, N=64, of32=0, acts=(0, 4)), dict(M=1, K=128, N=100, of32=1, resid=2, acts=(2,)),
    dict(M=127, K=64, N=72, of32=0, resid=1, acts=(1, 3)), dict(M=129, K=192, N=264, of32=1, acts=(0, 4)),
    dict(M=129, K=64, N=42, of32=0, resid=2, acts=(2,)),
    dict(M=128 * 400 + 3, K=64, N=64, of32=0, resid=1, acts=(1,)),
    dict(M=128 * 300 + 77, K=128, N=250, of32=1, acts=(0,)),
    dict(M=300, K=128, N=200, of32=0, lda=200, acts=(0, 2)), dict(M=1000, K=64, N=120, of32=1, lda=72, resid=2, acts=(4,)),
    dict(M=517, K=128, N=200, of32=0, bias=False, acts=(0, 3)), dict(M=517, K=64, N=122, of32=1, bias=False, resid=1,
                                                                     acts=(4,)),
    dict(M=128 * 90 + 17, K=256, N=256, of32=1, resid=2, in_place=True, acts=(0,)),
    dict(M=128 * 90 + 17, K=256, N=256, of32=0, resid=1, in_place=True, acts=(0, 1)),
    dict(M=300, K=128, N=42, of32=0, resid=1, in_place=True, acts=(0,)),
]


@pytest.mark.parametrize("kw", EDGE_LINEAR, ids=["edge%d" % i for i in range(len(EDGE_LINEAR))])
def test_linear_edges(kw):
    _check_linear("linear edges", _linear_case(**kw), "edge %s" % kw)


# ------------------------------------------------------------------------------------------------ convolution cases
def _conv_case(n, H, W, Cin, Cout, k, s, p, d, acts=(0,), in_ld=None, of32=0, resid=0, coff=0, ldc=None, mode=0,
               a_scale=0.5, seed=0):
    key = ("conv", n, H, W, Cin, Cout, k, s, p, d, tuple(acts), in_ld, of32, resid, coff, ldc, mode, seed)
    if key in _RESULTS:
        return _RESULTS[key]
    L = _lib.lib()
    g = torch.Generator(device=DEV).manual_seed(seed * 7919 + H * W + Cout)
    in_ld = in_ld or Cin
    es = 4 if of32 else 2
    x = (torch.randn(n, H, W, in_ld, generator=g, device=DEV) * a_scale).half()
    w = (torch.randn(Cout, Cin, k, k, generator=g, device=DEV) / (Cin * k * k) ** 0.5).half()
    wp = w.permute(0, 2, 3, 1).contiguous()
    b = torch.randn(Cout, generator=g, device=DEV)
    Ho = (H + 2 * p - d * (k - 1) - 1) // s + 1
    Wo = (W + 2 * p - d * (k - 1) - 1) // s + 1
    x64 = x[..., :Cin].double().permute(0, 3, 1, 2)
    pre = F.conv2d(x64, w.double(), b.double(), stride=s, padding=p, dilation=d).permute(0, 2, 3, 1)
    S = F.conv2d(x64.abs(), w.double().abs(), stride=s, padding=p, dilation=d).permute(0, 2, 3, 1)
    extra = b.double().abs().expand_as(pre)
    if mode == 1:          # 2x2 pixel shuffle: column block (i, j) of width Cout / 4 -> pixel (2h + i, 2w + j)
        shuf = lambda t: t.reshape(n, Ho, Wo, 2, 2, Cout // 4).permute(0, 1, 3, 2, 4, 5).reshape(n * 4 * Ho * Wo, -1)
        pre, S, extra = shuf(pre), shuf(S), shuf(extra)
        rows, width = n * 4 * Ho * Wo, Cout // 4
    else:
        pre, S, extra = pre.reshape(-1, Cout), S.reshape(-1, Cout), extra.reshape(-1, Cout)
        rows, width = n * Ho * Wo, Cout
    ldc = ldc or (coff + _up(width, 16 // es) + 16 // es)
    R, rf32, ldr = None, 0, 0
    if resid:
        rf32 = 1 if resid == 2 else 0
        ldr = _up(Cout, 8) + 8
        R = torch.randn(rows, ldr, generator=g, device=DEV).to(torch.float32 if rf32 else torch.float16)
        pre = pre + R[:, :Cout].double()
        extra = extra + R[:, :Cout].double().abs()
    snap = [t.clone() for t in (x, wp, b, R) if t is not None]
    out = {}
    for act in acts:
        buf = _guarded(rows, ldc, of32)
        before = buf.clone()
        optr = buf.data_ptr() + coff * es
        recs = _launches(lambda: _lib.check(L.ytk_op_conv2d_f16(
            _lib.ptr(x), n, H, W, Cin, in_ld, _lib.ptr(wp), _lib.ptr(b), k, k, s, p, d, Cout, _lib.ptr(R), rf32, ldr,
            optr, of32, ldc, act, mode, None)))
        torch.cuda.synchronize()
        tag = "conv n %d %dx%d Cin %d Cout %d k %d s %d d %d mode %d act %d" % (n, H, W, Cin, Cout, k, s, d, mode, act)
        _check_guards(tag, buf, before, rows, coff, width)
        out[act] = (buf[:rows, coff:coff + width].double(), recs)
    for t, sn in zip([t for t in (x, wp, b, R) if t is not None], snap):
        assert torch.equal(t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32),
                           sn.view(torch.int16) if sn.dtype == torch.float16 else sn.view(torch.int32)), "operand changed"
    res = dict(K=Cin * k * k, pre=pre, S=S, extra=extra, out=out, of32=of32)
    _RESULTS[key] = res
    return res


# (n, H, W, Cin, Cout, k, s, p, d) + options; bw = the tile patch (BW = 1 << bw_log2) pick_bw_log2 chooses
CONV = [
    (dict(n=2, H=40, W=8, Cin=64, Cout=96, k=3, s=1, p=1, d=1, acts=(1,), resid=1), 3),
    (dict(n=1, H=9, W=16, Cin=64, Cout=64, k=3, s=1, p=1, d=1, acts=(0, 4)), 4),
    (dict(n=3, H=13, W=30, Cin=128, Cout=40, k=1, s=1, p=0, d=1, acts=(4,), resid=1, coff=8), 5),
    (dict(n=2, H=7, W=60, Cin=64, Cout=128, k=1, s=1, p=0, d=1, acts=(1, 4), of32=1), 6),
    (dict(n=1, H=2, W=120, Cin=64, Cout=64, k=3, s=1, p=1, d=1, acts=(4,), of32=1, resid=2), 7),
    # stride 2 at odd H and W, dilation 2, input channel pitch > Cin, images whose last patch row sticks out
    (dict(n=1, H=37, W=51, Cin=64, Cout=128, k=3, s=2, p=1, d=1, acts=(1, 4)), None),
    (dict(n=1, H=37, W=50, Cin=128, Cout=128, k=3, s=1, p=2, d=2, acts=(4,), resid=1), None),
    (dict(n=2, H=20, W=24, Cin=64, in_ld=88, Cout=64, k=3, s=1, p=1, d=1, acts=(1,)), None),
    (dict(n=3, H=21, W=19, Cin=64, in_ld=136, Cout=72, k=1, s=1, p=0, d=1, acts=(4,), of32=1, coff=4), None),
    (dict(n=3, H=45, W=46, Cin=64, Cout=264, k=3, s=2, p=1, d=1, acts=(1,), resid=2), None),
    # ConvTranspose2d(2, 2) as a 1x1 conv with the pixel-shuffle epilogue, fp16 and fp32 output
    (dict(n=1, H=20, W=28, Cin=64, Cout=256, k=1, s=1, p=0, d=1, acts=(1,), mode=1), None),
    (dict(n=2, H=13, W=17, Cin=128, Cout=128, k=1, s=1, p=0, d=1, acts=(0, 4), mode=1, of32=1), None),
]


@pytest.mark.parametrize("kw,bw", CONV, ids=["conv%d" % i for i in range(len(CONV))])
def test_conv(kw, bw):
    res = _conv_case(**kw)
    for act, (got, recs) in res["out"].items():
        assert len(recs) == 1
        if bw is not None:
            assert recs[0]["bw_log2"] == bw, (kw, recs[0])
        assert recs[0]["mode"] == kw.get("mode", 0)
        _assert_close("conv %s" % kw, "conv", res["K"], res["pre"], res["S"], res["extra"], act, got, res["of32"])
        _CHECKED.add(_instance(recs[0]))


def test_every_conv_patch_shape_reached():
    reached = {_conv_case(**kw)["out"][kw["acts"][0]][1][0]["bw_log2"] for kw, _ in CONV}
    missing = sorted({3, 4, 5, 6, 7} - reached)
    assert not missing, "tile patches bw_log2 never used: %s" % missing


# ------------------------------------------------------------------------------------------------ the engines' plans
def _rt_linears(S, Q, n=2, D=256, ffn=1024, layers=6):
    lv = (S // 8) ** 2 + (S // 16) ** 2 + (S // 32) ** 2
    RM, RQ, R5 = n * lv, n * Q, n * (S // 32) ** 2
    return [
        dict(M=RM, K=D, N=layers * D, of32=0), dict(M=RM, K=D, N=D, of32=1), dict(M=RM, K=D, N=8, of32=1),  # value_all,
        dict(M=RQ, K=D, N=D, of32=0, acts=(1,)), dict(M=RQ, K=D, N=4, of32=1, ldc=4),     # enc_out, enc_score, box MLP
        dict(M=RQ, K=D, N=288, of32=1, ldc=288), dict(M=RQ, K=2 * D, N=D, of32=0),         # ow, qpos1
        dict(M=RQ, K=D, N=2 * D, of32=0, ldc=3 * D), dict(M=RQ, K=D, N=D, of32=0, ldc=3 * D, coff=2 * D),   # qk, v
        dict(M=RQ, K=D, N=D, of32=1, resid=2, ldr=D),                                      # out / cross_out
        dict(M=RQ, K=D, N=ffn, of32=0, acts=(1,)), dict(M=RQ, K=ffn, N=D, of32=1, resid=2, ldr=D),   # lin1, lin2
        dict(M=R5, K=D, N=D, of32=1, resid=1, ldr=D), dict(M=R5, K=D, N=ffn, of32=0, acts=(2,)),   # AIFI out, l1
    ]


def _rt_convs(S, n=2, D=256):
    g3, g4, g5 = S // 8, S // 16, S // 32
    return [
        dict(n=n, H=g4, W=g4, Cin=2 * D, Cout=D, k=1, s=1, p=0, d=1, acts=(4,)),             # CSP conv1 / conv2
        dict(n=n, H=g3, W=g3, Cin=D, Cout=D, k=3, s=1, p=1, d=1, acts=(4,)),                 # CSP RepVGG
        dict(n=n, H=g5, W=g5, Cin=D, Cout=D, k=1, s=1, p=0, d=1, acts=(4,), ldc=2 * D, coff=D),   # lateral
        dict(n=n, H=g3, W=g3, Cin=D, Cout=D, k=3, s=2, p=1, d=1, acts=(4,), ldc=2 * D),      # down
        dict(n=n, H=g3, W=g3, Cin=2 * D, Cout=D, k=1, s=1, p=0, d=1, ldc=2 * D, coff=D),     # enc_proj
    ]


# PARSeq: the encoder's and the AR step's linears (test_gpu_gemm_epilogue.py)
PARSEQ = [dict(M=128 * 400 + 37, K=768, N=2304, of32=0), dict(M=128 * 400 + 37, K=768, N=768, of32=1, resid=2,
                                                                in_place=True),
          dict(M=128 * 400 + 37, K=768, N=3072, of32=0, acts=(2,)),
          dict(M=128 * 400 + 37, K=3072, N=768, of32=1, resid=2, in_place=True),
          dict(M=3200, K=768, N=768, of32=0), dict(M=3200, K=768, N=768, of32=1, resid=2, in_place=True),
          dict(M=3200, K=768, N=3072, of32=0, acts=(2,)), dict(M=3200, K=3072, N=768, of32=1, resid=2, in_place=True)]
ENGINE_LINEAR = ([("rtdetr640", kw) for kw in _rt_linears(640, 300)] + [("rtdetr960", kw) for kw in
                                                                         _rt_linears(960, 1500)] +
                 [("parseq", kw) for kw in PARSEQ])
ENGINE_CONV = ([("rtdetr640", kw) for kw in _rt_convs(640)] + [("rtdetr960", kw) for kw in _rt_convs(960)] +
               # DBNet: outproj[0] into fuse + 192 (pitch 256), the others at their own resolution
               [("dbnet", dict(n=1, H=296, W=400, Cin=256, Cout=64, k=3, s=1, p=1, d=1, ldc=256, coff=192)),
                ("dbnet", dict(n=1, H=74, W=100, Cin=256, Cout=64, k=3, s=1, p=1, d=1))])


@pytest.mark.parametrize("eng,kw", ENGINE_LINEAR, ids=["%s-%d" % (e, i) for i, (e, _) in enumerate(ENGINE_LINEAR)])
def test_engine_linear_shapes(eng, kw):
    _check_linear("engine linear", _linear_case(**kw), "%s %s" % (eng, kw))


@pytest.mark.parametrize("eng,kw", ENGINE_CONV, ids=["%s-%d" % (e, i) for i, (e, _) in enumerate(ENGINE_CONV)])
def test_engine_conv_shapes(eng, kw):
    res = _conv_case(**kw)
    for act, (got, recs) in res["out"].items():
        _assert_close("%s %s" % (eng, kw), "engine conv", res["K"], res["pre"], res["S"], res["extra"], act, got,
                      res["of32"])
        _CHECKED.add(_instance(recs[0]))


def _all_checked():
    """Every instance this file checks against float64 (runs whatever case has not run yet)."""
    for idx in range(30):
        test_linear_instance_all_activations(idx)
    for kw in EDGE_LINEAR:
        test_linear_edges(kw)
    for kw, bw in CONV:
        test_conv(kw, bw)
    for eng, kw in ENGINE_LINEAR:
        test_engine_linear_shapes(eng, kw)
    for eng, kw in ENGINE_CONV:
        test_engine_conv_shapes(eng, kw)
    return set(_CHECKED)


# seeded engines, as the engine tests build them
def _rtdetr(kind, n):
    from oracle import rtdetr as R
    from yomitoku_b200.config import (LayoutParserRTDETRv2V2Config, TableCellParserRTDETRv2Config,
                                      TableStructureRecognizerRTDETRv2Config, to_config)
    from yomitoku_b200.models import RTDETRv2
    cfg = {"layout": LayoutParserRTDETRv2V2Config, "table": TableStructureRecognizerRTDETRv2Config,
           "cell": TableCellParserRTDETRv2Config}[kind]
    spec = R.RTDETRSpec(num_classes=6, num_queries=1500, img_size=[960, 960]) if kind == "cell" else R.SPECS[kind]
    m = RTDETRv2(cfg=to_config(cfg()))
    m.load_state_dict(R.make_state_dict(spec, seed=3))
    m = m.to("cuda")
    x = torch.rand(n, 3, spec.img_size[0], spec.img_size[1], generator=torch.Generator().manual_seed(4))
    return lambda: m(x.cuda())


def _dbnet():
    from yomitoku_b200 import TextDetector
    from yomitoku_b200.synth import synthetic_page
    det = TextDetector(from_pretrained=False, device="cuda")
    page, _ = synthetic_page(0)
    return lambda: det.model.detect_pages_u8(page)


def _parseq():
    from oracle import parseq as ops
    from oracle import weights
    from yomitoku_b200 import TextRecognizer
    name = "parseq-large-v4_1"
    rec = TextRecognizer(model_name=name, from_pretrained=False, device="cuda", dynamic_width=True,
                         batch_bucketing=True)
    rec.model.load_state_dict(weights.make_parseq_state_dict(ops.SPECS[name], seed=4, peaked=True))
    img = torch.rand(8, 3, 32, 160, generator=torch.Generator().manual_seed(5)) * 2 - 1
    return lambda: rec.model(img)


ENGINES = {"layout": lambda: _rtdetr("layout", 2), "table": lambda: _rtdetr("table", 2),
           "cell": lambda: _rtdetr("cell", 2), "dbnet": _dbnet, "parseq": _parseq}


@pytest.mark.parametrize("engine", list(ENGINES))
def test_engine_instances_are_checked(engine):
    """Every instance a forward launches is one this file checks against float64; EPI_CONVT_FINAL (2), EPI_ROWMAX
    (3) and the 7-tap stem plan belong to the decode-tail and DBNet kernel tests."""
    fwd = ENGINES[engine]()
    fwd()                                      # first call: plans and buffers
    torch.cuda.synchronize()
    recs = _launches(fwd)
    torch.cuda.synchronize()
    assert recs, "no gemm launches recorded"
    launched = {_instance(r) for r in recs if r["mode"] not in (2, 3) and r["ntaps"] != 7}
    missing = sorted(launched - _all_checked())
    assert not missing, "%s launches instances (block_n, out_f32, resid, mode, act, epi) not checked here: %s" % (
        engine, missing)


# ------------------------------------------------------------------------------------------------ wrong variants
def test_wrong_variants_miss_the_bound():
    """Each perturbation of the reference misses the bound by >= 10x on some element; the true reference passes."""
    factors = {}
    # one 64-wide K block dropped; bias shifted by one column; residual read one row off (fp32 output, K = 256)
    res = _linear_case(M=1000, K=256, N=120, of32=1, resid=2, acts=(0,), seed=11)
    got = res["out"][0][0]
    K, pre, S, extra = res["K"], res["pre"], res["S"], res["extra"]
    e = _e_pre(K, S, extra)
    assert _ratio(got, pre, e, 1) <= 1
    a64, w64 = res["A"][:, :K].double(), res["W"].double()
    drop = pre - a64[:, 64:128] @ w64[:, 64:128].t()
    factors["K block 64..127 dropped"] = _ratio(got, drop, e, 1)
    b = res["b"].double()
    factors["bias shifted by one column"] = _ratio(got, pre - b + torch.roll(b, -1), e, 1)
    r = res["R_vals"].double()
    factors["residual one row off"] = _ratio(got, pre - r + torch.roll(r, -1, 0), e, 1)
    # tanh-GELU for erf-GELU (fp32 output, pre-activations spread over [-4, 4] by the bias)
    res = _linear_case(M=600, K=64, N=64, of32=1, acts=(2,), a_scale=0.05, b_scale=2.0, seed=12)
    got, pre, e = res["out"][2][0], res["pre"], _e_pre(64, res["S"], res["extra"])
    y = _act(pre, 2)
    assert _ratio(got, y, _inner(pre, e, 2, y), 1) <= 1
    yt = F.gelu(pre, approximate="tanh")
    factors["tanh GELU"] = _ratio(got, yt, _inner(pre, e, 2, yt), 1)
    # SiLU computed as sigmoid
    res = _linear_case(M=600, K=64, N=64, of32=1, acts=(4,), seed=13)
    got, pre, e = res["out"][4][0], res["pre"], _e_pre(64, res["S"], res["extra"])
    ys = _act(pre, 3)
    factors["SiLU as sigmoid"] = _ratio(got, ys, _inner(pre, e, 4, ys), 1)
    # fp16 output truncated instead of rounded to nearest
    res = _linear_case(M=600, K=128, N=64, of32=0, acts=(0,), seed=14)
    got, pre, e = res["out"][0][0], res["pre"], _e_pre(128, res["S"], res["extra"])
    assert _rounding_ratio(got, pre, e, "rn") <= 1
    factors["fp16 truncated"] = _rounding_ratio(got, pre, e, "rz")
    for name, f in factors.items():
        print("[gemm variants] wrong variant %-28s misses the bound by %.3g x" % (name, f))
    weak = {k: v for k, v in factors.items() if not v >= 10}
    assert not weak, weak
