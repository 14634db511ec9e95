"""CPU: the bound helpers of tests/stage_bounds.py, checked two ways without a GPU at the RT-DETRv2 engine's shapes.

  holds      a CPU emulation of the kernel's arithmetic - fp16 operands (BatchNorm folded in fp32, then rounded),
             fp32 accumulation and epilogue, fp16 or fp32 output - lies within the bound of the float64 result
  not vacuous  the emulated error reaches a stated fraction of the bound somewhere (FRACTION below; the worst-case
             bounds sum every rounding with the same sign, so a real error sits well below them), and the float64
             result moved by twice its bound misses it

The emulation is not the kernel: torch's fp32 CPU sums and expf are correctly rounded or nearly so, so it exercises
the operand and output roundings that dominate every bound, not the tensor-core adders' truncation."""
import math

import pytest
import torch
import torch.nn.functional as F

import stage_bounds as B

# measured emulated worst ratios: lin 0.077 - 0.25, conv 0.053 - 0.48, ln 0.0073 - 0.012 (fp32 output: the fp32
# statistics terms are worst case, the CPU's are nearly exact) and 0.83 - 0.95 (fp16), attend 0.33 - 0.54,
# sample_shift 0.99, deform 0.095 (op-level) and 0.61 (offset / logit errors)
FRACTION = {"lin": 0.05, "conv": 0.025, "ln": 0.005, "attend": 0.2, "sample_shift": 0.5, "deform": 0.05}


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ratios(name, got, ref, e):
    r = float(((got.double() - ref).abs() / e).max())
    moved = ref + 2 * e * torch.where(torch.rand(ref.shape, generator=_gen(9), dtype=torch.float64) < 0.5, -1.0, 1.0)
    r2 = float(((moved - ref).abs() / e).max())
    print("[stage-bounds] %-40s emulated worst |d| / bound %.3g" % (name, r))
    assert r <= 1.0, (name, r)
    assert r >= FRACTION[name.split()[0]], (name, r)
    assert r2 > 1.0
    return r


def _h(t):
    """fp16 rounding, as float32"""
    return t.half().float()


@pytest.mark.parametrize("M,K,N,act,out16", [(300, 256, 256, None, True), (300, 256, 288, None, False),
                                             (400, 256, 1024, "gelu", True), (400, 1024, 256, None, False),
                                             (300, 256, 256, "relu", True), (300, 512, 256, None, True)])
def test_lin_bound(M, K, N, act, out16):
    g = _gen(M + K + N)
    x = _h(torch.randn(M, K, generator=g))
    W = torch.randn(N, K, generator=g, dtype=torch.float64) / math.sqrt(K)
    b = 0.02 * torch.randn(N, generator=g, dtype=torch.float64)
    r = _h(torch.randn(M, N, generator=g)) if not out16 else None
    pre = x @ _h(W.float()).T + b.float()
    if r is not None:
        pre = pre + r
    y = {None: pre, "relu": F.relu(pre), "gelu": F.gelu(pre)}[act]
    y = _h(y) if out16 else y
    ref, e = B.lin(x.double(), None, W, b, out16, resid=None if r is None else r.double(), act=act)
    _ratios("lin %dx%d->%d %s" % (M, K, N, act), y, ref, e)


def _bn_sd(C, g):
    return {"n.weight": 1.0 + 0.1 * torch.randn(C, generator=g), "n.bias": 0.1 * torch.randn(C, generator=g),
            "n.running_mean": 0.1 * torch.randn(C, generator=g), "n.running_var": 1.0 + 0.2 * torch.rand(C, generator=g)}


def _fold32(sd, w):
    """the engine's fp32 fold (rtdetr_engine.cu bn_fold), weight rounded to fp16"""
    s = sd["n.weight"] / torch.sqrt(sd["n.running_var"] + 1e-5)
    return _h(w * s.view(-1, 1, 1, 1)), sd["n.bias"] - sd["n.running_mean"] * s


@pytest.mark.parametrize("Cin,Cout,k,stride,hw,act", [(256, 256, 3, 1, 20, "silu"), (512, 256, 1, 1, 20, "silu"),
                                                      (256, 256, 3, 2, 20, "silu"), (3, 32, 3, 2, 48, "relu"),
                                                      (64, 256, 1, 1, 24, None)])
def test_conv_bound(Cin, Cout, k, stride, hw, act):
    g = _gen(Cin + Cout + k + hw)
    x = _h(torch.rand(1, Cin, hw, hw, generator=g) * 2 - 0.5)
    w = torch.randn(Cout, Cin, k, k, generator=g) * math.sqrt(2.0 / (Cin * k * k))
    sd = _bn_sd(Cout, g)
    W16, b32 = _fold32(sd, w)
    pre = F.conv2d(x, W16, b32, stride, (k - 1) // 2)
    if act == "silu":
        y = pre / (1 + torch.exp(-pre))
    else:
        y = F.relu(pre) if act == "relu" else pre
    sd64 = {kk: v.double() for kk, v in sd.items()}
    W, b, e_b = B.fold_bn(sd64, "n", w.double())
    ref, e = B.conv(x.double(), None, W, b, stride, True, act=act, e_b=e_b)
    _ratios("conv %d->%d k%d s%d %s" % (Cin, Cout, k, stride, act), _h(y), ref, e)


def test_conv_repvgg_fold_matches_two_branches():
    g = _gen(5)
    sd = {}
    for br, k in (("conv1", 3), ("conv2", 1)):
        sd["b.%s.conv.weight" % br] = torch.randn(16, 16, k, k, generator=g, dtype=torch.float64) * 0.2
        for kk, v in _bn_sd(16, g).items():
            sd["b.%s.norm.%s" % (br, kk[2:])] = v.double()
    x = torch.randn(2, 16, 9, 9, generator=g, dtype=torch.float64)
    from oracle import rtdetr as R
    W, b, _ = B.fold_repvgg(sd, "b")
    assert torch.allclose(F.silu(F.conv2d(x, W, b, 1, 1)), R.repvgg(sd, "b", x), rtol=0, atol=1e-12)
    W0, b0, _ = B.fold_repvgg(sd, "b", tap=(0, 0))
    assert not torch.allclose(F.conv2d(x, W0, b0, 1, 1), F.conv2d(x, W, b, 1, 1), rtol=0, atol=1e-3)


def test_silu_and_sigmoid_terms():
    """the epilogue terms bound fp32 evaluations with a perturbed exponential (the __expf error model)"""
    v = torch.linspace(-60, 60, 200001, dtype=torch.float64)
    v32 = v.float()
    for sgn in (-1.0, 1.0):
        t = torch.exp(-v32) * (1 + sgn * ((2 + 1.16 * v32.abs()) * 2.0 ** -24).float())   # within the ulp model
        y = v32 / (1 + t)
        r = float(((y.double() - F.silu(v)).abs() / B.silu_term(v)).max())
        assert r <= 1.0, r
        s = 1 / (1 + t)
        r2 = float(((s.double() - torch.sigmoid(v)).abs() / B.sigmoid_term(v)).max())
        assert r2 <= 1.0, r2
    assert r > 0.1 and r2 > 0.05, (r, r2)


@pytest.mark.parametrize("rows,shift", [(300, 0.0), (1600, 3.0), (300, 30.0)])
@pytest.mark.parametrize("out16", [False, True])
def test_ln_bound(rows, shift, out16):
    g = _gen(rows + int(shift))
    D = 256
    x = torch.randn(rows, D, generator=g) * (0.5 + torch.rand(rows, 1, generator=g) * 3) + shift
    sd = {"n.weight": 1.0 + 0.05 * torch.randn(D, generator=g, dtype=torch.float64),
          "n.bias": 0.05 * torch.randn(D, generator=g, dtype=torch.float64)}
    y = F.layer_norm(x, (D,), sd["n.weight"].float(), sd["n.bias"].float(), 1e-5)
    ref, e = B.ln(sd, "n", x.double(), None, 1e-5, out16)
    _ratios("ln rows %d shift %g fp16 %d" % (rows, shift, out16), _h(y) if out16 else y, ref, e)


@pytest.mark.parametrize("L,scale", [(400, 1.0), (300, 3.0), (900, 2.0)])
def test_attend_bound(L, scale):
    g = _gen(L)
    D, H = 256, 8
    q, k, v = (_h(torch.randn(L, D, generator=g) * scale) for _ in range(3))
    hd = D // H
    qh, kh, vh = (t.reshape(L, H, hd).transpose(0, 1) for t in (q, k, v))
    p = torch.softmax(qh @ kh.transpose(-1, -2) / math.sqrt(hd), -1)
    o = (_h(p) @ vh).transpose(0, 1).reshape(L, D)
    ref, e = B.attend(q.double(), k.double(), v.double(), H)
    _ratios("attend %d tokens x%g" % (L, scale), _h(o), ref, e)


def test_sample_shift_bound():
    g = _gen(11)
    M, c, h, w, Q = 8, 32, 20, 30, 500
    v = torch.randn(M, c, h, w, generator=g, dtype=torch.float64)
    loc = torch.rand(M, Q, 2, generator=g, dtype=torch.float64) * 1.1 - 0.05       # a few samples in the padding
    e_loc = torch.full((M, Q, 2), 2e-3, dtype=torch.float64)

    def sample(lc):
        return F.grid_sample(v, (2 * lc - 1)[:, :, None, :], mode="bilinear", padding_mode="zeros",
                             align_corners=False)[..., 0]

    bound = B.sample_shift(v, loc, e_loc) + 1e-300
    worst = 0.0
    for trial in range(6):
        d = (torch.rand(M, Q, 2, generator=g, dtype=torch.float64) * 2 - 1) * e_loc
        if trial < 4:                                                 # the four corners of the error box
            d = torch.stack([e_loc[..., 0] * (1 - 2 * (trial & 1)), e_loc[..., 1] * (1 - 2 * (trial >> 1))], -1)
        r = float(((sample(loc + d) - sample(loc)).abs() / bound).max())
        assert r <= 1.0, r
        worst = max(worst, r)
    print("[stage-bounds] sample_shift worst |d| / bound %.3g" % worst)
    assert worst >= FRACTION["sample_shift"]


def test_deform_bound():
    """deform_core in fp32 on fp16 values (offsets and weights exact) within the op-level term, and with perturbed
    offsets and logits within the composite's sampling and weight terms"""
    from oracle import rtdetr as R
    spec = R.RTDETRSpec()
    shapes = [(16, 16), (8, 8), (4, 4)]
    g = _gen(12)
    n, K, H, P = 2, 50, spec.heads, sum(spec.num_points)
    total = sum(a * b for a, b in shapes)
    value = _h(torch.randn(n, total, H, 32, generator=g)).double()
    ref4 = torch.rand(n, K, 4, generator=g, dtype=torch.float64) * 0.6 + 0.2
    off = torch.randn(n, K, H, P, 2, generator=g, dtype=torch.float64) * 2
    lg = torch.randn(n, K, H, P, generator=g, dtype=torch.float64)
    out32 = R.deform_core(spec, value.float(), shapes, ref4.float(), off.float(), torch.softmax(lg.float(), -1))
    ref, e = B.deform(spec, value, shapes, ref4, off, torch.softmax(lg, -1))
    _ratios("deform op-level", _h(out32), ref, e)
    e_off = torch.full_like(off, 1e-2)
    e_lg = torch.full_like(lg, 1e-3)
    worst = 0.0
    for sgn in (-1.0, 1.0):
        moved = R.deform_core(spec, value, shapes, ref4, off + sgn * e_off, torch.softmax(lg + sgn * e_lg, -1))
        _, e2 = B.deform(spec, value, shapes, ref4, off, torch.softmax(lg, -1), e_off=e_off, e_logit=e_lg)
        worst = max(worst, float(((moved - ref).abs() / e2).max()))
    print("[stage-bounds] deform with offset / logit errors worst |d| / bound %.3g" % worst)
    assert FRACTION["deform"] <= worst <= 1.0
