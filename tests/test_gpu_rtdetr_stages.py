"""GPU: the RT-DETRv2 engine stage by stage against float64, every stage fed the engine's own input to it.

The engine (csrc/rtdetr_engine.cu) exposes its stages through RTDETRv2.set_debug / RTDETRv2.debug_tensor: the buffers it
keeps, and copies of the ones it overwrites in place (CSP steps, the AIFI residual sum, the encoder box head, every
decoder layer).  Each check takes the engine's input to one stage as read through that hook, runs the same stage in
float64 on the device (oracle/rtdetr.py's stage functions where the stage is one of them) and compares against an
a-priori componentwise bound computed from the operands by tests/stage_bounds.py, whose docstring derives every rule.
Errors therefore do not accumulate across stages.

  single GEMMs and convolutions   worst-case bound (stage_bounds.lin / conv): stem, every bottleneck convolution with
                                  the avg-pool shortcut and the residual + ReLU output, input_proj, AIFI qk / v / out /
                                  linear1 (GELU) / linear2, lateral and downsample convolutions, every CSP convolution
                                  and RepVGG step (SiLU), the decoder input_proj into the level-major memory and each
                                  value column block (layer i's value_proj), enc_output (valid mask), the score head,
                                  the encoder box MLP, query_pos linear1, and per decoder layer qk / v / out / ow /
                                  cross_out / linear1 / linear2 / box MLP, and the last score head
  LayerNorm                       fp32 output against stage_bounds.ln; the fp16 output must equal the fp32 output
                                  rounded once, bit for bit
  attention                       stage_bounds.attend per image: AIFI over 400 / 900 tokens, decoder self-attention
                                  over 300 / 1500 queries
  deformable attention            the op-level bound of test_gpu_decoder_kernels.py (2^-10 max|v| + 2^-11 |o|) on the
                                  engine's ow / ref / value block
  exact                           max-pool, the up-sampling halves of the FPN concat buffers, the CSP sum, the query
                                  inputs tgt + qpos; ref_update and query_pos layer 0 against their op-level bounds of
                                  test_gpu_glue_kernels.py
  composites                      root-sum-square chains at 6 sigma (stage_bounds docstring): the AIFI layer, each CSP
                                  block, each whole decoder layer from (x_in, ref) to (x3, next ref), and the final
                                  logits and boxes from the last layer's input
Padded columns (Cout < 64, the score heads at a pitch of 8) must be exactly zero.

Every comparator is also given a wrong reference that must miss its bound somewhere (the factor is printed): the
RepVGG 1x1 branch at tap 0, a variant-b shortcut (stride-2 1x1 convolution), the FPN concat halves swapped, AIFI V from
src + pos, enc_output without the valid mask, decoder V from tgt + qpos, the cross-attention query without qpos, layer
i reading value block i +- 1, offsets without the 1 / num_points scale, ref not refreshed between layers, and
norm2 / norm3 swapped against the composite bound.

Configurations (seeded trained-like weights, nonzero enc_output.proj bias): layout 640 n = 3 (image interleaving in the
level-major memory), table 640 n = 1, cell 960 n = 2 with 1500 queries; the layout run also goes through forward_u8,
whose captures must equal forward_f32's on the same packed input."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import stage_bounds as B
from oracle import rtdetr as R
from yomitoku_b200 import _lib
from yomitoku_b200.config import (LayoutParserRTDETRv2V2Config, TableCellParserRTDETRv2Config,
                                  TableStructureRecognizerRTDETRv2Config, to_config)
from yomitoku_b200.models import RTDETRv2

pytestmark = pytest.mark.gpu
DEV = "cuda"
D = 256
U, E, SUB = B.U, B.E, B.SUB
RATIOS = {}
MISSES = {}


# ------------------------------------------------------------------------------------------------------ comparators
def _check(run, stage, got, ref, bound):
    r = float(((got - ref).abs() / bound).max()) if got.numel() else 0.0
    key = (stage, run["tag"])
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)
    assert r <= 1.0, "%s %s: worst |d| / bound = %.3g" % (run["tag"], stage, r)


def _miss(run, what, got, wrong, bound):
    r = float(((got - wrong).abs() / bound).max())
    MISSES[what] = min(MISSES.get(what, float("inf")), r)
    print("[rt-stages] %s wrong reference %-44s worst |d| / bound %.3g (must exceed 1)" % (run["tag"], what, r))
    assert r > 1.0, "%s: wrong reference '%s' within the bound" % (run["tag"], what)


def _report(run):
    for (stage, tag), r in sorted(RATIOS.items()):
        if tag == run["tag"]:
            print("[rt-stages] %-12s %-48s %.3g" % (tag, stage, r))


def _exact16(run, what, got16, ref):
    """the fp16 output equals the float32 value rounded once"""
    assert torch.equal(got16, ref.float().half().double()), "%s %s" % (run["tag"], what)


# ------------------------------------------------------------------------------------------------------ runs
def _model(cfg, spec, seed, n):
    sd = R.make_state_dict(spec, seed=seed)
    sd["decoder.enc_output.proj.bias"] = 0.1 * torch.randn(D, generator=torch.Generator().manual_seed(seed))
    m = RTDETRv2(cfg=to_config(cfg()))
    m.load_state_dict(sd)
    m = m.to("cuda")
    x = torch.rand(n, 3, spec.img_size[0], spec.img_size[0], generator=torch.Generator().manual_seed(seed + 1))
    return m, sd, x


def _run(tag, cfg, spec, seed, n):
    m, sd, x = _model(cfg, spec, seed, n)
    m.set_debug(True)
    out = m(x.to(DEV))
    torch.cuda.synchronize()
    S = spec.img_size[0]
    shapes = [(S // s, S // s) for s in spec.strides]
    off = [0]
    for h, w in shapes:
        off.append(off[-1] + h * w)
    return dict(tag=tag, m=m, sd64={k: v.to(DEV, torch.float64) for k, v in sd.items()}, spec=spec, n=n, S=S, x=x,
                shapes=shapes, off=off, out={k: v.to(DEV, torch.float64) for k, v in out.items()})


_RUNS = {}


def _get(name):
    if name not in _RUNS:
        _RUNS.clear()          # one engine's float64 state at a time
        torch.cuda.empty_cache()
        if name == "layout640":
            _RUNS[name] = _run("layout640n3", LayoutParserRTDETRv2V2Config, R.SPECS["layout"], 31, 3)
        elif name == "table640":
            _RUNS[name] = _run("table640n1", TableStructureRecognizerRTDETRv2Config, R.SPECS["table"], 32, 1)
        else:
            spec = R.RTDETRSpec(num_classes=6, num_queries=1500, img_size=[960, 960])
            _RUNS[name] = _run("cell960n2", TableCellParserRTDETRv2Config, spec, 33, 2)
    return _RUNS[name]


CONFIGS = ["layout640", "table640", "cell960"]


@pytest.fixture(scope="module", params=CONFIGS)
def run(request):
    """module scope: pytest runs every stage test of one configuration before it builds the next"""
    return _get(request.param)


def _t(run, name):
    """debug tensor as float64 on the device, in the engine's shape (NHWC maps, [1, 1, rows, c] token matrices)"""
    return torch.from_numpy(run["m"].debug_tensor(run["n"], name)).to(DEV, torch.float64)


def _rows(run, name):
    t = _t(run, name)
    return t.reshape(-1, t.shape[-1])


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def _conv(run, x, p, stride=1, act=None, resid=None, fold=None, rss=False, e_x=None, e_r=None):
    """stage_bounds.conv of the ConvNormLayer p (or the folded (W, b, e_b)) on an NHWC tensor -> NHWC (y, bound)"""
    W, b, e_b = fold if fold is not None else B.fold_conv_norm(run["sd64"], p)
    y, e = B.conv(nchw(x[..., :W.shape[1]]), None if e_x is None else nchw(e_x), W, b, stride, True,
                  resid=None if resid is None else nchw(resid), e_r=None if e_r is None else nchw(e_r), act=act,
                  e_b=e_b, rss=rss)
    return nhwc(y), nhwc(e)


def _zero_pad_cols(run, what, t, real):
    if t.shape[-1] > real:
        assert bool((t[..., real:] == 0).all()), "%s %s: padded columns are not exactly zero" % (run["tag"], what)


# ------------------------------------------------------------------------------------------------------ backbone
def test_backbone_stages(run):
    sd = run["sd64"]
    bb = "backbone."
    x = _t(run, "input")
    _zero_pad_cols(run, "input", x, 3)
    assert torch.equal(x[..., :3], run["x"].permute(0, 2, 3, 1).half().to(DEV, torch.float64)), "packed input"
    for i, (name, stride) in enumerate((("conv1_1", 2), ("conv1_2", 1), ("conv1_3", 1))):
        y = _t(run, "stem%d" % (i + 1))
        ref, e = _conv(run, x, bb + "conv1." + name, stride, "relu")
        real = ref.shape[-1]
        _zero_pad_cols(run, "stem%d" % (i + 1), y, real)
        _check(run, "stem conv%d (ReLU)" % (i + 1), y[..., :real], ref, e)
        x = y
    pool = _t(run, "pool")
    assert torch.equal(pool, nhwc(F.max_pool2d(nchw(x), 3, 2, 1))), "max-pool"
    x = pool
    for s, nb in enumerate(run["spec"].blocks):
        for b in range(nb):
            nm, p = "res%d.%d" % (s, b), bb + "res_layers.%d.blocks.%d" % (s, b)
            stride = 2 if (b == 0 and s != 0) else 1
            a, bt, o = _t(run, nm + ".a"), _t(run, nm + ".b"), _t(run, nm)
            ref, e = _conv(run, x, p + ".branch2a", 1, "relu")
            _check(run, "bottleneck branch2a (1x1, ReLU)", a, ref, e)
            ref, e = _conv(run, a, p + ".branch2b", stride, "relu")
            _check(run, "bottleneck branch2b (3x3, ReLU)", bt, ref, e)
            res = x
            if b == 0:
                sc = _t(run, nm + ".short")
                sin = x
                if stride == 2:
                    pl = _t(run, nm + ".pool")
                    mean = nhwc(F.avg_pool2d(nchw(x), 2, 2))
                    tol = torch.ldexp(torch.ones_like(mean), torch.frexp(mean.abs().clamp(min=2.0 ** -14))[1] - 11) + \
                        3 * E * nhwc(F.avg_pool2d(nchw(x.abs()), 2, 2))
                    _check(run, "shortcut avg-pool", pl, mean, tol)
                    sin = pl
                ref, e = _conv(run, sin, p + (".short.conv" if s else ".short"))
                _check(run, "shortcut conv (1x1)", sc, ref, e)
                if stride == 2 and s == 1:
                    wrong, _ = _conv(run, x, p + ".short.conv", 2)
                    _miss(run, "variant-b shortcut (stride-2 1x1)", sc, wrong, e)
                res = sc
            ref, e = _conv(run, bt, p + ".branch2c", 1, "relu", resid=res)
            _check(run, "bottleneck branch2c + residual (ReLU)", o, ref, e)
            x = o
    _report(run)


# ------------------------------------------------------------------------------------------------------ encoder
def _lin_sd(sd, p, x, out16=True, **kw):
    return B.lin(x, kw.pop("e_x", None), sd[p + ".weight"], sd[p + ".bias"], out16, **kw)


def _csp(run, name, p, cat, mutate=False):
    """one CSPRepLayer from its concat input: every convolution, the exact sum and the 6-sigma composite"""
    sd = run["sd64"]
    c1, r0, r1 = _t(run, name + ".c1"), _t(run, name + ".r0"), _t(run, name + ".r1")
    t2, x2 = _t(run, name + ".t2"), _t(run, name + ".x2")
    ref, e = _conv(run, cat, p + ".conv1", act="silu")
    _check(run, "CSP conv1 (SiLU)", c1, ref, e)
    if mutate:
        sw = torch.cat([cat[..., D:], cat[..., :D]], -1)
        _miss(run, "FPN concat halves swapped", c1, _conv(run, sw, p + ".conv1", act="silu")[0], e)
    for i, (xin, got) in enumerate(((c1, r0), (r0, r1), (r1, t2))):
        b = "%s.bottlenecks.%d" % (p, i)
        fold = B.fold_repvgg(sd, b)
        ref, e = _conv(run, xin, None, act="silu", fold=fold)
        two = nhwc(R.repvgg(sd, b, nchw(xin)))                          # the fused weight restates the two branches
        assert float((ref - two).abs().max()) <= 1e-9 * (1 + float(two.abs().max()))
        _check(run, "RepVGG (fused 3x3, SiLU)", got, ref, e)
        if mutate and i == 0:
            wrong, _ = _conv(run, xin, None, act="silu", fold=B.fold_repvgg(sd, b, tap=(0, 0)))
            _miss(run, "RepVGG 1x1 branch at tap 0", got, wrong, e)
    ref, e = _conv(run, cat, p + ".conv2", act="silu")
    _check(run, "CSP conv2 (SiLU)", x2, ref, e)
    # composite: conv1 -> 3 RepVGG -> + conv2, root-sum-square at 6 sigma
    y, ey = _conv(run, cat, p + ".conv1", act="silu", rss=True)
    for i in range(3):
        y, ey = _conv(run, y, None, act="silu", fold=B.fold_repvgg(sd, "%s.bottlenecks.%d" % (p, i)), rss=True, e_x=ey)
    z, ez = _conv(run, cat, p + ".conv2", act="silu", rss=True)
    ref = y + z
    e = B.LAMBDA * (torch.sqrt(ey * ey + ez * ez) + U * ref.abs() + SUB)
    assert float((ref - nhwc(R.csp_rep(sd, p, nchw(cat[..., :2 * D]), 3))).abs().max()) <= 1e-9 * (1 + float(ref.abs().max()))
    return (t2 + x2).float().half().double(), ref, e


def test_encoder_stages(run):
    sd, spec, n = run["sd64"], run["spec"], run["n"]
    en = "encoder."
    c3, c4, c5 = _t(run, "c3"), _t(run, "c4"), _t(run, "c5")
    cat3, cat4, pcat4, pcat5, proj5 = (_t(run, k) for k in ("cat3", "cat4", "pcat4", "pcat5", "proj5"))
    for i, (src, got) in enumerate(((c3, cat3[..., D:]), (c4, cat4[..., D:]), (c5, proj5))):
        ref, e = _conv(run, src, en + "input_proj.%d" % i)
        _check(run, "encoder input_proj", got, ref, e)
    # ---- AIFI
    p = en + "encoder.0.layers.0"
    g5 = run["S"] // 32
    T5 = g5 * g5
    src = proj5.reshape(n * T5, D)
    q = _rows(run, "aifi.q")
    qkv, att, y1 = _rows(run, "aifi.qkv"), _rows(run, "aifi.att"), _rows(run, "aifi.y1")
    s32, s16, ffn, y, out = (_rows(run, k) for k in ("aifi.s32", "aifi.s16", "aifi.ffn", "aifi.y", "aifi.out"))
    W, b = sd[p + ".self_attn.in_proj_weight"], sd[p + ".self_attn.in_proj_bias"]
    ref, e = B.lin(q, None, W[:2 * D], b[:2 * D], True)
    _check(run, "AIFI qk", qkv[:, :2 * D], ref, e)
    ref, e = B.lin(src, None, W[2 * D:], b[2 * D:], True)
    _check(run, "AIFI v", qkv[:, 2 * D:], ref, e)
    _miss(run, "AIFI V from src + pos", qkv[:, 2 * D:], B.lin(q, None, W[2 * D:], b[2 * D:], True)[0], e)
    for i in range(n):
        r = slice(i * T5, (i + 1) * T5)
        ref, e = B.attend(qkv[r, :D], qkv[r, D:2 * D], qkv[r, 2 * D:], spec.heads)
        _check(run, "AIFI attention (%d tokens)" % T5, att[r], ref, e)
    ref, e = _lin_sd(sd, p + ".self_attn.out_proj", att, False, resid=src)
    _check(run, "AIFI out_proj + residual", y1, ref, e)
    ref, e = B.ln(sd, p + ".norm1", y1, None, 1e-5, False)
    _check(run, "AIFI norm1 (fp32)", s32, ref, e)
    _exact16(run, "AIFI norm1 fp16", s16, s32)
    ref, e = _lin_sd(sd, p + ".linear1", s16, True, gelu=True)
    _check(run, "AIFI linear1 (GELU)", ffn, ref, e)
    ref, e = _lin_sd(sd, p + ".linear2", ffn, False, resid=s32)
    _check(run, "AIFI linear2 + residual", y, ref, e)
    ref, e = B.ln(sd, p + ".norm2", y, None, 1e-5, True)
    _check(run, "AIFI norm2 (fp16)", out, ref, e)
    # composite AIFI layer from proj5 (q = fp16(proj5 + pos), exact in the engine's add)
    pos = R.sincos_2d(g5, g5, D, spec.pe_temperature, DEV, torch.float64)[0].repeat(n, 1)
    q64 = src + pos
    e_q = U * q64.abs() + 2.0 ** -21 * (1 + g5)                     # the engine's fp32 table (test_gpu_glue_kernels)
    (qk, e_qk), (v, e_v) = B.lin(q64, e_q, W[:2 * D], b[:2 * D], True, rss=True), B.lin(src, None, W[2 * D:], b[2 * D:], True, rss=True)
    a_parts, e_parts = [], []
    for i in range(n):
        r = slice(i * T5, (i + 1) * T5)
        o, eo = B.attend(qk[r, :D], qk[r, D:], v[r], spec.heads, e_qk[r, :D], e_qk[r, D:], e_v[r], rss=True)
        a_parts.append(o)
        e_parts.append(eo)
    a1, e1 = _lin_sd(sd, p + ".self_attn.out_proj", torch.cat(a_parts), False, e_x=torch.cat(e_parts), resid=src, rss=True)
    h, eh = B.ln(sd, p + ".norm1", a1, e1, 1e-5, False, rss=True)
    f, ef = _lin_sd(sd, p + ".linear1", h, True, e_x=eh + U * h.abs() + SUB, gelu=True, rss=True)
    z, ez = _lin_sd(sd, p + ".linear2", f, False, e_x=ef, resid=h, e_r=eh, rss=True)
    ref, e = B.ln(sd, p + ".norm2", z, ez, 1e-5, True, rss=True)
    oracle = R.aifi_layer(sd, p, src.reshape(n, T5, D), pos[:T5][None], spec.heads).reshape(n * T5, D)
    assert float((oracle - ref).abs().max()) <= 1e-9                # the chain restates the oracle's AIFI layer
    _check(run, "AIFI layer (composite, 6 sigma)", out, oracle, B.LAMBDA * e)
    # ---- FPN / PAN
    aifi_out = out.reshape(n, g5, g5, D)
    l5 = pcat5[..., D:]
    ref, e = _conv(run, aifi_out, en + "lateral_convs.0", act="silu")
    _check(run, "lateral conv (SiLU)", l5, ref, e)
    up = lambda t: t.repeat_interleave(2, 1).repeat_interleave(2, 2)      # noqa: E731
    assert torch.equal(cat4[..., :D], up(l5))
    got, ref, e = _csp(run, "fpn0", en + "fpn_blocks.0", cat4, mutate=True)
    fpn4 = _t(run, "fpn4")
    assert torch.equal(fpn4, got)
    _check(run, "CSP block (composite, 6 sigma)", fpn4, ref, e)
    l4 = pcat4[..., D:]
    ref, e = _conv(run, fpn4, en + "lateral_convs.1", act="silu")
    _check(run, "lateral conv (SiLU)", l4, ref, e)
    assert torch.equal(cat3[..., :D], up(l4))
    f3 = _t(run, "enc_out3")
    got, ref, e = _csp(run, "fpn1", en + "fpn_blocks.1", cat3)
    assert torch.equal(f3, got)
    _check(run, "CSP block (composite, 6 sigma)", f3, ref, e)
    ref, e = _conv(run, f3, en + "downsample_convs.0", 2, "silu")
    _check(run, "downsample conv (3x3 s2, SiLU)", pcat4[..., :D], ref, e)
    o4 = _t(run, "enc_out4")
    got, ref, e = _csp(run, "pan0", en + "pan_blocks.0", pcat4)
    assert torch.equal(o4, got)
    _check(run, "CSP block (composite, 6 sigma)", o4, ref, e)
    ref, e = _conv(run, o4, en + "downsample_convs.1", 2, "silu")
    _check(run, "downsample conv (3x3 s2, SiLU)", pcat5[..., :D], ref, e)
    o5 = _t(run, "enc_out5")
    got, ref, e = _csp(run, "pan1", en + "pan_blocks.1", pcat5)
    assert torch.equal(o5, got)
    _check(run, "CSP block (composite, 6 sigma)", o5, ref, e)
    _report(run)


# ------------------------------------------------------------------------------------------------------ decoder input
def _level_rows(run, i):
    """the level-major rows of image i, in the image's own token order (level by level, raster)"""
    n, off, shapes = run["n"], run["off"], run["shapes"]
    return torch.cat([torch.arange(off[l] * n + i * h * w, off[l] * n + (i + 1) * h * w) for l, (h, w) in
                      enumerate(shapes)]).to(DEV)


def _ref_tol(t, s, e_base):
    """ref_update's op-level bound (test_gpu_glue_kernels.py)"""
    return s * (1 - s) * (t.abs() * 2.0 ** -24 + e_base + 2.0 ** -21) + 2.0 ** -22 * s + 1e-300


def _refine_base(ref):
    base = R.inverse_sigmoid(ref)
    return base, 2.0 ** -22 + 2.0 ** -22 * base.abs() + 4e-8


def test_query_selection_stages(run):
    sd, spec, n = run["sd64"], run["spec"], run["n"]
    de = "decoder."
    C, K = spec.num_classes, spec.num_queries
    mem, val = _rows(run, "memory"), _rows(run, "value")
    off = run["off"]
    for l, (nm, (h, w)) in enumerate(zip(("enc_out3", "enc_out4", "enc_out5"), run["shapes"])):
        ref, e = _conv(run, _t(run, nm), de + "input_proj.%d" % l)
        blk = slice(off[l] * n, off[l + 1] * n)
        _check(run, "decoder input_proj (level-major memory)", mem[blk], ref.reshape(-1, D), e.reshape(-1, D))
    for i in range(spec.num_layers):
        p = de + "decoder.layers.%d.cross_attn.value_proj" % i
        ref, e = _lin_sd(sd, p, mem)
        _check(run, "value_proj (column block i)", val[:, i * D:(i + 1) * D], ref, e)
    # enc_output: rows of anchors outside the valid mask see a zero memory row
    valid = sd[de + "valid_mask"].reshape(-1)
    order = torch.cat([_level_rows(run, i) for i in range(n)])          # image i's anchors 0 .. total, in order
    vmask = torch.empty(mem.shape[0], dtype=torch.float64, device=DEV)
    vmask[order] = valid.repeat(n).double()
    ey_ = _rows(run, "enc.y")
    ref, e = _lin_sd(sd, de + "enc_output.proj", mem * vmask[:, None], False)
    _check(run, "enc_output (valid mask)", ey_, ref, e)
    _miss(run, "enc_output without the valid mask", ey_, _lin_sd(sd, de + "enc_output.proj", mem, False)[0], e)
    om32, om16 = _rows(run, "enc.om32"), _rows(run, "enc.om16")
    ref, e = B.ln(sd, de + "enc_output.norm", ey_, None, 1e-5, False)
    _check(run, "enc_output norm (fp32)", om32, ref, e)
    _exact16(run, "enc_output norm fp16", om16, om32)
    lg = _rows(run, "enc.logits")
    ref, e = _lin_sd(sd, de + "enc_score_head", om16, False)
    _check(run, "encoder score head", lg[:, :C], ref, e)
    _zero_pad_cols(run, "encoder score head", lg, C)
    # the selected queries: tgt = om32[rows of topk]; the encoder box head and ref0
    topk = torch.from_numpy(run["m"].debug_tensor(n, "topk").view(np.int32).reshape(n, K).astype(np.int64)).to(DEV)
    rows = torch.cat([order.reshape(n, -1)[i][topk[i]] for i in range(n)])
    x_in, x_in16 = _rows(run, "dec0.x_in"), _rows(run, "dec0.x_in16")
    assert torch.equal(x_in, om32[rows]) and torch.equal(x_in16, om16[rows])
    h1, h2, delta = _rows(run, "enc.h1"), _rows(run, "enc.h2"), _rows(run, "enc.delta")
    bh = de + "enc_bbox_head.layers."
    ref, e = _lin_sd(sd, bh + "0", x_in16, act="relu")
    _check(run, "encoder box MLP layer 0 (ReLU)", h1, ref, e)
    ref, e = _lin_sd(sd, bh + "1", h1, act="relu")
    _check(run, "encoder box MLP layer 1 (ReLU)", h2, ref, e)
    ref, e = _lin_sd(sd, bh + "2", h2, False)
    _check(run, "encoder box MLP layer 2", delta, ref, e)
    asel = _rows(run, "anchor_sel")
    t = delta + asel
    s = torch.sigmoid(t)
    fin = torch.isfinite(t)
    ref0 = _rows(run, "ref0")
    assert bool((ref0[~fin] == 1.0).all())
    _check(run, "ref_update (anchors)", ref0[fin], s[fin], _ref_tol(t[fin], s[fin], 0.0))
    assert torch.equal(ref0, _rows(run, "dec0.ref"))
    _report(run)


# ------------------------------------------------------------------------------------------------------ decoder layers
def _split_ow(spec, ow, n, K):
    H, P = spec.heads, sum(spec.num_points)
    return ow[:, :H * P * 2].reshape(n, K, H, P, 2), ow[:, H * P * 2:H * P * 3].reshape(n, K, H, P)


def _value(run, val, i):
    """(n, total, heads, hd) of decoder layer i's value block"""
    n = run["n"]
    v = val[:, i * D:(i + 1) * D]
    return torch.stack([v[_level_rows(run, b)] for b in range(n)]).reshape(n, run["off"][-1], 8, D // 8)


def _qpos_l0(sd, ref):
    W, b = sd["decoder.query_pos_head.layers.0.weight"], sd["decoder.query_pos_head.layers.0.bias"]
    y = ref @ W.T + b
    Eq = 6 * 2.0 ** -24 * (ref.abs() @ W.abs().T + b.abs())
    want = y.clamp(min=0)
    ulp = torch.ldexp(torch.ones_like(want), torch.frexp((want + Eq).clamp(min=2.0 ** -14))[1] - 11)
    return want, 0.5 * ulp + Eq


def _layer_chain(run, i, x_in, x16, ref, val, sd):
    """whole decoder layer i (and its box refinement) from (x_in, its fp16 copy x16, ref), root-sum-square, with the
    engine's fp16 roundings of intermediate values as error terms: (x3, e_x3, bound of x3's fp16 copy, next ref, its
    bound) at 1 sigma"""
    spec, n = run["spec"], run["n"]
    K = spec.num_queries
    p = "decoder.decoder.layers.%d" % i
    qp0, e0 = _qpos_l0(sd, ref)
    qp, eqp = _lin_sd(sd, "decoder.query_pos_head.layers.1", qp0, e_x=e0, rss=True)
    tq = x16 + qp
    etq = eqp + U * tq.abs()
    W, b = sd[p + ".self_attn.in_proj_weight"], sd[p + ".self_attn.in_proj_bias"]
    qk, eqk = B.lin(tq, etq, W[:2 * D], b[:2 * D], True, rss=True)
    v, ev = B.lin(x16, None, W[2 * D:], b[2 * D:], True, rss=True)
    ap, ep = [], []
    for im in range(n):
        r = slice(im * K, (im + 1) * K)
        o, eo = B.attend(qk[r, :D], qk[r, D:], v[r], spec.heads, eqk[r, :D], eqk[r, D:], ev[r], rss=True)
        ap.append(o)
        ep.append(eo)
    y1, ey1 = _lin_sd(sd, p + ".self_attn.out_proj", torch.cat(ap), False, e_x=torch.cat(ep), resid=x_in, rss=True)
    x1, ex1 = B.ln(sd, p + ".norm1", y1, ey1, 1e-5, False, rss=True)
    tq2 = x1 + qp
    etq2 = ex1 + U * x1.abs() + SUB + eqp + U * tq2.abs()
    ca = p + ".cross_attn"
    Wow = torch.cat([sd[ca + ".sampling_offsets.weight"], sd[ca + ".attention_weights.weight"]])
    bow = torch.cat([sd[ca + ".sampling_offsets.bias"], sd[ca + ".attention_weights.bias"]])
    ow, eow = B.lin(tq2, etq2, Wow, bow, False, rss=True)
    off, lg = _split_ow(spec, ow, n, K)
    eoff, elg = _split_ow(spec, eow, n, K)
    samp, es = B.deform(spec, _value(run, val, i), run["shapes"], ref.reshape(n, K, 4), off, torch.softmax(lg, -1),
                        e_off=eoff, e_logit=elg, rss=True)
    samp, es = samp.reshape(n * K, D), es.reshape(n * K, D)
    y2, ey2 = _lin_sd(sd, ca + ".output_proj", samp, False, e_x=es, resid=x1, e_r=ex1, rss=True)
    x2, ex2 = B.ln(sd, p + ".norm2", y2, ey2, 1e-5, False, rss=True)
    f, ef = _lin_sd(sd, p + ".linear1", x2, e_x=ex2 + U * x2.abs() + SUB, act="relu", rss=True)
    y3, ey3 = _lin_sd(sd, p + ".linear2", f, False, e_x=ef, resid=x2, e_r=ex2, rss=True)
    x3, ex3 = B.ln(sd, p + ".norm3", y3, ey3, 1e-5, False, rss=True)
    ex3h = ex3 + U * x3.abs() + SUB                                  # the fp16 copy the box and score heads read
    bh = "decoder.dec_bbox_head.%d.layers." % i
    h1, eh1 = _lin_sd(sd, bh + "0", x3, e_x=ex3h, act="relu", rss=True)
    h2, eh2 = _lin_sd(sd, bh + "1", h1, e_x=eh1, act="relu", rss=True)
    dl, edl = _lin_sd(sd, bh + "2", h2, False, e_x=eh2, rss=True)
    base, eb = _refine_base(ref)
    t = dl + base
    s = torch.sigmoid(t)
    return x3, ex3, ex3h, s, s * (1 - s) * edl + _ref_tol(t, s, eb)


def test_decoder_layer_stages(run):
    sd, spec, n = run["sd64"], run["spec"], run["n"]
    K, C, NL = spec.num_queries, spec.num_classes, spec.num_layers
    val = _rows(run, "value")
    for i in range(NL):
        g = lambda k: _rows(run, "dec%d.%s" % (i, k))      # noqa: E731
        p = "decoder.decoder.layers.%d" % i
        x_in, x16, ref = g("x_in"), g("x_in16"), g("ref")
        _exact16(run, "x_in fp16", x16, x_in)
        qp0, qpos, qkv, att, y1 = g("qp0"), g("qpos"), g("qkv"), g("att"), g("y1")
        want, tol = _qpos_l0(sd, ref)
        _check(run, "query_pos layer 0 (qpos_l0)", qp0, want, tol)
        rf, e = _lin_sd(sd, "decoder.query_pos_head.layers.1", qp0)
        _check(run, "query_pos linear1", qpos, rf, e)
        tq = (x16.float() + qpos.float()).half().double()
        W, b = sd[p + ".self_attn.in_proj_weight"], sd[p + ".self_attn.in_proj_bias"]
        rf, e = B.lin(tq, None, W[:2 * D], b[:2 * D], True)
        _check(run, "decoder qk", qkv[:, :2 * D], rf, e)
        rf, e = B.lin(x16, None, W[2 * D:], b[2 * D:], True)
        _check(run, "decoder v", qkv[:, 2 * D:], rf, e)
        if i == 0:
            _miss(run, "decoder V from tgt + qpos", qkv[:, 2 * D:], B.lin(tq, None, W[2 * D:], b[2 * D:], True)[0], e)
        for im in range(n):
            r = slice(im * K, (im + 1) * K)
            rf, e = B.attend(qkv[r, :D], qkv[r, D:2 * D], qkv[r, 2 * D:], spec.heads)
            _check(run, "decoder self-attention (%d queries)" % K, att[r], rf, e)
        rf, e = _lin_sd(sd, p + ".self_attn.out_proj", att, False, resid=x_in)
        _check(run, "decoder out_proj + residual", y1, rf, e)
        x1, x1h = g("x1"), g("x1_16")
        rf, e = B.ln(sd, p + ".norm1", y1, None, 1e-5, False)
        _check(run, "decoder norm1 (fp32)", x1, rf, e)
        _exact16(run, "norm1 fp16", x1h, x1)
        ow, samp, y2 = g("ow"), g("samp"), g("y2")
        ca = p + ".cross_attn"
        Wow = torch.cat([sd[ca + ".sampling_offsets.weight"], sd[ca + ".attention_weights.weight"]])
        bow = torch.cat([sd[ca + ".sampling_offsets.bias"], sd[ca + ".attention_weights.bias"]])
        tq2 = (x1h.float() + qpos.float()).half().double()
        rf, e = B.lin(tq2, None, Wow, bow, False)
        _check(run, "sampling offsets / attention weights (ow)", ow, rf, e)
        if i == 0:
            _miss(run, "cross-attention query without qpos", ow, B.lin(x1h, None, Wow, bow, False)[0], e)
        off, lg = _split_ow(spec, ow, n, K)
        wts = torch.softmax(lg, -1)
        r4 = ref.reshape(n, K, 4)
        rf, e = B.deform(spec, _value(run, val, i), run["shapes"], r4, off, wts)
        rf, e = rf.reshape(n * K, D), e.reshape(n * K, D)
        _check(run, "deformable attention", samp, rf, e)
        if i == 1:
            for j in (i - 1, i + 1):
                w = R.deform_core(spec, _value(run, val, j), run["shapes"], r4, off, wts).reshape(n * K, D)
                _miss(run, "value block i %+d" % (j - i), samp, w, e)
            P = torch.tensor([n_ for n_ in spec.num_points for _ in range(n_)], dtype=torch.float64, device=DEV)
            w = R.deform_core(spec, _value(run, val, i), run["shapes"], r4, off * P[:, None], wts).reshape(n * K, D)
            _miss(run, "offsets without the 1 / num_points scale", samp, w, e)
        rf, e = _lin_sd(sd, ca + ".output_proj", samp, False, resid=x1)
        _check(run, "cross-attention output_proj + residual", y2, rf, e)
        x2, x2h, ffn, y3, x3, x3h = g("x2"), g("x2_16"), g("ffn"), g("y3"), g("x3"), g("x3_16")
        rf, e = B.ln(sd, p + ".norm2", y2, None, 1e-5, False)
        _check(run, "decoder norm2 (fp32)", x2, rf, e)
        _exact16(run, "norm2 fp16", x2h, x2)
        rf, e = _lin_sd(sd, p + ".linear1", x2h, act="relu")
        _check(run, "decoder linear1 (ReLU)", ffn, rf, e)
        rf, e = _lin_sd(sd, p + ".linear2", ffn, False, resid=x2)
        _check(run, "decoder linear2 + residual", y3, rf, e)
        rf, e = B.ln(sd, p + ".norm3", y3, None, 1e-5, False)
        _check(run, "decoder norm3 (fp32)", x3, rf, e)
        _exact16(run, "norm3 fp16", x3h, x3)
        h1, h2, delta, nref = g("h1"), g("h2"), g("delta"), _rows(run, "dec%d.ref" % (i + 1))
        bh = "decoder.dec_bbox_head.%d.layers." % i
        rf, e = _lin_sd(sd, bh + "0", x3h, act="relu")
        _check(run, "box MLP layer 0 (ReLU)", h1, rf, e)
        rf, e = _lin_sd(sd, bh + "1", h1, act="relu")
        _check(run, "box MLP layer 1 (ReLU)", h2, rf, e)
        rf, e = _lin_sd(sd, bh + "2", h2, False)
        _check(run, "box MLP layer 2", delta, rf, e)
        base, eb = _refine_base(ref)
        t = delta + base
        s = torch.sigmoid(t)
        tol = _ref_tol(t, s, eb)
        _check(run, "ref_update (refinement)", nref, s, tol)
        if i == 0:
            _miss(run, "ref not refreshed between layers", nref, ref, tol)
        # composite: the whole layer from (x_in, ref)
        cx3, ex3, e16, cref, eref = _layer_chain(run, i, x_in, x16, ref, val, sd)
        _check(run, "whole decoder layer x3 (composite, 6 sigma)", x3, cx3, B.LAMBDA * ex3)
        _check(run, "whole decoder layer next ref (composite, 6 sigma)", nref, cref, B.LAMBDA * eref)
        if i == NL - 1:
            bad = dict(sd)
            for k in ("weight", "bias"):
                bad["%s.norm2.%s" % (p, k)], bad["%s.norm3.%s" % (p, k)] = sd["%s.norm3.%s" % (p, k)], sd["%s.norm2.%s" % (p, k)]
            w3, *_ = _layer_chain(run, i, x_in, x16, ref, val, bad)
            _miss(run, "norm2 / norm3 swapped (composite)", x3, w3, B.LAMBDA * ex3)
            # the final logits and boxes from the last layer's input
            lgt = _rows(run, "logits")
            sh = "decoder.dec_score_head.%d" % i
            rf, e = _lin_sd(sd, sh, x3h, False)
            _check(run, "last score head", lgt[:, :C], rf, e)
            _zero_pad_cols(run, "last score head", lgt, C)
            assert torch.equal(run["out"]["pred_logits"].reshape(n * K, C), lgt[:, :C])
            assert torch.equal(run["out"]["pred_boxes"].reshape(n * K, 4), nref)
            rf, e = _lin_sd(sd, sh, cx3, False, e_x=e16, rss=True)
            _check(run, "final logits (composite, 6 sigma)", lgt[:, :C], rf, B.LAMBDA * e)
            _check(run, "final boxes (composite, 6 sigma)", run["out"]["pred_boxes"].reshape(n * K, 4), cref,
                   B.LAMBDA * eref)
    _report(run)


# ------------------------------------------------------------------------------------------------------ capture
def _names(spec):
    """every stage name the hook exposes: the engine's buffers and its captures"""
    out = ["input", "stem1", "stem2", "stem3", "pool", "cat3", "cat4", "pcat4", "pcat5", "proj5", "fpn4", "enc_out3",
           "enc_out4", "enc_out5", "memory", "value", "enc.y", "enc.om32", "enc.om16", "enc.logits", "enc.scores",
           "topk", "anchor_sel", "ref", "logits", "aifi.y1", "enc.h1", "enc.h2", "enc.delta", "ref0"]
    out += ["aifi." + k for k in ("q", "qkv", "att", "y", "s32", "s16", "ffn", "out")]
    for s_, nb in enumerate(spec.blocks):
        for b in range(nb):
            nm = "res%d.%d" % (s_, b)
            out += [nm, nm + ".a", nm + ".b"] + ([nm + ".short"] if b == 0 else []) + \
                ([nm + ".pool"] if b == 0 and s_ else [])
    out += ["%s.%s" % (c, k) for c in ("fpn0", "fpn1", "pan0", "pan1") for k in ("c1", "r0", "r1", "t2", "x2")]
    for i in range(spec.num_layers):
        out += ["dec%d.%s" % (i, k) for k in ("x_in", "x_in16", "ref", "qp0", "qpos", "qkv", "att", "y1", "x1", "x1_16",
                                               "ow", "samp", "y2", "x2", "x2_16", "ffn", "y3", "x3", "x3_16", "h1",
                                               "h2", "delta")]
    return out + ["dec%d.ref" % spec.num_layers]


CAPTURED_ONLY = ("fpn0.c1", "pan1.r1", "aifi.y1", "enc.delta", "ref0", "dec0.x_in", "dec5.ffn", "dec6.ref")


def _kernels(m, x):
    """(outputs, kernels the profiler saw, launches the library counted) of one forward"""
    from torch.profiler import ProfilerActivity, profile
    c0 = _lib.lib().ytk_launch_count()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = m(x)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    k = sum(1 for nm in names if not nm.startswith(("Memcpy", "Memset")))
    return {a: b.cpu() for a, b in out.items()}, k, _lib.lib().ytk_launch_count() - c0


def test_capture_changes_nothing_and_refusals():
    """Capture on and off: pred_logits and pred_boxes bit-equal, the same kernels launched.  The read-out refuses a
    batch size that has not run (or was evicted), a captured name after a forward without capture, and null
    arguments; a null host_out is a shape query."""
    _RUNS.clear()
    m, sd, x = _model(LayoutParserRTDETRv2V2Config, R.SPECS["layout"], 34, 1)
    L = _lib.lib()
    h = m._ensure()
    shape = (ctypes.c_int * 4)()
    assert L.ytk_rtdetr_debug_tensor(h, 1, b"enc.scores", None, 0, shape) != 0
    assert b"no engine for batch size 1" in L.ytk_last_error()
    assert m.flops(1) > 0                                            # builds the engine without running it
    assert L.ytk_rtdetr_debug_tensor(h, 1, b"enc.scores", None, 0, shape) != 0
    assert b"no forward of this batch size" in L.ytk_last_error()
    for args in ((None, 1, b"c3", None, 0, shape), (h, 1, None, None, 0, shape), (h, 1, b"c3", None, 0, None)):
        assert L.ytk_rtdetr_debug_tensor(*args) != 0 and b"null argument" in L.ytk_last_error()
    assert L.ytk_rtdetr_set_debug(None, 1) != 0
    xs = x.to(DEV)
    res = []
    for on in (False, True, False):
        m.set_debug(on)
        res.append(_kernels(m, xs))
        for nm in CAPTURED_ONLY:
            if on:
                assert m.debug_tensor(1, nm).size > 0
            else:
                with pytest.raises(_lib.YtkError, match="captured only when"):
                    m.debug_tensor(1, nm)
        assert m.debug_tensor(1, "c3").shape == (1, 80, 80, 512)     # the engine's own buffers read either way
    (o0, k0, n0), (o1, k1, n1), (o2, k2, n2) = res
    for a in (o1, o2):
        for key in ("pred_logits", "pred_boxes"):
            assert torch.equal(o0[key].view(torch.int32), a[key].view(torch.int32)), key
    print("[rt-stages] kernels per forward (off, on, off): profiler %d %d %d, library count %d %d %d"
          % (k0, k1, k2, n0, n1, n2))
    assert k0 == k1 == k2 and n0 == n1 == n2 and k0 > 0 and n0 > 0
    assert L.ytk_rtdetr_debug_tensor(h, 1, b"c3", None, 0, shape) == 0 and list(shape) == [1, 80, 80, 512]
    buf = torch.empty(10, dtype=torch.float32)
    assert L.ytk_rtdetr_debug_tensor(h, 1, b"c3", ctypes.c_void_p(buf.data_ptr()), 10, shape) != 0
    assert b"capacity" in L.ytk_last_error()
    for bad in ("dec6.x3", "res4.0", "nothing"):
        with pytest.raises(_lib.YtkError, match="unknown name"):
            m.debug_tensor(1, bad)
    # four more batch sizes evict batch size 1's engine (the handle keeps 4)
    for nb in (2, 3, 4, 5):
        m(xs.repeat(nb, 1, 1, 1))
    with pytest.raises(_lib.YtkError, match="no engine for batch size 1"):
        m.debug_tensor(1, "c3")


def test_forward_u8_captures_equal_forward_f32():
    """forward_u8 on two pages of other sizes, with capture: every stage equals forward_f32's on the engine's packed
    input of that call (the fp16 pixels, exact in fp32), bit for bit."""
    _RUNS.clear()
    from yomitoku_b200.layout_parser import rtdetr_sources
    spec = R.SPECS["layout"]
    m, _, _ = _model(LayoutParserRTDETRv2V2Config, spec, 35, 2)
    rng = np.random.default_rng(3)
    pages = [rng.integers(0, 256, (700, 500, 3), dtype=np.uint8), rng.integers(0, 256, (480, 900, 3), dtype=np.uint8)]
    recs, _ = rtdetr_sources([p.shape for p in pages], [(0, (0, 0, 500, 700)), (1, (30, 20, 880, 470))])
    m.set_debug(True)
    o8 = m.forward_u8(np.concatenate([p.reshape(-1) for p in pages]), recs)
    names = _names(spec)
    a = {k: m.debug_tensor(2, k) for k in names}
    x = torch.from_numpy(a["input"][..., :3]).permute(0, 3, 1, 2).contiguous()
    o32 = m(x.to(DEV))
    for key in ("pred_logits", "pred_boxes"):
        assert torch.equal(o8[key].view(torch.int32), o32[key].cpu().view(torch.int32)), key
    for k in names:
        assert np.array_equal(a[k].view(np.uint32), m.debug_tensor(2, k).view(np.uint32)), k
