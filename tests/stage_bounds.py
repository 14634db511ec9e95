"""Error bounds of the engines' stages against a float64 restatement (shared by the stage-by-stage GPU tests and checked
on the CPU by tests/test_stage_bounds_host.py).  Every function returns the float64 result of the stage on the engine's
own input and a componentwise bound on how far a correct kernel may lie from it.

Notation: u = 2^-11 (fp16 rounding, to nearest), e = 2^-24 (fp32 rounding), g(n) = n 2^-23 (n fp32 additions, each
within one unit of a 24-bit significand as truncating tensor-core adders give), s = 2^-25 (half the fp16 subnormal
spacing).  |.| is elementwise, e_x the bound carried by an input x (zero when x is the engine's own stored value).

  GEMM y = x W^T + b (+ r), fp16 operands, fp32 accumulation over K (padded to 64):         lin
      S = |x| |W|^T,  e_pre = e_x |W|^T + (u + e) S + s sum|x| + g(K) S + 2^-23 (S + |b| + |r|) + e_r
      (the weight's fp16 rounding; the accumulation; bias and residual adds)
      GELU epilogue: e_y = 1.13 e_pre + 5e-7 + e |y| (1.13 = max |GELU'|, 5e-7 = gelu_fast's maximum error);
      output: + u |y| + s (fp16) or + e |y| (fp32).
  Convolution (implicit GEMM, K = k^2 Cin with Cin padded to 64):                            conv
      the GEMM rule with S = conv2d(|x|, |W|) and sum|x| over the receptive field, and W the float64 BatchNorm-folded
      (for RepVGG, branch-summed) weight.  The engine folds in fp32 (scale = g / sqrt(v + eps): three roundings, the
      product w scale one more, the RepVGG centre sum one more) and rounds to fp16, so the weight term is (u + 8 e) S;
      the folded bias b - m scale carries 8 e (|b| + |m scale|).
      ReLU is 1-Lipschitz and exact.  SiLU epilogue __fdividef(v, 1 + __expf(-v)): __expf is within (2 + 1.16 |v|) ulp
      (the model of test_gpu_dbnet_kernels.py), 1 + t rounds once and __fdividef is within 2 ulp, so
      e_y = 1.1 e_pre + |y| ((1 - sig(v)) (2 + 1.16 |v|) 2^-23 + 2^-24 + 2^-22) + 2^-126   (1.1 > max |SiLU'|).
      The sigmoid epilogue __fdividef(1, 1 + __expf(-v)): e_y = e_pre / 4 + (2 + 1.16 |v|) 2^-25 + 2^-23.
  LayerNorm y = g (x - m) r + b over the D features, fp32 statistics:                           ln
      e_y = |g| r (e_x + mean(e_x) + |xh| mean(|xh| e_x))              (first-order propagation of the input bound)
          + |g| r D e mean|x| + (D + 16) e |g| |xh| + 2 e (|y| + |b|)   (fp32 sums, rsqrt, the final fma)
          + u |y| + s when the output is stored fp16.
  Attention o = softmax(q k^T / sqrt(hd)) v per head, p the float64 probabilities over the visible keys:    attend
      score error  d_j = (|q| |k_j| 2 hd 2^-23 + e_q |k_j| + |q| e_kj) / sqrt(hd) + 4 e |s_j| + 2^-21  (ex2.approx)
      D = max_j d_j,  P = p |v|:
      e_o = (exp(2 D) - 1) P + p e_v + (u + g(Lk) + 8 e) P + s sum_j |v_j| + u |o| + s
  Deformable sampling (bilinear, zero padding, align_corners False):                      sample_shift, deform
      a location error e_loc (in [0, 1] units) moves a bilinear sample of level l (W_l x H_l) by at most
      W_l max|v(x + 1) - v(x)| e_loc,x + H_l max|v(y + 1) - v(y)| e_loc,y, the maxima over the differences of the
      sample's corner values and of the neighbouring cells (a shift of under one pixel may cross a cell edge), in
      float64 from the value tensor.  An offset error e_off gives e_loc = e_off / num_points * ref_wh * offset_scale.
      A softmax weight with logit errors e_l moves by at most w (exp(2 max e_l) - 1).  The kernel's own arithmetic
      (test_gpu_decoder_kernels.py) adds 2^-10 max|v| + 2^-11 |o|.
  A composite stage chains these rules.  Carried through several GEMMs, worst-case propagation (e_x |W|^T) grows by
  about sqrt(K) |W| per layer and says nothing; the chain instead uses the probabilistic model of rounding-error
  analysis (Higham & Mary, SIAM J. Sci. Comput. 41 (2019)): the errors of distinct features are independent and
  zero-mean, so an input bound propagates in root-sum-square, sqrt(e_x^2 (W^2)^T) (likewise through LayerNorm's mean
  terms, the scores, p v and the sum over sampling points), every local term keeps its local size above except that
  the sums over K in S = |x| |W|^T and P = p |v| become root-sum-squares too (sqrt(x^2 (W^2)^T), sqrt(p^2 v^2), and
  g(K) becomes sqrt(K) g(1)), and the result sigma is treated as a standard deviation: |d| <= LAMBDA sigma, LAMBDA = 6.
"""
import math

import torch
import torch.nn.functional as F

from oracle import parseq as _pq

U, E, G, SUB = 2.0 ** -11, 2.0 ** -24, 2.0 ** -23, 2.0 ** -25
LAMBDA = 6.0
WFOLD = U + 8 * E            # a BatchNorm-folded fp32 weight rounded to fp16, relative


def _prop(e, M, rss):
    """input bound e through the linear map M^T: worst case e |M|^T, or root-sum-square sqrt(e^2 (M^2)^T)"""
    return torch.sqrt((e * e) @ (M * M).T) if rss else e @ M.abs().T


def _out(y, e, out16):
    return e + (U * y.abs() + SUB if out16 else E * y.abs())


def _act_bound(pre, e, act):
    """(y, e_y) of an epilogue activation of pre carrying the bound e"""
    if act is None:
        return pre, e
    if act == "relu":
        return F.relu(pre), e
    if act == "gelu":
        y = F.gelu(pre)
        return y, 1.13 * e + 5e-7 + E * y.abs()
    if act == "silu":
        y = F.silu(pre)
        return y, 1.1 * e + silu_term(pre, y)
    if act == "sigmoid":
        y = torch.sigmoid(pre)
        return y, e / 4 + sigmoid_term(pre)
    raise ValueError(act)


def silu_term(v, y=None):
    """arithmetic error of the SiLU epilogue __fdividef(v, 1 + __expf(-v)) at the exact argument v"""
    y = F.silu(v) if y is None else y
    return y.abs() * ((1 - torch.sigmoid(v)) * (2 + 1.16 * v.abs()) * G + E + 2 * G) + 2.0 ** -126


def sigmoid_term(v):
    """arithmetic error of the sigmoid epilogue __fdividef(1, 1 + __expf(-v)) at the exact argument v"""
    return (2 + 1.16 * v.abs()) * 2.0 ** -25 + 2 * G


def lin(x, e_x, W, b, out16, resid=None, e_r=None, gelu=False, rss=False, act=None):
    """float64 x W^T + b (+ resid) (activation) and its bound (module docstring)."""
    pre = x @ W.T + b
    if resid is not None:
        pre = pre + resid
    S = x.abs() @ W.abs().T
    K = (W.shape[1] + 63) // 64 * 64
    if rss:     # independent weight roundings and accumulation errors: root-sum-square, sqrt(K) g(1) S
        R = torch.sqrt((x * x) @ (W * W).T)
        e = (U + E) * R + SUB * x.norm(dim=-1, keepdim=True) + math.sqrt(K) * G * S + \
            G * (R + b.abs() + (resid.abs() if resid is not None else 0))
    else:
        e = (U + E) * S + SUB * x.abs().sum(-1, keepdim=True) + K * G * S + \
            G * (S + b.abs() + (resid.abs() if resid is not None else 0))
    if e_x is not None:
        e = e + _prop(e_x, W, rss)
    if e_r is not None:
        e = e + e_r
    y, e = _act_bound(pre, e, "gelu" if gelu else act)
    return y, _out(y, e, out16)


def conv(x, e_x, W, b, stride, out16, resid=None, e_r=None, act=None, e_b=None, rss=False):
    """float64 conv2d(x, W) + b (+ resid) (activation) on NCHW x and its bound (module docstring).  W is the float64
    folded weight; e_b the folded bias's bound (see fold_bn)."""
    k = W.shape[-1]
    pad = (k - 1) // 2
    pre = F.conv2d(x, W, b, stride, pad)
    if resid is not None:
        pre = pre + resid
    S = F.conv2d(x.abs(), W.abs(), None, stride, pad)
    ones = torch.ones((1,) + tuple(W.shape[1:]), dtype=x.dtype, device=x.device)
    K = k * k * ((W.shape[1] + 63) // 64 * 64)
    bb = b.abs().view(1, -1, 1, 1)
    r_abs = resid.abs() if resid is not None else 0
    if rss:
        R = torch.sqrt(F.conv2d(x * x, W * W, None, stride, pad))
        e = WFOLD * R + SUB * torch.sqrt(F.conv2d(x * x, ones, None, stride, pad)) + math.sqrt(K) * G * S + \
            G * (R + bb + r_abs)
    else:
        e = WFOLD * S + SUB * F.conv2d(x.abs(), ones, None, stride, pad) + K * G * S + G * (S + bb + r_abs)
    if e_b is not None:
        e = e + e_b.view(1, -1, 1, 1)
    if e_x is not None:
        e = e + (torch.sqrt(F.conv2d(e_x * e_x, W * W, None, stride, pad)) if rss else
                 F.conv2d(e_x, W.abs(), None, stride, pad))
    if e_r is not None:
        e = e + e_r
    y, e = _act_bound(pre, e, act)
    return y, _out(y, e, out16)


def fold_bn(sd, p, w):
    """(W * scale, shift, bound of the fp32 shift) of a conv weight w followed by BatchNorm p, in float64"""
    scale = sd[p + ".weight"] / torch.sqrt(sd[p + ".running_var"] + 1e-5)
    shift = sd[p + ".bias"] - sd[p + ".running_mean"] * scale
    return w * scale.view(-1, 1, 1, 1), shift, 8 * E * (sd[p + ".bias"].abs() + (sd[p + ".running_mean"] * scale).abs())


def fold_conv_norm(sd, p):
    return fold_bn(sd, p + ".norm", sd[p + ".conv.weight"])


def fold_repvgg(sd, b, tap=None):
    """RepVgg block b as one 3x3 weight: the 1x1 branch added at the centre tap (tap = (r, s): another tap, for a wrong
    reference)"""
    w3, b3, e3 = fold_conv_norm(sd, b + ".conv1")
    w1, b1, e1 = fold_conv_norm(sd, b + ".conv2")
    r, s = (1, 1) if tap is None else tap
    w = w3.clone()
    w[:, :, r, s] += w1[:, :, 0, 0]
    return w, b3 + b1, e3 + e1


def ln(sd, name, x, e_x, eps, out16, rss=False):
    y = _pq.layer_norm(sd, name, x, eps)
    g, bb = sd[name + ".weight"], sd[name + ".bias"]
    D = x.shape[-1]
    mu = x.mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + eps)
    xh = (x - mu) * r
    e = g.abs() * r * D * E * x.abs().mean(-1, keepdim=True) + (D + 16) * E * g.abs() * xh.abs() + 2 * E * (y.abs() + bb.abs())
    if e_x is not None:
        if rss:
            m1, m2 = e_x.norm(dim=-1, keepdim=True) / D, (xh * e_x).norm(dim=-1, keepdim=True) / D
        else:
            m1, m2 = e_x.mean(-1, keepdim=True), (xh.abs() * e_x).mean(-1, keepdim=True)
        e = e + g.abs() * r * (e_x + m1 + xh.abs() * m2)
    if out16:
        e = e + U * y.abs() + SUB
    return y, e


def attend(q, k, v, heads, e_q=None, e_k=None, e_v=None, amask=None, pmask=None, rss=False):
    """oracle.parseq.mha_attend for one batch row (q (Lq, D), k / v (Lk, D)) and its bound."""
    o = _pq.mha_attend(q[None], k[None], v[None], heads, amask, None if pmask is None else pmask[None])[0]
    Lq, D = q.shape
    Lk = k.shape[0]
    hd = D // heads
    H = lambda t, n: t.reshape(n, heads, hd).transpose(0, 1)      # noqa: E731
    qh, kh, vh = H(q, Lq), H(k, Lk), H(v, Lk)
    s = qh @ kh.transpose(-1, -2) / math.sqrt(hd)
    vis = torch.ones(Lq, Lk, dtype=torch.bool, device=q.device)
    if amask is not None:
        vis &= ~amask
    if pmask is not None:
        vis = vis & ~pmask[None, :]
    vis = vis[None].expand(heads, -1, -1)
    p = torch.softmax(s.masked_fill(~vis, float("-inf")), -1)
    d = (qh.abs() @ kh.abs().transpose(-1, -2)) * (2 * hd * G) / math.sqrt(hd) + 4 * E * s.abs() + 2.0 ** -21
    sq = (lambda a, b: torch.sqrt((a * a) @ (b * b).transpose(-1, -2))) if rss else \
        (lambda a, b: a.abs() @ b.abs().transpose(-1, -2))
    if e_q is not None:
        d = d + sq(H(e_q, Lq), kh) / math.sqrt(hd)
    if e_k is not None:
        d = d + sq(qh, H(e_k, Lk)) / math.sqrt(hd)
    dmax = d.masked_fill(~vis, 0).amax(-1, keepdim=True)
    P = torch.sqrt((p * p) @ (vh * vh)) if rss else p @ vh.abs()
    e = (torch.exp(2 * dmax) - 1) * P + (U + Lk * G + 8 * E) * P + SUB * (vis.double() @ vh.abs())
    if e_v is not None:
        e = e + (torch.sqrt((p * p) @ H(e_v * e_v, Lk)) if rss else p @ H(e_v, Lk))
    e = e.transpose(0, 1).reshape(Lq, D)
    return o, e + U * o.abs() + SUB


def sample_shift(v, loc, e_loc):
    """How far a location error moves bilinear samples (grid_sample, zeros padding, align_corners False).

    v (M, c, h, w) float64 values of one level; loc (M, Q, 2) sampling locations (x, y) in [0, 1] units; e_loc
    (M, Q, 2) their bounds.  Returns (M, c, Q): w max|dx v| e_x + h max|dy v| e_y over the sample's corner differences
    and the neighbouring cells' (module docstring)."""
    M, c, h, w = v.shape
    vp = F.pad(v, (2, 2, 2, 2))                                    # the zeros outside the level, two cells deep
    dx = (vp[..., :, 1:] - vp[..., :, :-1]).abs()                  # (h + 4, w + 3): column j pairs padded j, j + 1
    dy = (vp[..., 1:, :] - vp[..., :-1, :]).abs()                  # (h + 3, w + 4)
    mx = F.max_pool2d(dx, (2, 3), 1)                               # rows r, r + 1; columns c - 1 .. c + 1 of the cell
    my = F.max_pool2d(dy, (3, 2), 1)
    px, py = loc[..., 0] * w - 0.5, loc[..., 1] * h - 0.5
    x0, y0 = torch.floor(px).long(), torch.floor(py).long()

    def at(m, r, col):
        r = r.clamp(0, m.shape[-2] - 1)
        col = col.clamp(0, m.shape[-1] - 1)
        idx = (r * m.shape[-1] + col)[:, None, :].expand(-1, c, -1)
        return m.flatten(2).gather(2, idx)

    gx = at(mx, y0 + 2, x0 + 1)                                     # corners y0, y0 + 1 sit at padded rows y0 + 2, + 3
    gy = at(my, y0 + 1, x0 + 2)
    return w * gx * e_loc[:, None, :, 0] + h * gy * e_loc[:, None, :, 1]


def deform(spec, value, shapes, ref4, off, wts, e_off=None, e_logit=None, rss=False):
    """oracle.rtdetr.deform_core on (B, Q, .) operands and its bound: the kernel's own arithmetic, the sample shifts of
    the offset bounds e_off (B, Q, heads, P, 2) and the weight changes of the attention-logit bounds e_logit
    (B, Q, heads, P)."""
    from oracle import rtdetr as R
    out = R.deform_core(spec, value, shapes, ref4, off, wts)
    vmax = value.abs().max()
    e = 2.0 ** -10 * vmax + 2.0 ** -11 * out.abs()
    if e_off is None and e_logit is None:
        return out, e
    B, Q, H, P = wts.shape
    c = value.shape[-1]
    loc = R.deform_locations(spec, ref4, off)                       # (B, Q, H, P, 2)
    vals = value.permute(0, 2, 3, 1).flatten(0, 1).split([h * w for h, w in shapes], dim=-1)
    samples, shifts, p0 = [], [], 0
    for l, (h, w) in enumerate(shapes):
        n = spec.num_points[l]
        vl = vals[l].reshape(B * H, c, h, w)
        ll = loc[:, :, :, p0:p0 + n].permute(0, 2, 1, 3, 4).reshape(B * H, Q * n, 2)
        g = (2 * ll - 1)[:, :, None, :]
        samples.append(F.grid_sample(vl, g, mode="bilinear", padding_mode="zeros", align_corners=False)[..., 0])
        if e_off is not None:
            sc = (ref4[:, :, None, None, 2:] * spec.offset_scale / n).expand(-1, -1, H, n, -1)
            el = (e_off[:, :, :, p0:p0 + n] * sc).permute(0, 2, 1, 3, 4).reshape(B * H, Q * n, 2)
            shifts.append(sample_shift(vl, ll, el))
        p0 += n
    samp = torch.cat([s.reshape(B * H, c, Q, -1) for s in samples], -1)     # (B H, c, Q, P)
    w_ = wts.permute(0, 2, 1, 3).reshape(B * H, 1, Q, P)
    terms = []
    if e_off is not None:
        terms.append(w_ * torch.cat([s.reshape(B * H, c, Q, -1) for s in shifts], -1))
    if e_logit is not None:
        dw = w_ * (torch.exp(2 * e_logit.amax(-1, keepdim=True)) - 1).permute(0, 2, 1, 3).reshape(B * H, 1, Q, 1)
        terms.append(dw * samp.abs())
    t = sum(terms)
    t = torch.sqrt((t * t).sum(-1)) if rss else t.sum(-1)           # (B H, c, Q)
    return out, e + t.reshape(B, H * c, Q).permute(0, 2, 1)
