"""GPU: the PARSeq engine stage by stage against float64, every stage fed the engine's own input to it.

The engine (csrc/parseq_engine.cu) exposes its stages through PARSeq.set_debug / PARSeq.debug_tensor.  Each check below
takes the engine's input to one stage as read through that hook, runs the same stage of the one restatement of the
model (oracle/parseq.py: patch_embed, encoder_block, encoder_norm, content_embed, mha_q / mha_kv / mha_attend / mha_out,
mlp_hidden / mlp_out, final_norm, head) in float64 on the device, and compares.  Errors therefore do not accumulate
across stages, and every stage has its own a-priori componentwise bound, computed here from the operands.  The engine
runs some models zero-padded (parseq-tiny: D 368 as 384, heads of 46 as 48): its tensors are read at the padded width,
the padded columns must be exactly zero, and the comparison runs in the real model's feature space.

The bound rules are implemented in tests/stage_bounds.py (lin, ln, attend), shared with the RT-DETRv2 stage test.
Notation: u = 2^-11 (fp16 rounding, to nearest), e = 2^-24 (fp32 rounding), g(n) = n 2^-23 (n fp32 additions, each
within one unit of a 24-bit significand as truncating tensor-core adders give), s = 2^-25 (half the fp16 subnormal
spacing).  |.| is elementwise, e_x the bound carried by an input x (zero when x is the engine's own stored value).

  GEMM y = x W^T + b (+ r), fp16 operands, fp32 accumulation over K (padded to 64):
      S = |x| |W|^T,  e_pre = e_x |W|^T + (u + e) S + s sum|x| + g(K) S + 2^-23 (S + |b| + |r|) + e_r
      (the weight's fp16 rounding with the folded softmax / sqrt(D) scales; the accumulation; bias and residual adds)
      GELU epilogue: e_y = 1.13 e_pre + 5e-7 + e |y| (1.13 = max |GELU'|, 5e-7 = gelu_fast's maximum error);
      output: + u |y| + s (fp16) or + e |y| (fp32).
  LayerNorm y = g (x - m) r + b over the real D features, fp32 statistics:
      e_y = |g| r (e_x + mean(e_x) + |xh| mean(|xh| e_x))              (first-order propagation of the input bound)
          + |g| r D e mean|x| + (D + 16) e |g| |xh| + 2 e (|y| + |b|)   (fp32 sums, rsqrt, the final fma)
          + u |y| + s when the output is stored fp16.
  Attention o = softmax(q k^T / sqrt(hd)) v per head, p the float64 probabilities over the visible keys:
      score error  d_j = (|q| |k_j| 2 hd 2^-23 + e_q |k_j| + |q| e_kj) / sqrt(hd) + 4 e |s_j| + 2^-21  (ex2.approx)
      D = max_j d_j,  P = p |v|:
      e_o = (exp(2 D) - 1) P + p e_v + (u + g(Lk) + 8 e) P + s sum_j |v_j| + u |o| + s
      (a score perturbation of at most D moves every p_j by a factor within exp(+-2 D); the probabilities are rounded
      to fp16 for the P V product; the fp32 sums; the fp16 output).
  A composite stage (an encoder block, a whole AR step from its context tokens) chains these rules.  Carried through
  several GEMMs, worst-case propagation (e_x |W|^T) grows by about sqrt(K) |W| per layer and says nothing; the chain
  instead uses the probabilistic model of rounding-error analysis (Higham & Mary, SIAM J. Sci. Comput. 41 (2019)):
  the errors of distinct features are independent and zero-mean, so an input bound propagates in root-sum-square,
  sqrt(e_x^2 (W^2)^T) (likewise through LayerNorm's mean terms, the scores and p v), every local term keeps its
  local size above except that the sums over K in S = |x| |W|^T and P = p |v| become root-sum-squares too
  (sqrt(x^2 (W^2)^T), sqrt(p^2 v^2), and g(K) becomes sqrt(K) g(1)), and the result sigma is treated as a standard
  deviation: |d| <= 6 sigma.

The AR decode is checked teacher-forced: the decoder has depth 1 and never updates the content stream, so one causal
float64 decode over the engine's own context tokens ar.tgt gives the logits of every AR step it ran, with the chained
bound of a whole step.  With refine_iters = 0 the AR logits are compared directly; with refinement every AR decision
must be the float64 arg-max unless the float64 gap between the two tokens is within the sum of their two logit
bounds, e[a] + e[t] (a near-tie; their number is printed).

Every check prints the worst |d| / bound.  Wrong references (pos_queries row i + 1, norm1 / norm2 swapped, kpad one past
the first EOS, rows 0 and 1 not opened, the neighbouring crop's memory, pos_embed indexed with the crop's grid width)
must miss their bound on some element: the bounds are tight enough to see wiring mistakes of that size.  The composite
6-sigma bounds get wrong references too: an encoder block with norm1 / norm2 swapped, and whole AR steps with the
decoder's norm1 / norm2 swapped or pos_queries row i + 1 added at step i (the AR step pointer off by one)."""
import dataclasses
import math

import numpy as np
import pytest
import torch

from oracle import parseq as ops
from oracle import weights
from stage_bounds import E, LAMBDA, SUB, U, attend, lin, ln
from yomitoku_b200 import TextRecognizer, _lib

pytestmark = pytest.mark.gpu
DEV = "cuda"
SA, CA, DEC = ops.DEC + "self_attn.", ops.DEC + "cross_attn.", ops.DEC
RATIOS = {}         # stage -> worst |d| / bound
LOGIT_BOUNDS = {}   # configuration -> largest logit bound of a teacher-forced AR step (absolute, logits)


def _ratio(tag, got, ref, bound):
    r = float(((got - ref).abs() / bound).max()) if got.numel() else 0.0
    RATIOS[tag] = max(RATIOS.get(tag, 0.0), r)
    return r


def _check(tag, got, ref, bound):
    r = _ratio(tag, got, ref, bound)
    assert r <= 1.0, "%s: worst |d| / bound = %.3g" % (tag, r)
    return r


def _miss(tag, got, wrong, bound):
    """A wrong reference: the engine must lie outside its bound somewhere."""
    r = float(((got - wrong).abs() / bound).max())
    print("[stages] mutation %-34s worst |d| / bound %.3g (must exceed 1)" % (tag, r))
    assert r > 1.0, tag
    return r


# ------------------------------------------------------------------------------------------------------ layout
class Layout:
    """The engine's padded layout (ParseqModel::load): residual-stream tensors hold the real D features first; head
    tensors put real feature i of the decoder at (i / hd) hdp + i % hd; q projections carry sqrt(hdp / hd)."""

    def __init__(self, spec):
        D, he, hd = spec.embed_dim, spec.enc_heads, spec.dec_heads
        hd_e, hd_d = D // he, D // hd
        hdp_e = (hd_e + 15) // 16 * 16
        while (he * hdp_e) % 64:
            hdp_e += 16
        self.D, self.Dp = D, he * hdp_e
        hdp_d = self.Dp // hd
        self.hdm = torch.tensor([(i // hd_d) * hdp_d + i % hd_d for i in range(D)], device=DEV)
        self.qs = float(np.sqrt(np.float32(hdp_d) / np.float32(hd_d), dtype=np.float32)) if self.Dp != D else 1.0

    def _zero_rest(self, t, keep, tag):
        rest = torch.ones(t.shape[-1], dtype=torch.bool, device=t.device)
        rest[keep] = False
        if rest.any():
            assert (t[..., rest] == 0).all(), "%s: padded columns are not exactly zero" % tag

    def res(self, t, tag):
        self._zero_rest(t, torch.arange(self.D, device=t.device), tag)
        return t[..., :self.D]

    def heads(self, t, tag, scale=1.0):
        self._zero_rest(t, self.hdm, tag)
        return t[..., self.hdm] / scale

    def kv(self, t, tag):
        Dp = self.Dp
        return self.heads(t[..., :Dp], tag + ".k"), self.heads(t[..., Dp:], tag + ".v")


def _dbg(m, name):
    t = m.debug_tensor(name)
    return t if t.dtype == torch.int32 else t.to(DEV, torch.float64)


def _sd64(sd):
    return {k: v.to(DEV, torch.float64) for k, v in sd.items()}


# ------------------------------------------------------------------------------------------------------ encoder
def encoder_block(sd, spec, i, x):
    """ops.encoder_block for one crop (x (N, D), the engine's residual stream) and its chained bound."""
    p = "encoder.blocks.%d." % i
    D, heads = spec.embed_dim, spec.enc_heads
    ref = ops.encoder_block(sd, spec, i, x[None])[0]
    h, e_h = ln(sd, p + "norm1", x, None, 1e-6, True, rss=True)
    qkv, e_qkv = lin(h, e_h, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"], True, rss=True)
    sl = [slice(j * D, (j + 1) * D) for j in range(3)]
    att, e_att = attend(*(qkv[:, s] for s in sl), heads, *(e_qkv[:, s] for s in sl), rss=True)
    x2, e_x2 = lin(att, e_att, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"], False, resid=x, rss=True)
    h2, e_h2 = ln(sd, p + "norm2", x2, e_x2, 1e-6, True, rss=True)
    f, e_f = lin(h2, e_h2, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"], True, gelu=True, rss=True)
    y, e_y = lin(f, e_f, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"], False, resid=x2, e_r=e_x2, rss=True)
    assert (y - ref).abs().max() <= 1e-9 * (1 + ref.abs().max())      # the chain restates ops.encoder_block
    return ref, LAMBDA * e_y


def _swap_norms(sd, a, b):
    bad = dict(sd)
    for k in ("weight", "bias"):
        bad["%s.%s" % (a, k)], bad["%s.%s" % (b, k)] = sd["%s.%s" % (b, k)], sd["%s.%s" % (a, k)]
    return bad


def check_encoder(tag, m, sd, spec, lay, crops, img16=None, memory_out=None, mutate=False):
    """crops: [(tok_off, ntok, gw)].  img16: the seam's images rounded to fp16 (L = 0 against the patch embed)."""
    depth = spec.enc_depth
    xs = [lay.res(_dbg(m, "enc.x.%d" % L), "enc.x.%d" % L) for L in range(depth + 1)]
    mem = lay.res(_dbg(m, "enc.mem"), "enc.mem")
    mk, mv = lay.kv(_dbg(m, "enc.memkv"), "enc.memkv")
    if img16 is not None:
        x0 = ops.patch_embed(sd, spec, img16).reshape(-1, spec.embed_dim)
        W = sd["encoder.patch_embed.proj.weight"].reshape(spec.embed_dim, -1)
        B, N = img16.shape[0], x0.shape[0] // img16.shape[0]
        A = torch.nn.functional.unfold(img16, spec.patch, stride=spec.patch).transpose(1, 2).reshape(B * N, -1)
        pos = x0 - (A @ W.T + sd["encoder.patch_embed.proj.bias"])
        _, e0 = lin(A, None, W, sd["encoder.patch_embed.proj.bias"], False, resid=pos)
        _check(tag + " enc.x.0 (patch embed + pos)", xs[0], x0, e0)
        # wrong: pos_embed indexed with the crop's grid width in place of the model's full grid width
        gh, gw = spec.img_size[0] // spec.patch[0], img16.shape[-1] // spec.patch[1]
        fgh, fgw = spec.grid
        if gw < fgw:
            bad = dict(sd)
            flat = sd["encoder.pos_embed"].reshape(fgh * fgw, -1)
            pe = flat.clone().reshape(fgh, fgw, -1)
            pe[:gh, :gw] = flat[:gh * gw].reshape(gh, gw, -1)
            bad["encoder.pos_embed"] = pe.reshape(1, fgh * fgw, -1)
            _miss("pos_embed row gy*gw+gx", xs[0], ops.patch_embed(bad, spec, img16).reshape(-1, spec.embed_dim), e0)
    for L in range(1, depth + 1):
        for (t0, n, _) in crops:
            ref, e = encoder_block(sd, spec, L - 1, xs[L - 1][t0:t0 + n])
            _check(tag + " enc.x.L (block)", xs[L][t0:t0 + n], ref, e)
        if mutate and L == 1:      # the composite 6-sigma bound of a block still sees a swapped pair of norms
            t0, n, _ = crops[0]
            p = "encoder.blocks.0."
            wrong, e_w = encoder_block(_swap_norms(sd, p + "norm1", p + "norm2"), spec, 0, xs[0][t0:t0 + n])
            _miss("encoder norm1 / norm2 swapped (block)", xs[1][t0:t0 + n], wrong, e_w)
    ref, e = ln(sd, "encoder.norm", xs[depth], None, 1e-6, True)
    _check(tag + " enc.mem (final norm)", mem, ref, e)
    if memory_out is not None:
        ref32, e32 = ln(sd, "encoder.norm", xs[depth], None, 1e-6, False)
        _check(tag + " memory_out", memory_out.to(DEV, torch.float64), ref32, e32 + E * ref32.abs())
    (k, e_k), (v, e_v) = [lin(mem, None, sd[CA + "in_proj_weight"][j * spec.embed_dim:(j + 1) * spec.embed_dim],
                              sd[CA + "in_proj_bias"][j * spec.embed_dim:(j + 1) * spec.embed_dim], True)
                          for j in (1, 2)]
    assert torch.allclose(torch.cat(ops.mha_kv(sd, CA, mem), -1), torch.cat([k, v], -1), rtol=0, atol=1e-9)
    _check(tag + " enc.memkv", torch.cat([mk, mv], -1), torch.cat([k, v], -1), torch.cat([e_k, e_v], -1))
    return mem, mk, mv


# ------------------------------------------------------------------------------------------------------ constants
def check_constants(tag, m, sd, spec, lay):
    S, D = spec.max_label_length + 1, spec.embed_dim
    pos = sd["pos_queries"][0, :S]
    assert torch.equal(lay.res(_dbg(m, "model.pos_q"), "model.pos_q"), pos)
    emb = sd["text_embed.embedding.weight"]
    got = lay.res(_dbg(m, "model.embed"), "model.embed") * math.sqrt(lay.Dp)      # the kernels scale by sqrt(Dp)
    _check(tag + " model.embed * sqrt(Dp)", got, math.sqrt(D) * emb, 4 * E * math.sqrt(D) * emb.abs() + 1e-300)
    # q_self = fp16(sqrt(hdp/hd) * (W_q LN_q(pos_q) + b_q)): host LN in fp32, double accumulation
    qn, e_qn = ln(sd, DEC + "norm_q", pos, None, 1e-5, False)
    q = ops.mha_q(sd, SA, qn)
    Wq = sd[SA + "in_proj_weight"][:D]
    e_q = e_qn @ Wq.abs().T + 4 * E * q.abs() + U * q.abs() + SUB / lay.qs
    q_got = lay.heads(_dbg(m, "model.q_self"), "model.q_self", lay.qs)
    _check(tag + " model.q_self", q_got, q, e_q)
    bos = torch.full((1, 1), spec.bos_id, dtype=torch.long, device=DEV)
    c0, e_c0 = ln(sd, DEC + "norm_c", math.sqrt(D) * emb[spec.bos_id][None], None, 1e-5, False)
    assert torch.allclose(c0, ops.content_embed(sd, spec, bos)[0], rtol=0, atol=1e-12)
    k, v = ops.mha_kv(sd, SA, c0)
    Wkv = sd[SA + "in_proj_weight"][D:]
    kv = torch.cat([k, v], -1)
    e_kv = (e_c0 + 4 * E * math.sqrt(D) * emb[spec.bos_id].abs()) @ Wkv.abs().T + 4 * E * kv.abs() + U * kv.abs() + SUB
    kg, vg = lay.kv(_dbg(m, "model.ckv0"), "model.ckv0")
    _check(tag + " model.ckv0", torch.cat([kg, vg], -1), kv, e_kv)
    return q, e_q          # the float64 queries and the bound the engine's stored ones carry


# ------------------------------------------------------------------------------------------------------ decoder
def a1_masks(ctx, S):
    """The refinement pass's masks (parseq.py:267-297, Appendix A1) for S queries over one row's context ctx (L,)."""
    L = ctx.shape[0]
    causal = torch.triu(torch.ones(S, L, dtype=torch.bool, device=ctx.device), 1)
    causal[:2] = False
    return causal, (ctx == 0).int().cumsum(-1) > 0


def content_in(sd, spec, ctx):
    """float64 content stream before LN_c (what the engine forms in fp32) and its bound 4 e |terms|."""
    D = spec.embed_dim
    emb = sd["text_embed.embedding.weight"][ctx]
    pos = torch.cat([torch.zeros_like(emb[:1]), sd["pos_queries"][0, :ctx.shape[0] - 1]])
    c = math.sqrt(D) * emb + pos
    return c, 4 * E * (math.sqrt(D) * emb.abs() + pos.abs())


def step_chain(sd, spec, ctx, qpos, amask, pmask, q_all, e_q_all, memk, memv, e_memk, e_memv, pos_shift=0):
    """A whole decoder step / pass for one row from its context tokens, float64, with the chained bound: the content
    K/V, masked self-attention with the precomputed queries, cross-attention over the row's memory K/V, MLP, final norm
    and head.  Returns (logits, bound)."""
    D, heads = spec.embed_dim, spec.dec_heads
    c, e_c = content_in(sd, spec, ctx)
    cn, e_cn = ln(sd, DEC + "norm_c", c, e_c, 1e-5, True, rss=True)
    assert torch.allclose(cn, ops.content_embed(sd, spec, ctx[None])[0], rtol=0, atol=1e-9)
    (k, e_k), (v, e_v) = [lin(cn, e_cn, sd[SA + "in_proj_weight"][j * D:(j + 1) * D],
                              sd[SA + "in_proj_bias"][j * D:(j + 1) * D], True, rss=True) for j in (1, 2)]
    o, e_o = attend(q_all[qpos], k, v, heads, e_q_all[qpos], e_k, e_v, amask, pmask, rss=True)
    pos = sd["pos_queries"][0, qpos + pos_shift]       # pos_shift != 0 only for a wrong reference
    x, e_x = lin(o, e_o, sd[SA + "out_proj.weight"], sd[SA + "out_proj.bias"], False, resid=pos, rss=True)
    e_x = e_x + E * x.abs()
    h, e_h = ln(sd, DEC + "norm1", x, e_x, 1e-5, True, rss=True)
    qc, e_qc = lin(h, e_h, sd[CA + "in_proj_weight"][:D], sd[CA + "in_proj_bias"][:D], True, rss=True)
    oc, e_oc = attend(qc, memk, memv, heads, e_qc, e_memk, e_memv, rss=True)
    x2, e_x2 = lin(oc, e_oc, sd[CA + "out_proj.weight"], sd[CA + "out_proj.bias"], False, resid=x, e_r=e_x, rss=True)
    h2, e_h2 = ln(sd, DEC + "norm2", x2, e_x2, 1e-5, True, rss=True)
    f, e_f = lin(h2, e_h2, sd[DEC + "linear1.weight"], sd[DEC + "linear1.bias"], True, gelu=True, rss=True)
    x3, e_x3 = lin(f, e_f, sd[DEC + "linear2.weight"], sd[DEC + "linear2.bias"], False, resid=x2, e_r=e_x2, rss=True)
    out, e_out = ln(sd, "decoder.norm", x3, e_x3, 1e-5, True, rss=True)
    lg, e = lin(out, e_out, sd["head.weight"], sd["head.bias"], False, rss=True)
    return lg, LAMBDA * e


def teacher_forced_ar(sd, spec, tgt, n, q_all, e_q_all, mem_kv, pos_shift=0):
    """logits (n, C) of the n AR steps of one row, from its context tgt[:n] (causal mask), and their bound."""
    ctx = tgt[:n].long().to(DEV)
    causal = torch.triu(torch.ones(n, n, dtype=torch.bool, device=DEV), 1)
    lg, e = step_chain(sd, spec, ctx, torch.arange(n, device=DEV), causal, None, q_all, e_q_all, *mem_kv[1:],
                       pos_shift=pos_shift)
    if pos_shift == 0:
        ref = ops.head(sd, ops.decode(sd, spec, ctx[None], mem_kv[0][None], sd["pos_queries"][:, :n], causal))[0]
        assert (lg - ref).abs().max() < 1e-6 * (1 + ref.abs().max())   # chain == ops.decode (memory K/V exact)
    return lg, e


def check_ar(tag, m, sd, spec, rows, glen_rows, q_all, e_q_all, memkv_rows, ar_logits=None, rep_cut=None,
             mutate=False):
    """AR decode, teacher-forced on the engine's own ar.tgt.  ar_logits (B, steps, C): the seam's AR logits
    (refine_iters = 0); otherwise every decision in ar.raw is checked.  mutate (with ar_logits): wrong whole-step
    references (norm1 / norm2 swapped, pos_queries row i + 1 added at step i) must miss their composite bound."""
    tgt, raw = m.debug_tensor("ar.tgt"), m.debug_tensor("ar.raw")
    ties = n_dec = 0
    mut = {}
    for r in rows:
        n = int(glen_rows[r])
        lg, e = teacher_forced_ar(sd, spec, tgt[r], n, q_all, e_q_all, memkv_rows[r])
        LOGIT_BOUNDS[tag] = max(LOGIT_BOUNDS.get(tag, 0.0), float(e.max()))
        if ar_logits is not None:
            keep = torch.ones(n, dtype=torch.bool, device=DEV)
            if rep_cut is not None and 0 <= int(rep_cut[r]) < n:
                keep[int(rep_cut[r])] = False                  # the repetition patch (parseq.py:301-309)
            got = ar_logits[r, :n].to(DEV, torch.float64)[keep]
            _check(tag + " AR logits (teacher-forced)", got, lg[keep], e[keep])
            if mutate:
                bad = _swap_norms(sd, DEC + "norm1", DEC + "norm2")
                for k, (w, ew) in (("AR step norm1 / norm2 swapped",
                                    teacher_forced_ar(bad, spec, tgt[r], n, q_all, e_q_all, memkv_rows[r])),
                                   ("AR step pos_q row i+1",
                                    teacher_forced_ar(sd, spec, tgt[r], n, q_all, e_q_all, memkv_rows[r], pos_shift=1))):
                    mut.setdefault(k, []).append((got, w[keep], ew[keep]))
            continue
        a = lg.argmax(-1).cpu()
        got = raw[r, :n].long()
        for i in range(n):
            n_dec += 1
            if int(got[i]) == int(a[i]):
                continue
            # the engine may take the other token only if the two float64 logits are within their two bounds
            gap = float(lg[i, a[i]] - lg[i, got[i]])
            lim = float(e[i, a[i]] + e[i, got[i]])
            assert gap <= lim, "%s row %d step %d: engine token %d, float64 arg-max %d, gap %.4g > bounds %.4g" % (
                tag, r, i, int(got[i]), int(a[i]), gap, lim)
            ties += 1
    for k, v in mut.items():
        _miss(k, torch.cat([a for a, _, _ in v]), torch.cat([b for _, b, _ in v]), torch.cat([c for _, _, c in v]))
    if ar_logits is None:
        print("[stages] %s: %d AR decisions, %d near-ties within the two tokens' logit bounds" % (tag, n_dec, ties))


def check_ar_control(tag, m, spec, row_group, ngroups):
    """ar.tgt / ar.rep_cut / ar.group_len follow from the engine's raw arg-max tokens under the oracle's rules
    (forced EOS at a repetition onset, detect_repeat_onset, a group ends at the first step where all its rows hold
    an EOS)."""
    S, eos = spec.max_label_length + 1, spec.eos_id
    raw, tgt = m.debug_tensor("ar.raw").numpy(), m.debug_tensor("ar.tgt").numpy()
    glen, cut = m.debug_tensor("ar.group_len").numpy()[:, 0], m.debug_tensor("ar.rep_cut").numpy()[:, 0]
    B = raw.shape[0]
    for g in range(ngroups):
        rows = [r for r in range(B) if row_group[r] == g]
        sim = np.full((len(rows), S), spec.pad_id, dtype=np.int64)
        sim[:, 0] = spec.bos_id
        rc = [-1] * len(rows)
        n = S
        for i in range(S):
            j = i + 1
            if j < S:
                for k, r in enumerate(rows):
                    tok = int(raw[r, i])
                    sim[k, j] = tok
                    if spec.repetition_stop and rc[k] < 0 and tok != eos:
                        hit = ops.detect_repeat_onset(sim[k, 1:j + 1].tolist(), spec.rep_period_max,
                                                      spec.rep_min_run_p1, spec.rep_min_repeats)
                        if hit is not None:
                            rc[k] = hit[0] + hit[1]
                            sim[k, j] = eos
            if j >= S or (sim[:, 1:j + 1] == eos).any(-1).all():
                n = min(j, S)
                break
        assert int(glen[g]) == n, "%s group %d: group_len %d, rules give %d" % (tag, g, glen[g], n)
        for k, r in enumerate(rows):
            assert np.array_equal(tgt[r, :n], sim[k, :n]), "%s row %d: ar.tgt" % (tag, r)
            assert int(cut[r]) == rc[k], "%s row %d: rep_cut %d, rules give %d" % (tag, r, cut[r], rc[k])
    return glen, cut


def check_last_pass(tag, m, sd, spec, lay, row_group, glen_pass, mem_rows, prev_ids=None, logits=None, rep_cut=None,
                    mutate=False):
    """The last decoder pass, one sub-layer at a time, each from the engine's own input to it."""
    S, D, heads = spec.max_label_length + 1, spec.embed_dim, spec.dec_heads
    B = len(row_group)
    ctx_raw, klen, kpad = m.debug_tensor("dec.ctx"), m.debug_tensor("dec.klen")[:, 0], m.debug_tensor("dec.kpad")[:, 0]
    if prev_ids is not None:
        for r in range(B):
            n = int(glen_pass[row_group[r]]) - 1
            keep = [i for i in range(n) if rep_cut is None or int(rep_cut[r]) != i]
            assert torch.equal(ctx_raw[r, keep].long(), torch.as_tensor(prev_ids[r])[keep].long()), "%s row %d ctx" % (tag, r)
    eng = {k: _dbg(m, "dec." + k) for k in ("cin", "ckv", "sa", "qc", "oc", "mlp", "x", "out", "x_self", "x_cross")}
    cin = lay.res(eng["cin"], "dec.cin")
    ck, cv = lay.kv(eng["ckv"], "dec.ckv")
    sa = lay.heads(eng["sa"], "dec.sa")
    qc = lay.heads(eng["qc"], "dec.qc", lay.qs)
    oc = lay.heads(eng["oc"], "dec.oc")
    xs, xc, x = (lay.res(eng[k], "dec." + k) for k in ("x_self", "x_cross", "x"))
    out = lay.res(eng["out"], "dec.out")
    mlp = eng["mlp"]
    q_all = lay.heads(_dbg(m, "model.q_self"), "model.q_self", lay.qs)
    pos = sd["pos_queries"][0, :S]
    bad = dict(sd)
    bad[DEC + "norm1.weight"], bad[DEC + "norm1.bias"] = sd[DEC + "norm2.weight"], sd[DEC + "norm2.bias"]
    mut = {}
    for r in range(B):
        L = int(glen_pass[row_group[r]])
        ctx = torch.cat([torch.tensor([spec.bos_id]), ctx_raw[r, :L - 1].long()]).to(DEV)
        amask, pmask = a1_masks(ctx, S)
        first = int(pmask.int().argmax()) if bool(pmask.any()) else L
        assert int(klen[r]) == L and int(kpad[r]) == first, "%s row %d: klen %d kpad %d, expected %d %d" % (
            tag, r, klen[r], kpad[r], L, first)
        R = slice(r * S, (r + 1) * S)
        c, e_c = content_in(sd, spec, ctx)
        ref, e = ln(sd, DEC + "norm_c", c, e_c, 1e-5, True)
        _check(tag + " dec.cin (content + norm_c)", cin[R][:L], ref, e)
        kv_ref, e_kv = [], []
        for j in (1, 2):
            y, ey = lin(cin[R][:L], None, sd[SA + "in_proj_weight"][j * D:(j + 1) * D], sd[SA + "in_proj_bias"][j * D:(j + 1) * D], True)
            kv_ref.append(y)
            e_kv.append(ey)
        assert torch.allclose(torch.cat(ops.mha_kv(sd, SA, cin[R][:L]), -1), torch.cat(kv_ref, -1), rtol=0, atol=1e-9)
        _check(tag + " dec.ckv", torch.cat([ck[R][:L], cv[R][:L]], -1), torch.cat(kv_ref, -1), torch.cat(e_kv, -1))
        ref, e = attend(q_all, ck[R][:L], cv[R][:L], heads, amask=amask, pmask=pmask)
        _check(tag + " dec.sa (masked self-attention)", sa[R], ref, e)
        if mutate:
            causal = torch.triu(torch.ones(S, L, dtype=torch.bool, device=DEV), 1)
            w, _ = attend(q_all, ck[R][:L], cv[R][:L], heads, amask=causal, pmask=pmask)
            mut.setdefault("rows 0/1 not opened", []).append((sa[R], w, e))
            if first < L - 1:
                p2 = pmask.clone()
                p2[first] = False
                w, _ = attend(q_all, ck[R][:L], cv[R][:L], heads, amask=amask, pmask=p2)
                mut.setdefault("kpad one past the first EOS", []).append((sa[R], w, e))
        ref, e = lin(sa[R], None, sd[SA + "out_proj.weight"], sd[SA + "out_proj.bias"], False, resid=pos)
        e = e + E * ref.abs()
        _check(tag + " dec.x_self (self_out + pos_q)", xs[R], ref, e)
        if mutate:
            pos1 = torch.cat([pos[1:], pos[-1:]])
            w = ops.mha_out(sd, SA, sa[R]) + pos1
            mut.setdefault("pos_q row i+1", []).append((xs[R], w, e))
        h, e_h = ln(sd, DEC + "norm1", xs[R], None, 1e-5, True)
        ref, e = lin(h, e_h, sd[CA + "in_proj_weight"][:D], sd[CA + "in_proj_bias"][:D], True)
        _check(tag + " dec.qc (norm1 + cross q)", qc[R], ref, e)
        if mutate:
            w = ops.mha_q(bad, CA, ops.layer_norm(bad, DEC + "norm1", xs[R], 1e-5))
            mut.setdefault("norm1 / norm2 swapped", []).append((qc[R], w, e))
        mk, mv = mem_rows[r]
        ref, e = attend(qc[R], mk, mv, heads)
        _check(tag + " dec.oc (cross-attention)", oc[R], ref, e)
        if mutate and B > 1:
            nk, nv = mem_rows[(r + 1) % B]
            w, _ = attend(qc[R], nk, nv, heads)
            mut.setdefault("neighbouring crop's memory", []).append((oc[R], w, e))
        ref, e = lin(oc[R], None, sd[CA + "out_proj.weight"], sd[CA + "out_proj.bias"], False, resid=xs[R])
        _check(tag + " dec.x_cross (cross_out + residual)", xc[R], ref, e)
        h, e_h = ln(sd, DEC + "norm2", xc[R], None, 1e-5, True)
        ref, e = lin(h, e_h, sd[DEC + "linear1.weight"], sd[DEC + "linear1.bias"], True, gelu=True)
        assert torch.allclose(ref, ops.mlp_hidden(sd, h), rtol=0, atol=1e-12)
        _check(tag + " dec.mlp (norm2 + linear1 + GELU)", mlp[R], ref, e)
        ref, e = lin(mlp[R], None, sd[DEC + "linear2.weight"], sd[DEC + "linear2.bias"], False, resid=xc[R])
        _check(tag + " dec.x (linear2 + residual)", x[R], ref, e)
        ref, e = ln(sd, "decoder.norm", x[R], None, 1e-5, True)
        _check(tag + " dec.out (final norm)", out[R], ref, e)
        if logits is not None:
            ref, e = lin(out[R], None, sd["head.weight"], sd["head.bias"], False)
            got = logits[r].to(DEV, torch.float64)
            keep = torch.ones(S, dtype=torch.bool, device=DEV)
            if rep_cut is not None and 0 <= int(rep_cut[r]) < S:
                keep[int(rep_cut[r])] = False                  # the repetition patch (parseq.py:301-309)
            _check(tag + " logits (head)", got[keep], ref[keep], e[keep])
    for k, v in mut.items():
        _miss(k, torch.cat([a for a, _, _ in v]), torch.cat([b for _, b, _ in v]), torch.cat([c for _, _, c in v]))
    return mut


# ------------------------------------------------------------------------------------------------------ drivers
def _rec(name, sd, refine=1, decode_ar=1, recognizer=False):
    rec = TextRecognizer(model_name=name, from_pretrained=False, device="cuda", dynamic_width=True,
                         batch_bucketing=True)
    rec.model.decode_ar = decode_ar
    rec.model.refine_iters = refine
    rec.model.load_state_dict(sd)
    return rec if recognizer else rec.model


def _memkv_rows(mk, mv, crops):
    return [(mk[t0:t0 + n], mv[t0:t0 + n]) for (t0, n, _) in crops]


def _seam_case(name, refine=1, decode_ar=1, B=4, W=160, seed=3, mutate=False, repeat=False):
    spec = dataclasses.replace(ops.SPECS[name], refine_iters=refine, decode_ar=decode_ar)
    sd = weights.make_parseq_state_dict(spec, seed=seed, peaked=True, degenerate_repeat=repeat)
    m = _rec(name, sd, refine, decode_ar)
    lay = Layout(spec)
    tag = "%s r%d a%d%s" % (name, refine, decode_ar, " rep" if repeat else "")
    img = torch.rand(B, 3, 32, W, generator=torch.Generator().manual_seed(seed + 1)) * 2 - 1
    m.set_debug(True)
    N = (32 // spec.patch[0]) * (W // spec.patch[1])
    memory_out = torch.empty(B * N, spec.embed_dim)
    logits = m(img.cuda(), memory_out=memory_out).cpu()
    sd64 = _sd64(sd)
    img16 = img.half().to(DEV, torch.float64)
    crops = [(b * N, N, W // spec.patch[1]) for b in range(B)]
    q_all, e_q_all = check_constants(tag, m, sd64, spec, lay)
    mem, mk, mv = check_encoder(tag, m, sd64, spec, lay, crops, img16, memory_out, mutate=mutate)
    mem_rows = _memkv_rows(mk, mv, crops)
    row_group = [0] * B
    S = spec.max_label_length + 1
    if decode_ar:
        glen, cut = check_ar_control(tag, m, spec, row_group, 1)
        # teacher-forced steps use the float64 cross K/V of the engine's memory, with the memory K/V bound
        D = spec.embed_dim
        kvb = [lin(mem, None, sd64[CA + "in_proj_weight"][j * D:(j + 1) * D], sd64[CA + "in_proj_bias"][j * D:(j + 1) * D], True)
               for j in (1, 2)]
        mk64 = [(mem[t0:t0 + n], kvb[0][0][t0:t0 + n], kvb[1][0][t0:t0 + n], kvb[0][1][t0:t0 + n], kvb[1][1][t0:t0 + n])
                for (t0, n, _) in crops]
        check_ar(tag, m, sd64, spec, range(B), [glen[0]] * B, q_all, e_q_all, mk64,
                 ar_logits=logits if refine == 0 else None, rep_cut=cut, mutate=mutate)
    else:
        with pytest.raises(_lib.YtkError):
            m.debug_tensor("ar.raw")
        glen, cut = np.array([S]), np.full(B, -1)
    if refine == 0 and decode_ar:
        with pytest.raises(_lib.YtkError):
            m.debug_tensor("dec.sa")
        return m, tag
    # context length of the last pass: the AR steps for the first pass after the AR loop, 1 (<bos> alone) for the
    # non-autoregressive first pass, S for every later pass
    first_pass = refine == (1 if decode_ar else 0)
    glen_pass = [S] if not first_pass else ([int(glen[0])] if decode_ar else [1])
    prev_ids = None
    if decode_ar and refine == 1:
        prev_ids = m.debug_tensor("ar.raw")
    elif refine >= 2 or (not decode_ar and refine >= 1):
        # the context of the last pass is the arg-max of the pass before: the same forward with one pass fewer
        m.set_debug(False)
        m.refine_iters = refine - 1
        prev = m(img.cuda())
        m.refine_iters = refine
        prev_ids = prev.argmax(-1).cpu()
        m.set_debug(True)
        m(img.cuda())
    mut = check_last_pass(tag, m, sd64, spec, lay, row_group, glen_pass, mem_rows, prev_ids=prev_ids, logits=logits,
                          rep_cut=cut, mutate=mutate)
    if mutate and refine >= 2:
        assert "kpad one past the first EOS" in mut, "no row holds an EOS before the end of its context"
    return m, tag


def _report():
    for k in sorted(RATIOS):
        print("[stages] %-62s %.3g" % (k, RATIOS[k]))
    for k in sorted(LOGIT_BOUNDS):
        print("[stages] %s: largest AR logit bound %.3g logits" % (k, LOGIT_BOUNDS[k]))
    RATIOS.clear()
    LOGIT_BOUNDS.clear()


@pytest.mark.parametrize("name", ["parseq-tiny-dynw-v4", "parseq-tiny", "parseq-small", "parseq", "parseq-large-v4_1"])
def test_stages_catalogue(name):
    """Every catalogue model the engine accepts, refine_iters 1, with the wrong-reference checks on the first two."""
    _seam_case(name, B=4 if "large" not in name else 3, mutate=name in ("parseq-tiny-dynw-v4", "parseq-tiny"))
    _report()


@pytest.mark.parametrize("refine,decode_ar", [(0, 1), (2, 1), (1, 0), (0, 0)])
def test_stages_decoder_switches(refine, decode_ar):
    """refine_iters 0 (the AR logits themselves, with the wrong whole-step references), 2 (the last pass reads the
    previous pass's arg-max over all S positions, so rows hold an EOS well before the end of their context: the kpad
    mutation applies), decode_ar = 0 with a refinement pass after the non-autoregressive one, and decode_ar = 0 alone
    (the non-autoregressive pass, context <bos> only, is the last pass)."""
    _seam_case("parseq-tiny-dynw-v4", refine=refine, decode_ar=decode_ar, B=5, W=200, seed=4,
               mutate=decode_ar == 1 and refine in (0, 2))
    _report()


def test_stages_repetition_stop():
    m, tag = _seam_case("parseq-tiny-dynw-v4", B=3, W=120, seed=3, repeat=True)
    cut = m.debug_tensor("ar.rep_cut")[:, 0]
    assert (cut >= 0).all(), cut                       # the degenerate weights trip the detector on every row
    _report()


def _input_dependent_stops(spec, seed, ramp):
    """make_parseq_state_dict(peaked=True) with its positional EOS ramp scaled by `ramp`: the same random draws
    (peaked only rescales the head and adds the ramp to pos_queries), so the difference of the two is the ramp."""
    sd = weights.make_parseq_state_dict(spec, seed=seed, peaked=True)
    plain = weights.make_parseq_state_dict(spec, seed=seed)["pos_queries"]
    sd["pos_queries"] = plain + ramp * (sd["pos_queries"] - plain)
    return sd


def _ragged(rec, spec, seed, n_groups, per):
    """n_groups groups of `per` text-line crops of a synthetic page, each group padded to its own widest crop."""
    from yomitoku_b200.data import ParseqDataset
    from yomitoku_b200.synth import synthetic_page
    page, quads = synthetic_page(seed)
    n = n_groups * per
    canv = list(ParseqDataset(rec._cfg, page, quads[:n], num_workers=1, dynamic_width=True).data)
    pw = spec.patch[1]
    groups = [i // per for i in range(n)]
    wmax = [max(canv[j].shape[1] for j in range(n) if groups[j] == g) for g in range(n_groups)]
    padded = [-(-wmax[g] // pw) * pw for g in groups]
    return canv, padded, groups


@pytest.mark.parametrize("split", [False, True])
def test_stages_ragged_u8(split, monkeypatch):
    """One packed ragged u8 call of text-line crops: three groups of different padded widths that stop at different AR
    steps (and, with YTK_AR_SPLIT_MIN=1, the two-part AR loop, whose parts - group 0 and groups 1..2 - stop at
    different steps too).  The EOS ramp of the peaked weights is weakened to a quarter so that where a row stops
    depends on its image, not on the ramp alone (the fp32 oracle stops these groups after 16, 14 and 15 steps)."""
    name = "parseq-tiny-dynw-v4"
    spec = ops.SPECS[name]
    sd = _input_dependent_stops(spec, seed=7, ramp=0.25)
    rec = _rec(name, sd, recognizer=True)
    m = rec.model
    lay = Layout(spec)
    tag = "%s ragged%s" % (name, " split" if split else "")
    if split:
        monkeypatch.setenv("YTK_AR_SPLIT_MIN", "1")
    else:
        monkeypatch.delenv("YTK_AR_SPLIT_MIN", raising=False)
    canv, padded, groups = _ragged(rec, spec, 5, 3, 4)
    m.set_debug(True)
    ids, probs, glen = m.recognize_crops(canv, padded, groups, 3)
    assert len(set(padded)) > 1, padded                # groups of different padded widths
    assert len(set(glen.tolist())) > 1, glen           # ... that stop at different steps
    assert glen[0] != glen[1:].max(), glen             # the two parts of the split loop stop at different steps
    print("[stages] %s: group_len %s, padded widths %s" % (tag, glen.tolist(), sorted(set(padded))))
    sd64 = _sd64(sd)
    gh, pw = 32 // spec.patch[0], spec.patch[1]
    crops, t = [], 0
    for wp in padded:
        crops.append((t, gh * (wp // pw), wp // pw))
        t += gh * (wp // pw)
    q_all, e_q_all = check_constants(tag, m, sd64, spec, lay)
    mem, mk, mv = check_encoder(tag, m, sd64, spec, lay, crops)
    glen2, cut = check_ar_control(tag, m, spec, groups, 3)
    assert np.array_equal(glen2, glen)
    D = spec.embed_dim
    kvb = [lin(mem, None, sd64[CA + "in_proj_weight"][j * D:(j + 1) * D], sd64[CA + "in_proj_bias"][j * D:(j + 1) * D], True)
           for j in (1, 2)]
    mk64 = [(mem[t0:t0 + n], kvb[0][0][t0:t0 + n], kvb[1][0][t0:t0 + n], kvb[0][1][t0:t0 + n], kvb[1][1][t0:t0 + n])
            for (t0, n, _) in crops]
    check_ar(tag, m, sd64, spec, range(len(canv)), [glen[g] for g in groups], q_all, e_q_all, mk64)
    check_last_pass(tag, m, sd64, spec, lay, groups, glen, _memkv_rows(mk, mv, crops),
                    prev_ids=m.debug_tensor("ar.raw"), mutate=not split)
    _report()


def test_capture_changes_nothing():
    """Capture on and off: ids, probs, group_len and logits bit-equal, the same number of kernel launches; names the
    last forward did not produce are refused."""
    name = "parseq-tiny-dynw-v4"
    spec = ops.SPECS[name]
    sd = weights.make_parseq_state_dict(spec, seed=7, peaked=True)
    rec = _rec(name, sd, recognizer=True)
    m = rec.model
    canv, padded, groups = _ragged(rec, spec, 6, 2, 3)
    img = torch.rand(3, 3, 32, 160, generator=torch.Generator().manual_seed(2)) * 2 - 1
    L = _lib.lib()
    res = {}
    for on in (False, True, False):
        m.set_debug(on)
        c0 = L.ytk_launch_count()
        a = m.recognize_crops(canv, padded, groups, 2)
        lg = m(img.cuda()).cpu()
        res.setdefault(on, []).append((a, lg, L.ytk_launch_count() - c0))
        if not on:
            for nm in ("enc.x.0", "dec.x_self", "dec.x_cross", "dec.ctx"):
                with pytest.raises(_lib.YtkError):
                    m.debug_tensor(nm)
    (a0, l0, n0), (a1, l1, n1), (a2, l2, n2) = res[False][0], res[True][0], res[False][1]
    for x, y in ((a0, a1), (a0, a2)):
        for u, v in zip(x, y):
            assert np.array_equal(u.view(np.uint8), v.view(np.uint8))
    assert torch.equal(l0.view(torch.int32), l1.view(torch.int32)) and torch.equal(l0.view(torch.int32), l2.view(torch.int32))
    assert n0 == n1 == n2, (n0, n1, n2)
    for nm in ("enc.x.%d" % (spec.enc_depth + 1), "enc.x.-1", "dec.nothing", "model.none", "ar.x"):
        with pytest.raises(_lib.YtkError):
            m.debug_tensor(nm)
    # refine_iters 0: no full decoder pass ran, so no dec.* name has data from it
    m.refine_iters = 0
    m(img.cuda())
    with pytest.raises(_lib.YtkError):
        m.debug_tensor("dec.x")
    assert m.debug_tensor("ar.raw").shape == (3, spec.max_label_length + 1)
