"""Oracle: PARSeq forward, functional fp32 restatement (TEST INFRASTRUCTURE, see oracle/__init__.py).

Follows reference src/yomitoku/models/parseq.py:49-311 and models/layers/parseq_transformer.py:27-244.
The encoder is timm 1.0.27 `VisionTransformer(class_token=False, global_pool="", num_classes=0)` (pinned in the
reference's uv.lock; not installable here) restated from its published forward: patch conv -> + learned absolute
pos_embed cropped to the patch grid (parseq_transformer.py:212-234) -> depth x pre-LN block (LayerNorm eps 1e-6, fused
qkv Linear with bias, softmax(q k^T / sqrt(hd)) v with no mask, proj; exact-erf GELU MLP) -> final LayerNorm.
The decoder layer uses torch.nn.MultiheadAttention semantics (packed in_proj q,k,v; boolean masks, True = masked).

This module deliberately keeps the reference's *batch* semantics (no KV cache, early break when every row has an
EOS, per-batch padded width), because outputs depend on them (SURVEY.md Appendix A9, A11, A12).
"""
import math
from dataclasses import dataclass

import torch
import torch.nn.functional as F


@dataclass(frozen=True)
class ParseqSpec:
    """Architecture numbers of one catalog entry (reference configs/cfg_text_recognizer_parseq*.py)."""
    embed_dim: int
    enc_heads: int
    enc_depth: int
    patch: tuple          # (ph, pw)
    img_size: tuple       # (H, W) training canvas
    num_tokens: int
    max_label_length: int = 100
    dec_heads: int = 8
    mlp_ratio: int = 4
    dec_mlp_ratio: int = 4
    decode_ar: int = 1
    refine_iters: int = 1
    # repetition early-stop defaults (parseq.py:93-96)
    repetition_stop: bool = True
    rep_period_max: int = 8
    rep_min_run_p1: int = 8
    rep_min_repeats: int = 3

    @property
    def grid(self):
        return (self.img_size[0] // self.patch[0], self.img_size[1] // self.patch[1])

    @property
    def num_classes(self):
        return self.num_tokens - 2  # head does not predict BOS / PAD (parseq.py:71-72)

    @property
    def eos_id(self):
        return 0

    @property
    def bos_id(self):
        return self.num_tokens - 2

    @property
    def pad_id(self):
        return self.num_tokens - 1


SPECS = {
    # cfg_text_recognizer_parseq.py / _v2.py
    "parseq": ParseqSpec(512, 8, 12, (8, 8), (32, 800), 7312),
    "parseqv2": ParseqSpec(512, 8, 12, (8, 8), (32, 800), 7312),
    # cfg_text_recognizer_parseq_small.py
    "parseq-small": ParseqSpec(384, 8, 9, (16, 16), (32, 800), 7312),
    # cfg_text_recognizer_parseq_tiny.py
    "parseq-tiny": ParseqSpec(368, 8, 12, (8, 16), (32, 400), 7121, max_label_length=50),
    # cfg_text_recognizer_parseq_large_v4_1.py:7-53
    "parseq-large-v4_1": ParseqSpec(768, 8, 12, (8, 8), (32, 800), 7121),
    # cfg_text_recognizer_parseq_tiny_dynw_v4.py:7-74
    "parseq-tiny-dynw-v4": ParseqSpec(192, 6, 12, (4, 8), (32, 800), 7121, dec_heads=6),
}


# ----------------------------------------------------------------------------------------------- encoder
# The forward is written as a chain of stage functions so that a test can run any one stage on inputs of its choice
# (in float64, on the inputs a device engine gave that stage) with the same code that produces the fp32 results.
def layer_norm(sd, name, x, eps):
    """LayerNorm over the last dim with the parameters `name`.weight / `name`.bias."""
    return F.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], eps)


def patch_embed(sd, spec, images, prefix="encoder."):
    """patch conv -> (B, gh*gw, D) row-major grid + the learned absolute pos_embed cropped to the patch grid
    (parseq_transformer.py:212-234): grid cell (y, x) takes pos_embed row y * full_gw + x."""
    D = spec.embed_dim
    x = F.conv2d(images, sd[prefix + "patch_embed.proj.weight"], sd[prefix + "patch_embed.proj.bias"],
                 stride=spec.patch)
    B, _, gh, gw = x.shape
    x = x.flatten(2).transpose(1, 2)                                   # (B, gh*gw, D), row-major grid
    full_gh, full_gw = spec.grid
    pos = sd[prefix + "pos_embed"].reshape(1, full_gh, full_gw, D)[:, :gh, :gw].reshape(1, gh * gw, D)
    return x + pos


def encoder_block(sd, spec, i, x, prefix="encoder."):
    """timm pre-LN ViT block i: x + proj(attn(LN1 x)), then x + fc2(gelu(fc1(LN2 x))); LayerNorm eps 1e-6."""
    D, heads = spec.embed_dim, spec.enc_heads
    hd = D // heads
    B = x.shape[0]
    p = "%sblocks.%d." % (prefix, i)
    h = layer_norm(sd, p + "norm1", x, 1e-6)
    qkv = F.linear(h, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"])
    qkv = qkv.reshape(B, -1, 3, heads, hd).permute(2, 0, 3, 1, 4)   # (3,B,h,N,hd)
    att = torch.softmax((qkv[0] @ qkv[1].transpose(-1, -2)) * (hd ** -0.5), dim=-1) @ qkv[2]
    att = att.transpose(1, 2).reshape(B, -1, D)
    x = x + F.linear(att, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
    h = layer_norm(sd, p + "norm2", x, 1e-6)
    h = F.gelu(F.linear(h, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]))
    return x + F.linear(h, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])


def encoder_norm(sd, spec, x, prefix="encoder."):
    """final LayerNorm of the encoder (eps 1e-6): the decoder's memory."""
    return layer_norm(sd, prefix + "norm", x, 1e-6)


def encoder_forward(sd, spec, images, prefix="encoder."):
    """reference Encoder.forward / forward_features_dynamic (parseq_transformer.py:206-234). images (B,3,32,W)."""
    x = patch_embed(sd, spec, images, prefix)
    for i in range(spec.enc_depth):
        x = encoder_block(sd, spec, i, x, prefix)
    return encoder_norm(sd, spec, x, prefix)


# ----------------------------------------------------------------------------------------------- decoder
# torch.nn.MultiheadAttention(batch_first=True) forward (used at parseq_transformer.py:83-92) in its three parts:
# packed in_proj q / (k, v), scaled-dot-product attention with boolean masks (True = masked), out_proj.
def mha_q(sd, p, q_in):
    D = q_in.shape[-1]
    return F.linear(q_in, sd[p + "in_proj_weight"][:D], sd[p + "in_proj_bias"][:D])


def mha_kv(sd, p, kv_in):
    D = kv_in.shape[-1]
    w, b = sd[p + "in_proj_weight"], sd[p + "in_proj_bias"]
    return F.linear(kv_in, w[D:2 * D], b[D:2 * D]), F.linear(kv_in, w[2 * D:], b[2 * D:])


def mha_attend(q, k, v, heads, attn_mask=None, key_padding_mask=None):
    """q (B,Lq,D), k / v (B,Lk,D) -> (B,Lq,D).  attn_mask (Lq,Lk) bool, key_padding_mask (B,Lk) bool."""
    D = q.shape[-1]
    hd = D // heads
    B, Lq, Lk = q.shape[0], q.shape[1], k.shape[1]
    q = q.reshape(B, Lq, heads, hd).transpose(1, 2)
    k = k.reshape(B, Lk, heads, hd).transpose(1, 2)
    v = v.reshape(B, Lk, heads, hd).transpose(1, 2)
    s = (q @ k.transpose(-1, -2)) / math.sqrt(hd)                      # (B,h,Lq,Lk)
    if attn_mask is not None:
        s = s.masked_fill(attn_mask[None, None], float("-inf"))
    if key_padding_mask is not None:
        s = s.masked_fill(key_padding_mask[:, None, None, :], float("-inf"))
    o = torch.softmax(s, dim=-1) @ v
    return o.transpose(1, 2).reshape(B, Lq, D)


def mha_out(sd, p, o):
    return F.linear(o, sd[p + "out_proj.weight"], sd[p + "out_proj.bias"])


def _mha(sd, p, heads, q_in, kv_in, attn_mask=None, key_padding_mask=None):
    k, v = mha_kv(sd, p, kv_in)
    return mha_out(sd, p, mha_attend(mha_q(sd, p, q_in), k, v, heads, attn_mask, key_padding_mask))


DEC = "decoder.layers.0."


def content_embed(sd, spec, tgt):
    """LN_c of the content stream of context tokens tgt (B, L) (parseq.py:133-157): position 0 = sqrt(D) E[tgt0]
    (no positional term), position p >= 1 = pos_queries[p-1] + sqrt(D) E[tgt_p]."""
    D = spec.embed_dim
    L = tgt.shape[1]
    emb = sd["text_embed.embedding.weight"]
    scale = math.sqrt(D)
    null_ctx = scale * emb[tgt[:, :1]]
    content = torch.cat([null_ctx, sd["pos_queries"][:, :L - 1] + scale * emb[tgt[:, 1:]]], dim=1)
    return layer_norm(sd, DEC + "norm_c", content, 1e-5)


def self_attn_sublayer(sd, spec, tgt_query, content_n, attn_mask=None, key_padding_mask=None):
    """query stream + self-attention of LN_q(query) over the normalised content (parseq_transformer.py:83-87)."""
    qn = layer_norm(sd, DEC + "norm_q", tgt_query, 1e-5)
    return tgt_query + _mha(sd, DEC + "self_attn.", spec.dec_heads, qn, content_n, attn_mask, key_padding_mask)


def cross_attn_sublayer(sd, spec, x, memory):
    """x + cross-attention of LN1 x over the encoder memory (parseq_transformer.py:88-92)."""
    h = layer_norm(sd, DEC + "norm1", x, 1e-5)
    return x + _mha(sd, DEC + "cross_attn.", spec.dec_heads, h, memory)


def mlp_hidden(sd, h):
    return F.gelu(F.linear(h, sd[DEC + "linear1.weight"], sd[DEC + "linear1.bias"]))


def mlp_out(sd, hid):
    return F.linear(hid, sd[DEC + "linear2.weight"], sd[DEC + "linear2.bias"])


def mlp_sublayer(sd, spec, x):
    """x + linear2(gelu(linear1(LN2 x))) (parseq_transformer.py:93-94)."""
    return x + mlp_out(sd, mlp_hidden(sd, layer_norm(sd, DEC + "norm2", x, 1e-5)))


def final_norm(sd, spec, x):
    """Decoder.norm (eps 1e-5) of the query stream."""
    return layer_norm(sd, "decoder.norm", x, 1e-5)


def head(sd, out):
    """classification head over the normalised decoder output: logits (..., num_tokens - 2)."""
    return F.linear(out, sd["head.weight"], sd["head.bias"])


def decode(sd, spec, tgt, memory, tgt_query, tgt_query_mask, tgt_padding_mask=None):
    """reference PARSeq.decode (parseq.py:133-157) + Decoder.forward with depth 1 and update_content=False on the
    last (= only) layer (parseq_transformer.py:148-169,101-130): only the query stream is computed."""
    cn = content_embed(sd, spec, tgt)
    x = self_attn_sublayer(sd, spec, tgt_query, cn, tgt_query_mask, tgt_padding_mask)
    x = cross_attn_sublayer(sd, spec, x, memory)
    x = mlp_sublayer(sd, spec, x)
    return final_norm(sd, spec, x)


def detect_repeat_onset(seq, period_max=8, min_run_p1=8, min_repeats=3):
    """reference PARSeq._detect_repeat_onset (parseq.py:108-128): trailing period-p unit repeated >= min_run_p1
    (p == 1) or >= min_repeats (p > 1) times; smallest p wins.  Returns (onset, period) or None."""
    n = len(seq)
    for p in range(1, period_max + 1):
        if n < 2 * p:
            continue
        unit = seq[n - p:]
        reps, start = 1, n - p
        while start - p >= 0 and seq[start - p:start] == unit:
            reps += 1
            start -= p
        if reps >= (min_run_p1 if p == 1 else min_repeats):
            return start, p
    return None


@torch.inference_mode()
def parseq_forward(sd, spec, images, return_aux=False):
    """reference PARSeq.forward (parseq.py:159-311) for the inference configuration (max_length=None,
    export_onnx=False).  Returns logits (B, S, C): S = 101 when refine_iters > 0 or decode_ar == 0, else the number
    of AR steps run."""
    bs = images.shape[0]
    S = spec.max_label_length + 1
    memory = encoder_forward(sd, spec, images)
    pos_q = sd["pos_queries"][:, :S].expand(bs, -1, -1)
    causal = torch.triu(torch.ones(S, S, dtype=torch.bool), 1)
    tgt_in = torch.full((bs, S), spec.pad_id, dtype=torch.long)
    tgt_in[:, 0] = spec.bos_id
    rep_cut = [None] * bs
    rep_done = [False] * bs
    steps = []
    if not spec.decode_ar:
        # parseq.py:252-262: no prior context, the input is just <bos>; all positions are queried at once, no masks
        out = decode(sd, spec, tgt_in[:, :1], memory, pos_q, None)
        steps.append(head(sd, out))
    for i in range(S if spec.decode_ar else 0):
        j = i + 1
        out = decode(sd, spec, tgt_in[:, :j], memory, pos_q[:, i:j], causal[i:j, :j])
        p_i = head(sd, out)
        steps.append(p_i)
        if j < S:
            tgt_in[:, j] = p_i[:, 0].argmax(-1)
            if spec.repetition_stop:
                for b in range(bs):
                    tok = int(tgt_in[b, j])
                    if rep_done[b] or tok == spec.eos_id:
                        continue
                    hit = detect_repeat_onset(tgt_in[b, 1:j + 1].tolist(), spec.rep_period_max, spec.rep_min_run_p1,
                                              spec.rep_min_repeats)
                    if hit is not None:
                        rep_cut[b] = hit[0] + hit[1]
                        rep_done[b] = True
                        tgt_in[b, j] = spec.eos_id          # forced EOS context (parseq.py:242)
            if bool((tgt_in == spec.eos_id).any(dim=-1).all()):
                break
    logits = torch.cat(steps, dim=1)
    ar_steps = logits.shape[1]
    ar_tokens = tgt_in.clone()
    ar_top2 = logits.topk(2, -1).values
    ar_margin = (ar_top2[..., 0] - ar_top2[..., 1])                # (B, steps): decision margin of every AR step
    if spec.refine_iters:
        # Appendix A1: the int64 index tensor zeroes ROWS 0 and 1 of the causal mask (parseq.py:267-277)
        qmask = causal.clone()
        qmask[:2] = False
        bos = torch.full((bs, 1), spec.bos_id, dtype=torch.long)
        for _ in range(spec.refine_iters):
            t_in = torch.cat([bos, logits[:, :-1].argmax(-1)], dim=1)
            pad_mask = (t_in == spec.eos_id).int().cumsum(-1) > 0
            out = decode(sd, spec, t_in, memory, pos_q, qmask[:, :t_in.shape[1]], pad_mask)
            logits = head(sd, out)
    for b, cut in enumerate(rep_cut):
        if cut is not None and cut < logits.shape[1]:
            logits[b, cut, :] = -30.0
            logits[b, cut, spec.eos_id] = 30.0
    if return_aux:
        return logits, {"memory": memory, "ar_steps": ar_steps, "ar_tokens": ar_tokens, "rep_cut": rep_cut,
                        "ar_margin": ar_margin}
    return logits


# ----------------------------------------------------------------------------------------------- tokenizer
class Tokenizer:
    """reference ParseqTokenizer (postprocessor/parseq_tokenizer.py:91-126): [E]=0, charset 1..n, [B], [P]."""

    def __init__(self, charset):
        self.itos = ("[E]",) + tuple(charset) + ("[B]", "[P]")
        self.eos_id, self.bos_id, self.pad_id = 0, len(charset) + 1, len(charset) + 2

    def __len__(self):
        return len(self.itos)

    def decode(self, probs):
        """reference BaseTokenizer.decode + _filter (:64-88, :117-126). probs (B,S,C) softmax output.
        Returns (strings, scores): greedy ids cut at the first EOS; score = product of max-probs up to and
        including the EOS (all positions when there is none), computed in fp32 like numpy's float32 prod."""
        out_s, out_p = [], []
        for dist in probs:
            p, ids = dist.max(-1)
            ids = ids.tolist()
            n = ids.index(self.eos_id) if self.eos_id in ids else len(ids)
            out_s.append("".join(self.itos[t] for t in ids[:n]))
            out_p.append(float(p[:n + 1].cpu().numpy().prod()))
        return out_s, out_p
