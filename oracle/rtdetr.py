"""Oracle: RT-DETRv2 (layout parser / table structure recognizer) forward in fp32 torch (TEST INFRASTRUCTURE, see
__init__.py).  Inference only, functional, driven by a state_dict with the reference's key set.

Restates
  backbone   PResNet-50 variant d, frozen BN         models/layers/rtdetr_backbone.py:32-56, 98-146, 148-176, 245-334
  encoder    HybridEncoder: input_proj, AIFI layer on the stride-32 map (post-norm, q = k = x + 2-D sin-cos embedding),
             top-down FPN + bottom-up PAN of CSPRepLayer / RepVggBlock (not re-parameterised: both branches)
                                                       models/layers/rtdetr_hybrid_encoder.py:25-50, 71-122, 125-144,
                                                       181-213, 334-410
  decoder    RTDETRTransformerv2 (eval): input_proj, anchors / valid mask, enc_output + score / box heads, top-300
             query selection, 6 decoder layers (self-attention with query_pos, multi-scale deformable cross-attention
             with 4-d reference boxes, FFN, post-norms), iterative box refinement, outputs of the last layer
                                                       models/layers/rtdetrv2_decoder.py:36-40, 43-56, 155-222, 282-303,
                                                       306-388, 402-444, 648-678, 680-746, 782-815
  post       RTDETRPostProcessor (focal branch)        postprocessor/rtdetr_postprocessor.py:60-123
Pinned against the reference's own files executed by path with the same weights (oracle/refcheck.py: rtdetr cases,
tests/test_oracle_golden.py).
"""
import math
from dataclasses import dataclass, field
from typing import List

import torch
import torch.nn.functional as F


@dataclass
class RTDETRSpec:
    num_classes: int = 6
    hidden: int = 256
    heads: int = 8
    ffn: int = 1024
    num_queries: int = 300
    num_layers: int = 6
    num_levels: int = 3
    num_points: List[int] = field(default_factory=lambda: [4, 4, 4])
    strides: List[int] = field(default_factory=lambda: [8, 16, 32])
    img_size: List[int] = field(default_factory=lambda: [640, 640])
    blocks: List[int] = field(default_factory=lambda: [3, 4, 6, 3])          # PResNet-50
    csp_blocks: int = 3
    offset_scale: float = 0.5
    anchor_eps: float = 1e-2
    grid_size: float = 0.05
    pe_temperature: float = 10000.0


SPECS = {"layout": RTDETRSpec(num_classes=6), "table": RTDETRSpec(num_classes=3)}


# ------------------------------------------------------------------------------------------------ building blocks
def _bn(sd, p, x, eps=1e-5):
    scale = sd[p + ".weight"] * (sd[p + ".running_var"] + eps).rsqrt()
    return x * scale.view(1, -1, 1, 1) + (sd[p + ".bias"] - sd[p + ".running_mean"] * scale).view(1, -1, 1, 1)


def _act(x, act):
    if act is None:
        return x
    return {"relu": F.relu, "silu": F.silu, "gelu": F.gelu}[act](x)


def conv_norm(sd, p, x, stride=1, act=None):
    w = sd[p + ".conv.weight"]
    return _act(_bn(sd, p + ".norm", F.conv2d(x, w, None, stride, (w.shape[-1] - 1) // 2)), act)


def bottleneck(sd, p, x, stride, shortcut):
    out = conv_norm(sd, p + ".branch2a", x, 1, "relu")
    out = conv_norm(sd, p + ".branch2b", out, stride, "relu")          # variant d: the 3x3 conv carries the stride
    out = conv_norm(sd, p + ".branch2c", out, 1, None)
    if shortcut:
        short = x
    elif stride == 2:
        short = conv_norm(sd, p + ".short.conv", F.avg_pool2d(x, 2, 2, 0, ceil_mode=True), 1, None)
    else:
        short = conv_norm(sd, p + ".short", x, 1, None)
    return F.relu(out + short)


def backbone(sd, spec, x):
    p = "backbone."
    x = conv_norm(sd, p + "conv1.conv1_1", x, 2, "relu")
    x = conv_norm(sd, p + "conv1.conv1_2", x, 1, "relu")
    x = conv_norm(sd, p + "conv1.conv1_3", x, 1, "relu")
    x = F.max_pool2d(x, 3, 2, 1)
    outs = []
    for s, n in enumerate(spec.blocks):
        for b in range(n):
            x = bottleneck(sd, "%sres_layers.%d.blocks.%d" % (p, s, b), x, 2 if (b == 0 and s != 0) else 1, b != 0)
        if s >= 1:
            outs.append(x)
    return outs


def sincos_2d(w, h, dim, temperature, device=None, dtype=torch.float32):
    kw = dict(dtype=dtype, device=device)
    gw, gh = torch.meshgrid(torch.arange(int(w), **kw), torch.arange(int(h), **kw), indexing="ij")
    omega = 1.0 / (temperature ** (torch.arange(dim // 4, **kw) / (dim // 4)))
    ow, oh = gw.flatten()[:, None] @ omega[None], gh.flatten()[:, None] @ omega[None]
    return torch.cat([ow.sin(), ow.cos(), oh.sin(), oh.cos()], dim=1)[None]


def mha(sd, p, q_in, k_in, v_in, heads):
    """nn.MultiheadAttention(batch_first) forward without masks: packed in_proj, softmax(QK^T / sqrt d) V, out_proj."""
    W, b = sd[p + ".in_proj_weight"], sd[p + ".in_proj_bias"]
    D = W.shape[1]
    q = F.linear(q_in, W[:D], b[:D])
    k = F.linear(k_in, W[D:2 * D], b[D:2 * D])
    v = F.linear(v_in, W[2 * D:], b[2 * D:])
    B, Lq, _ = q.shape
    hd = D // heads
    q = q.view(B, Lq, heads, hd).transpose(1, 2)
    k = k.view(B, -1, heads, hd).transpose(1, 2)
    v = v.view(B, -1, heads, hd).transpose(1, 2)
    a = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(hd), dim=-1)
    o = (a @ v).transpose(1, 2).reshape(B, Lq, D)
    return F.linear(o, sd[p + ".out_proj.weight"], sd[p + ".out_proj.bias"])


def _ln(sd, p, x):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], 1e-5)


def aifi_attn(sd, p, src, pos, heads):
    """the AIFI self-attention sub-layer before its norm: src + MHA(q = k = src + pos, v = src)"""
    q = src + pos
    return src + mha(sd, p + ".self_attn", q, q, src, heads)


def ffn(sd, p, x, act):
    """linear2(act(linear1(x))) of a transformer layer"""
    return F.linear(_act(F.linear(x, sd[p + ".linear1.weight"], sd[p + ".linear1.bias"]), act), sd[p + ".linear2.weight"],
                    sd[p + ".linear2.bias"])


def aifi_layer(sd, p, src, pos, heads):
    src = _ln(sd, p + ".norm1", aifi_attn(sd, p, src, pos, heads))
    return _ln(sd, p + ".norm2", src + ffn(sd, p, src, "gelu"))


def repvgg(sd, b, x):
    """RepVggBlock in its two-branch (training) form: silu(conv3x3 + BN  +  conv1x1 + BN)"""
    return F.silu(conv_norm(sd, b + ".conv1", x, 1, None) + conv_norm(sd, b + ".conv2", x, 1, None))


def csp_rep(sd, p, x, n):
    x1 = conv_norm(sd, p + ".conv1", x, 1, "silu")
    for i in range(n):
        x1 = repvgg(sd, "%s.bottlenecks.%d" % (p, i), x1)
    return x1 + conv_norm(sd, p + ".conv2", x, 1, "silu")         # expansion 1.0: conv3 is the identity


def hybrid_encoder(sd, spec, feats):
    p = "encoder."
    proj = [_bn(sd, "%sinput_proj.%d.norm" % (p, i), F.conv2d(f, sd["%sinput_proj.%d.conv.weight" % (p, i)]))
            for i, f in enumerate(feats)]
    B, C, h, w = proj[2].shape
    src = proj[2].flatten(2).permute(0, 2, 1)
    mem = aifi_layer(sd, p + "encoder.0.layers.0", src, sincos_2d(w, h, C, spec.pe_temperature, src.device, src.dtype),
                     spec.heads)
    proj[2] = mem.permute(0, 2, 1).reshape(B, C, h, w)
    inner = [proj[2]]
    for idx in (2, 1):
        high = conv_norm(sd, "%slateral_convs.%d" % (p, 2 - idx), inner[0], 1, "silu")
        inner[0] = high
        up = F.interpolate(high, scale_factor=2.0, mode="nearest")
        inner.insert(0, csp_rep(sd, "%sfpn_blocks.%d" % (p, 2 - idx), torch.cat([up, proj[idx - 1]], 1), spec.csp_blocks))
    outs = [inner[0]]
    for idx in range(2):
        down = conv_norm(sd, "%sdownsample_convs.%d" % (p, idx), outs[-1], 2, "silu")
        outs.append(csp_rep(sd, "%span_blocks.%d" % (p, idx), torch.cat([down, inner[idx + 1]], 1), spec.csp_blocks))
    return outs


def generate_anchors(spec):
    """(anchors (1, L, 4) in logit space with inf at invalid positions, valid_mask (1, L, 1))."""
    out = []
    for lvl, s in enumerate(spec.strides):
        h, w = int(spec.img_size[0] / s), int(spec.img_size[1] / s)
        gy, gx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
        xy = (torch.stack([gx, gy], -1).unsqueeze(0) + 0.5) / torch.tensor([w, h], dtype=torch.float32)
        wh = torch.ones_like(xy) * spec.grid_size * (2.0 ** lvl)
        out.append(torch.cat([xy, wh], -1).reshape(-1, h * w, 4))
    a = torch.cat(out, 1)
    valid = ((a > spec.anchor_eps) * (a < 1 - spec.anchor_eps)).all(-1, keepdim=True)
    return torch.where(valid, torch.log(a / (1 - a)), torch.inf), valid


def mlp(sd, p, x, n):
    for i in range(n):
        x = F.linear(x, sd["%s.layers.%d.weight" % (p, i)], sd["%s.layers.%d.bias" % (p, i)])
        if i < n - 1:
            x = F.relu(x)
    return x


def inverse_sigmoid(x, eps=1e-5):
    x = x.clip(0.0, 1.0)
    return torch.log(x.clip(min=eps) / (1 - x).clip(min=eps))


def deformable_attention(spec, value, shapes, loc, weights):
    """value (B, L, heads, c); loc (B, Q, heads, P, 2) in [0, 1]; weights (B, Q, heads, P) -> (B, Q, heads * c)."""
    B, _, H, c = value.shape
    Q = loc.shape[1]
    vals = value.permute(0, 2, 3, 1).flatten(0, 1).split([h * w for h, w in shapes], dim=-1)
    grids = (2 * loc - 1).permute(0, 2, 1, 3, 4).flatten(0, 1).split(spec.num_points, dim=-2)
    sampled = [F.grid_sample(vals[l].reshape(B * H, c, h, w), grids[l], mode="bilinear", padding_mode="zeros",
                             align_corners=False) for l, (h, w) in enumerate(shapes)]
    wts = weights.permute(0, 2, 1, 3).reshape(B * H, 1, Q, sum(spec.num_points))
    return (torch.cat(sampled, -1) * wts).sum(-1).reshape(B, H * c, Q).permute(0, 2, 1)


def deform_value(sd, spec, p, memory):
    """value_proj of the memory as (B, L, heads, hidden / heads)"""
    B, _, D = memory.shape
    return F.linear(memory, sd[p + ".value_proj.weight"], sd[p + ".value_proj.bias"]).reshape(B, -1, spec.heads, D // spec.heads)


def deform_offsets_weights(sd, spec, p, query):
    """sampling offsets (B, Q, heads, P, 2) and softmax attention weights (B, Q, heads, P) of the query"""
    B, Q, D = query.shape
    H, P = spec.heads, sum(spec.num_points)
    off = F.linear(query, sd[p + ".sampling_offsets.weight"], sd[p + ".sampling_offsets.bias"]).reshape(B, Q, H, P, 2)
    wts = torch.softmax(F.linear(query, sd[p + ".attention_weights.weight"], sd[p + ".attention_weights.bias"])
                        .reshape(B, Q, H, P), dim=-1)
    return off, wts


def deform_locations(spec, ref4, off):
    """sampling locations in [0, 1]: ref centre + offset / num_points * ref size * offset_scale"""
    scale = torch.tensor([1.0 / n for n in spec.num_points for _ in range(n)], dtype=off.dtype,
                         device=off.device).unsqueeze(-1)
    ref = ref4.unsqueeze(2)                                          # (B, Q, 1, 4): the same box for every level
    return ref[:, :, None, :, :2] + off * scale * ref[:, :, None, :, 2:] * spec.offset_scale


def deform_core(spec, value, shapes, ref4, off, wts):
    """the multi-scale deformable attention of given offsets and weights (before output_proj) -> (B, Q, hidden)"""
    return deformable_attention(spec, value, shapes, deform_locations(spec, ref4, off), wts)


def ms_deform_attn(sd, spec, p, query, ref4, memory, shapes):
    value = deform_value(sd, spec, p, memory)
    off, wts = deform_offsets_weights(sd, spec, p, query)
    out = deform_core(spec, value, shapes, ref4, off, wts)
    return F.linear(out, sd[p + ".output_proj.weight"], sd[p + ".output_proj.bias"])


def self_attn_sublayer(sd, spec, p, tgt, qpos):
    """norm1(tgt + MHA(q = k = tgt + qpos, v = tgt))"""
    q = tgt + qpos
    return _ln(sd, p + ".norm1", tgt + mha(sd, p + ".self_attn", q, q, tgt, spec.heads))


def cross_attn_sublayer(sd, spec, p, tgt, qpos, ref4, memory, shapes):
    """norm2(tgt + MSDeformableAttention(tgt + qpos, ref4, memory))"""
    return _ln(sd, p + ".norm2", tgt + ms_deform_attn(sd, spec, p + ".cross_attn", tgt + qpos, ref4, memory, shapes))


def ffn_sublayer(sd, p, tgt):
    """norm3(tgt + linear2(relu(linear1(tgt))))"""
    return _ln(sd, p + ".norm3", tgt + ffn(sd, p, tgt, "relu"))


def decoder_layer(sd, spec, p, tgt, ref4, memory, shapes, qpos):
    tgt = self_attn_sublayer(sd, spec, p, tgt, qpos)
    tgt = cross_attn_sublayer(sd, spec, p, tgt, qpos, ref4, memory, shapes)
    return ffn_sublayer(sd, p, tgt)


def box_refine(sd, p, tgt, ref):
    """iterative box refinement: sigmoid(bbox MLP(tgt) + inverse_sigmoid(ref))"""
    return torch.sigmoid(mlp(sd, p, tgt, 3) + inverse_sigmoid(ref))


def decoder(sd, spec, feats, aux=None):
    p = "decoder."
    proj = [_bn(sd, "%sinput_proj.%d.norm" % (p, i), F.conv2d(f, sd["%sinput_proj.%d.conv.weight" % (p, i)]))
            for i, f in enumerate(feats)]
    shapes = [list(f.shape[2:]) for f in proj]
    memory = torch.cat([f.flatten(2).permute(0, 2, 1) for f in proj], 1)
    anchors, valid = sd[p + "anchors"], sd[p + "valid_mask"]
    om = _ln(sd, p + "enc_output.norm", F.linear(valid.to(memory.dtype) * memory, sd[p + "enc_output.proj.weight"],
                                                  sd[p + "enc_output.proj.bias"]))
    enc_logits = F.linear(om, sd[p + "enc_score_head.weight"], sd[p + "enc_score_head.bias"])
    enc_boxes = mlp(sd, p + "enc_bbox_head", om, 3) + anchors
    _, ind = torch.topk(enc_logits.max(-1).values, spec.num_queries, dim=-1)
    tgt = om.gather(1, ind.unsqueeze(-1).repeat(1, 1, om.shape[-1]))
    ref_unact = enc_boxes.gather(1, ind.unsqueeze(-1).repeat(1, 1, 4))
    ref = torch.sigmoid(ref_unact)
    if aux is not None:
        aux.update(memory=memory, enc_logits=enc_logits, topk=ind, tgt0=tgt, ref0=ref)
    for i in range(spec.num_layers):
        qpos = mlp(sd, p + "query_pos_head", ref, 2)
        tgt = decoder_layer(sd, spec, "%sdecoder.layers.%d" % (p, i), tgt, ref, memory, shapes, qpos)
        box = box_refine(sd, "%sdec_bbox_head.%d" % (p, i), tgt, ref)
        if i == spec.num_layers - 1:
            logits = F.linear(tgt, sd["%sdec_score_head.%d.weight" % (p, i)], sd["%sdec_score_head.%d.bias" % (p, i)])
            return {"pred_logits": logits, "pred_boxes": box}
        ref = box


@torch.no_grad()
def forward(sd, spec, x, aux=None):
    """x (B, 3, 640, 640) fp32 in [0, 1] -> {"pred_logits" (B, 300, C), "pred_boxes" (B, 300, 4) cxcywh in [0, 1]}."""
    feats = backbone(sd, spec, x)
    enc = hybrid_encoder(sd, spec, feats)
    if aux is not None:
        aux.update(backbone=feats, encoder=enc)
    return decoder(sd, spec, enc, aux)


def postprocess(spec, out, orig_wh, threshold):
    """Focal-loss branch of the reference post-processor: sigmoid, top-num_queries over queries x classes, boxes to
    xyxy pixels of the original image, score filter, clamp.  Returns dict(labels, boxes, scores) of numpy arrays."""
    logits, boxes = out["pred_logits"], out["pred_boxes"]
    cx, cy, w, h = boxes.unbind(-1)
    xyxy = torch.stack([cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h], -1)
    xyxy = xyxy * torch.tensor([orig_wh[0], orig_wh[1]] * 2, dtype=xyxy.dtype, device=xyxy.device)
    scores, index = torch.topk(torch.sigmoid(logits).flatten(1), spec.num_queries, dim=-1)
    labels = index - index // spec.num_classes * spec.num_classes
    sel = xyxy.gather(1, (index // spec.num_classes).unsqueeze(-1).repeat(1, 1, 4))
    lab, box, sco = labels[0], sel[0], scores[0]
    keep = sco > threshold
    box = box[keep].clone()
    box[:, 0].clamp_(min=0)
    box[:, 1].clamp_(min=0)
    box[:, 2].clamp_(min=0, max=orig_wh[0])
    box[:, 3].clamp_(min=0, max=orig_wh[1])
    return dict(labels=lab[keep].numpy(), boxes=box.numpy(), scores=sco[keep].numpy())


# ------------------------------------------------------------------------------------------------ weights
def make_state_dict(spec, seed=0, trained_like=True):
    """Seeded random weights with the reference's key set (tensor shapes as RTDETRv2(cfg).state_dict()).  trained_like:
    BN statistics / affine drawn away from the identity, heads not zero-initialised, so that every path matters."""
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    def conv(name, cout, cin, k):
        sd[name + ".weight"] = rn(cout, cin, k, k, std=math.sqrt(2.0 / (cin * k * k)))

    def bn(name, c, tracked):
        sd[name + ".weight"] = 1.0 + 0.1 * rn(c) if trained_like else torch.ones(c)
        sd[name + ".bias"] = 0.1 * rn(c) if trained_like else torch.zeros(c)
        sd[name + ".running_mean"] = 0.1 * rn(c) if trained_like else torch.zeros(c)
        sd[name + ".running_var"] = (1.0 + 0.2 * torch.rand(c, generator=g)) if trained_like else torch.ones(c)
        if tracked:
            sd[name + ".num_batches_tracked"] = torch.tensor(0)

    def cn(name, cout, cin, k, tracked):
        conv(name + ".conv", cout, cin, k)
        bn(name + ".norm", cout, tracked)

    def lin(name, cout, cin, std=None):
        sd[name + ".weight"] = rn(cout, cin, std=std if std is not None else math.sqrt(1.0 / cin))
        sd[name + ".bias"] = 0.02 * rn(cout)

    def ln(name, c):
        sd[name + ".weight"] = 1.0 + 0.05 * rn(c)
        sd[name + ".bias"] = 0.05 * rn(c)

    cn("backbone.conv1.conv1_1", 32, 3, 3, False)
    cn("backbone.conv1.conv1_2", 32, 32, 3, False)
    cn("backbone.conv1.conv1_3", 64, 32, 3, False)
    cin = 64
    for s, (n, ch) in enumerate(zip(spec.blocks, [64, 128, 256, 512])):
        for b in range(n):
            p = "backbone.res_layers.%d.blocks.%d" % (s, b)
            cn(p + ".branch2a", ch, cin, 1, False)
            cn(p + ".branch2b", ch, ch, 3, False)
            cn(p + ".branch2c", ch * 4, ch, 1, False)
            sd[p + ".branch2c.norm.weight"] *= 0.5                     # keeps the residual stream bounded over 16 blocks
            if b == 0:
                cn(p + (".short.conv" if s != 0 else ".short"), ch * 4, cin, 1, False)
            cin = ch * 4
    D = spec.hidden
    for i, c in enumerate([512, 1024, 2048]):
        conv("encoder.input_proj.%d.conv" % i, D, c, 1)
        bn("encoder.input_proj.%d.norm" % i, D, True)
    p = "encoder.encoder.0.layers.0"
    sd[p + ".self_attn.in_proj_weight"] = rn(3 * D, D, std=math.sqrt(1.0 / D))
    sd[p + ".self_attn.in_proj_bias"] = 0.02 * rn(3 * D)
    lin(p + ".self_attn.out_proj", D, D)
    lin(p + ".linear1", spec.ffn, D)
    lin(p + ".linear2", D, spec.ffn)
    ln(p + ".norm1", D)
    ln(p + ".norm2", D)

    def csp(name):
        cn(name + ".conv1", D, 2 * D, 1, True)
        cn(name + ".conv2", D, 2 * D, 1, True)
        for i in range(spec.csp_blocks):
            cn("%s.bottlenecks.%d.conv1" % (name, i), D, D, 3, True)
            cn("%s.bottlenecks.%d.conv2" % (name, i), D, D, 1, True)

    for i in range(2):
        cn("encoder.lateral_convs.%d" % i, D, D, 1, True)
        csp("encoder.fpn_blocks.%d" % i)
    for i in range(2):
        cn("encoder.downsample_convs.%d" % i, D, D, 3, True)
        csp("encoder.pan_blocks.%d" % i)
    anchors, valid = generate_anchors(spec)
    sd["decoder.anchors"], sd["decoder.valid_mask"] = anchors, valid
    for i in range(3):
        conv("decoder.input_proj.%d.conv" % i, D, D, 1)
        bn("decoder.input_proj.%d.norm" % i, D, True)
    P = sum(spec.num_points)
    for i in range(spec.num_layers):
        p = "decoder.decoder.layers.%d" % i
        sd[p + ".self_attn.in_proj_weight"] = rn(3 * D, D, std=math.sqrt(1.0 / D))
        sd[p + ".self_attn.in_proj_bias"] = 0.02 * rn(3 * D)
        lin(p + ".self_attn.out_proj", D, D)
        ln(p + ".norm1", D)
        sd[p + ".cross_attn.num_points_scale"] = torch.tensor([1.0 / n for n in spec.num_points for _ in range(n)])
        lin(p + ".cross_attn.sampling_offsets", spec.heads * P * 2, D, std=0.02 if trained_like else 0.0)
        th = torch.arange(spec.heads, dtype=torch.float32) * (2.0 * math.pi / spec.heads)
        gi = torch.stack([th.cos(), th.sin()], -1)
        gi = (gi / gi.abs().max(-1, keepdim=True).values).reshape(spec.heads, 1, 2).tile([1, P, 1])
        gi = gi * torch.cat([torch.arange(1, n + 1) for n in spec.num_points]).reshape(1, -1, 1)
        sd[p + ".cross_attn.sampling_offsets.bias"] = gi.flatten()
        lin(p + ".cross_attn.attention_weights", spec.heads * P, D, std=0.05 if trained_like else 0.0)
        lin(p + ".cross_attn.value_proj", D, D)
        lin(p + ".cross_attn.output_proj", D, D)
        ln(p + ".norm2", D)
        lin(p + ".linear1", spec.ffn, D)
        lin(p + ".linear2", D, spec.ffn)
        ln(p + ".norm3", D)
    sd["decoder.denoising_class_embed.weight"] = rn(spec.num_classes + 1, D)
    lin("decoder.query_pos_head.layers.0", 2 * D, 4, std=0.5)
    lin("decoder.query_pos_head.layers.1", D, 2 * D)
    lin("decoder.enc_output.proj", D, D)
    # positions outside the valid mask see a zero memory row: with a zero bias their LayerNorm input is exactly zero and
    # their class scores equal the head bias (low) - as in a trained model they never reach the top-300 (with a random
    # bias ~ 1900 identical scores would tie inside the selection)
    sd["decoder.enc_output.proj.bias"] = torch.zeros(D)
    ln("decoder.enc_output.norm", D)
    lin("decoder.enc_score_head", spec.num_classes, D, std=0.3 if trained_like else None)
    sd["decoder.enc_score_head.bias"] = torch.full((spec.num_classes,), -math.log(99.0)) + 0.1 * rn(spec.num_classes)
    for name in ["decoder.enc_bbox_head"] + ["decoder.dec_bbox_head.%d" % i for i in range(spec.num_layers)]:
        lin(name + ".layers.0", D, D)
        lin(name + ".layers.1", D, D)
        lin(name + ".layers.2", 4, D, std=0.02 if trained_like else 0.0)
    for i in range(spec.num_layers):
        lin("decoder.dec_score_head.%d" % i, spec.num_classes, D, std=0.3 if trained_like else None)
        sd["decoder.dec_score_head.%d.bias" % i] = torch.full((spec.num_classes,), -2.0) + 0.1 * rn(spec.num_classes)
    return sd
