"""GPU probe: DBNet engine vs the CPU oracle, layer by layer (writes gpurun_out/probe_dbnet.json)."""
import ctypes
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import dbnet as odb  # noqa: E402
from oracle import weights  # noqa: E402
from yomitoku_b200 import _lib  # noqa: E402
from yomitoku_b200.models import DBNet  # noqa: E402

L = _lib.lib()
out = []


def log(**kw):
    out.append(kw)
    print(json.dumps(kw), flush=True)


def cmp(name, got, ref):
    d = (got - ref).abs()
    log(name=name, shape=list(ref.shape), max_abs=d.max().item(), mean_abs=d.mean().item(),
        ref_absmax=ref.abs().max().item(), ref_absmean=ref.abs().mean().item(),
        rel_fro=(d.norm() / (ref.norm() + 1e-12)).item())


def main():
    torch.manual_seed(0)
    sd = weights.make_dbnet_state_dict(seed=1)
    model = DBNet().load_state_dict(sd)     # shortest 1280, limit 1600
    h = model._ensure()
    # ---------------- model-level seam on a small input, with intermediates
    H, W = 256, 384
    x = torch.randn(1, 3, H, W)
    prob = torch.empty(1, H, W)
    t0 = time.time()
    st = L.ytk_dbnet_forward_f32(h, x.data_ptr(), 0, 1, H, W, prob.data_ptr(), 0, None)
    if st != 0:
        log(fatal=L.ytk_last_error().decode())
        return
    log(name="forward_f32 small", wall_s=time.time() - t0)
    with torch.inference_mode():
        p = "backbone.body."
        s = F.relu(odb._bn(sd, p + "bn1", F.conv2d(x, sd[p + "conv1.weight"], stride=2, padding=3)))
        cmp("stem", model.debug_tensor(1, H, W, "stem"), s.permute(0, 2, 3, 1))
        cmp("pool", model.debug_tensor(1, H, W, "pool"), F.max_pool2d(s, 3, 2, 1).permute(0, 2, 3, 1))
        feats = odb.backbone_features(sd, x)
        for k in ("layer1", "layer2", "layer3", "layer4"):
            cmp(k, model.debug_tensor(1, H, W, k), feats[k].permute(0, 2, 3, 1))
        ref = odb.decoder_forward(sd, feats)
    cmp("prob small", prob, ref[:, 0])
    # ---------------- full-size page through the fused u8 path
    rng = np.random.default_rng(0)
    page = rng.integers(0, 256, size=(1200, 1600, 3), dtype=np.uint8)
    Hn, Wn = ctypes.c_int(), ctypes.c_int()
    L.ytk_dbnet_input_size(h, 1200, 1600, ctypes.byref(Hn), ctypes.byref(Wn))
    Hn, Wn = Hn.value, Wn.value
    log(name="input_size", Hn=Hn, Wn=Wn)
    pt = torch.from_numpy(page)
    prob = torch.empty(1, Hn, Wn)
    st = L.ytk_dbnet_forward_u8(h, pt.data_ptr(), 0, 1, 1200, 1600, prob.data_ptr(), 0, None)
    if st != 0:
        log(fatal=L.ytk_last_error().decode())
        return
    import cv2
    img = page[:, :, ::-1].astype(np.float32)
    res = cv2.resize(img, (Wn, Hn), interpolation=cv2.INTER_AREA)
    res = res[:, :, ::-1] / 255.0
    res = ((res - np.array((0.485, 0.456, 0.406))) / np.array((0.229, 0.224, 0.225))).astype(np.float32)
    xt = torch.from_numpy(np.transpose(res, (2, 0, 1)).copy())[None]
    t0 = time.time()
    ref = odb.dbnet_forward(sd, xt)
    log(name="oracle full page cpu_s", wall_s=time.time() - t0, threads=torch.get_num_threads())
    cmp("prob full u8", prob, ref[:, 0])
    # preprocessing alone: compare the padded canvas via the stem? use forward_f32 on the oracle-preprocessed tensor
    prob2 = torch.empty(1, Hn, Wn)
    L.ytk_dbnet_forward_f32(h, xt.data_ptr(), 0, 1, Hn, Wn, prob2.data_ptr(), 0, None)
    cmp("prob full f32-seam", prob2, ref[:, 0])
    cmp("u8 path vs f32-seam path", prob, prob2)
    # ---------------- timing, device-resident input
    for n in (1, 4):
        pages = torch.from_numpy(rng.integers(0, 256, size=(n, 1200, 1600, 3), dtype=np.uint8)).cuda()
        pout = torch.empty(n, Hn, Wn, device="cuda")
        for _ in range(3):
            L.ytk_dbnet_forward_u8(h, pages.data_ptr(), 1, n, 1200, 1600, pout.data_ptr(), 1, None)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = 10
        e0.record()
        for _ in range(iters):
            L.ytk_dbnet_forward_u8(h, pages.data_ptr(), 1, n, 1200, 1600, pout.data_ptr(), 1, None)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        fl = L.ytk_dbnet_flops(h, n, Hn, Wn)
        log(name="time dbnet n=%d" % n, ms=ms, pages_per_s=n / ms * 1e3, gflop=fl / 1e9, tflops=fl / ms / 1e9)
    model._release()


if __name__ == "__main__":
    try:
        main()
    except Exception as e:
        import traceback
        traceback.print_exc()
        log(fatal=repr(e))
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(out, open("gpurun_out/probe_dbnet.json", "w"), indent=1)
