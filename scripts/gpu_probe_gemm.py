"""GPU probe for the wgmma implicit-GEMM kernel: runs many shapes against torch fp32 references and writes
per-case error statistics to $YTK_REPORT_DIR/probe_gemm.json (default: the current directory).  Never aborts on a mismatch (diagnostics first)."""
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from yomitoku_b200 import _lib  # noqa: E402

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
L = _lib.lib()
dev = "cuda:0"
results = []


def stats(name, got, ref, extra=None):
    got = got.float()
    ref = ref.float()
    diff = (got - ref).abs()
    denom = ref.abs().max().item() + 1e-12
    r = {
        "case": name,
        "max_abs": diff.max().item(),
        "ref_absmax": denom,
        "rel": diff.max().item() / denom,
        "nan": bool(torch.isnan(got).any().item()),
        "got_absmax": got.abs().max().item(),
    }
    if r["rel"] > 2e-2 or r["nan"]:
        bad = (diff > 2e-2 * denom).nonzero()
        r["n_bad"] = int(bad.shape[0])
        r["first_bad"] = bad[:12].tolist()
        idx = tuple(bad[0].tolist()) if bad.shape[0] else None
        if idx is not None:
            r["bad_got"] = got[idx].item()
            r["bad_ref"] = ref[idx].item()
        # row / column structure of the error
        d2 = diff.reshape(-1, diff.shape[-1])
        r["bad_rows"] = (d2.max(1).values > 2e-2 * denom).nonzero().flatten()[:40].tolist()
        r["bad_cols"] = (d2.max(0).values > 2e-2 * denom).nonzero().flatten()[:40].tolist()
    if extra:
        r.update(extra)
    results.append(r)
    print(json.dumps(r), flush=True)


def run_linear(M, K, N, bias=True, act=0, resid=None, out_f32=False, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = (torch.randn(M, K, generator=g) * 0.5).to(dev).half()
    W = (torch.randn(N, K, generator=g) * 0.1).to(dev).half()
    b = torch.randn(N, generator=g).to(dev) if bias else None
    ldc = (N + 7) // 8 * 8
    R = None
    if resid == "f32":
        R = torch.randn(M, ldc, generator=g).to(dev)
    elif resid == "f16":
        R = torch.randn(M, ldc, generator=g).to(dev).half()
    out = torch.full((M, ldc), 7.0, device=dev, dtype=torch.float32 if out_f32 else torch.float16)
    st = L.ytk_op_linear_f16(_lib.ptr(A), K, M, K, _lib.ptr(W), N, _lib.ptr(b), _lib.ptr(R),
                              1 if resid == "f32" else 0, ldc, _lib.ptr(out), 1 if out_f32 else 0, ldc, act, None)
    name = "linear M%d K%d N%d b%d act%d res%s f32%d" % (M, K, N, bias, act, resid, out_f32)
    if st != 0:
        results.append({"case": name, "error": L.ytk_last_error().decode()})
        print(results[-1], flush=True)
        return
    torch.cuda.synchronize()
    ref = A.float() @ W.float().t()
    if bias:
        ref = ref + b
    if R is not None:
        ref = ref + R[:, :N].float()
    if act == 1:
        ref = ref.relu()
    elif act == 2:
        ref = F.gelu(ref)
    elif act == 3:
        ref = ref.sigmoid()
    stats(name, out[:, :N], ref)


def run_conv(N, H, W, Cin, Cout, k, stride, pad, dil, bias=True, act=0, resid=False, out_f32=False, mode=0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = (torch.randn(N, H, W, Cin, generator=g) * 0.5).to(dev).half()  # NHWC
    if mode == 1:
        # ConvTranspose2d(k=2,s=2) weight [Cin, Cq, 2, 2]; GEMM weight rows = (i,j,co)
        Cq = Cout // 4
        wt = (torch.randn(Cin, Cq, 2, 2, generator=g) * 0.1).to(dev).half()
        wp = wt.permute(2, 3, 1, 0).reshape(Cout, Cin).contiguous()
        b = torch.randn(Cq, generator=g).to(dev) if bias else None
        bfull = b.repeat(4).contiguous() if bias else None
        Ho, Wo = H, W
        out = torch.full((N, 2 * Ho, 2 * Wo, Cq), 7.0, device=dev, dtype=torch.float32 if out_f32 else torch.float16)
        st = L.ytk_op_conv2d_f16(_lib.ptr(x), N, H, W, Cin, Cin, _lib.ptr(wp), _lib.ptr(bfull), 1, 1, 1, 0, 1, Cout,
                                  None, 0, 0, _lib.ptr(out), 1 if out_f32 else 0, Cq, act, 1, None)
        name = "convT2x2 N%d H%d W%d Cin%d Cq%d act%d" % (N, H, W, Cin, Cq, act)
        if st != 0:
            results.append({"case": name, "error": L.ytk_last_error().decode()})
            print(results[-1], flush=True)
            return
        torch.cuda.synchronize()
        ref = F.conv_transpose2d(x.float().permute(0, 3, 1, 2), wt.float(), b, stride=2)
        if act == 1:
            ref = ref.relu()
        stats(name, out, ref.permute(0, 2, 3, 1))
        return
    w = (torch.randn(Cout, Cin, k, k, generator=g) * (1.0 / (Cin * k * k) ** 0.5)).to(dev).half()
    wp = w.permute(0, 2, 3, 1).contiguous()  # [Cout][kh][kw][Cin]
    b = torch.randn(Cout, generator=g).to(dev) if bias else None
    Ho = (H + 2 * pad - dil * (k - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - dil * (k - 1) - 1) // stride + 1
    R = (torch.randn(N, Ho, Wo, Cout, generator=g)).to(dev).half() if resid else None
    out = torch.full((N, Ho, Wo, Cout), 7.0, device=dev, dtype=torch.float32 if out_f32 else torch.float16)
    t0 = time.time()
    st = L.ytk_op_conv2d_f16(_lib.ptr(x), N, H, W, Cin, Cin, _lib.ptr(wp), _lib.ptr(b), k, k, stride, pad, dil, Cout,
                              _lib.ptr(R), 0, Cout, _lib.ptr(out), 1 if out_f32 else 0, Cout, act, 0, None)
    name = "conv N%d H%d W%d Cin%d Cout%d k%d s%d p%d d%d act%d res%d f32%d" % (
        N, H, W, Cin, Cout, k, stride, pad, dil, act, resid, out_f32)
    if st != 0:
        results.append({"case": name, "error": L.ytk_last_error().decode()})
        print(results[-1], flush=True)
        return
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b, stride=stride, padding=pad, dilation=dil)
    ref = ref.permute(0, 2, 3, 1)
    if R is not None:
        ref = ref + R.float()
    if act == 1:
        ref = ref.relu()
    stats(name, out, ref, {"wall_s": time.time() - t0})


def timed_conv(N, H, W, Cin, Cout, k, stride, pad, dil, iters=20):
    x = (torch.randn(N, H, W, Cin, device=dev) * 0.5).half()
    wp = (torch.randn(Cout, k, k, Cin, device=dev) * 0.02).half()
    b = torch.randn(Cout, device=dev)
    Ho = (H + 2 * pad - dil * (k - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - dil * (k - 1) - 1) // stride + 1
    out = torch.empty((N, Ho, Wo, Cout), device=dev, dtype=torch.float16)
    args = (_lib.ptr(x), N, H, W, Cin, Cin, _lib.ptr(wp), _lib.ptr(b), k, k, stride, pad, dil, Cout, None, 0, 0,
            _lib.ptr(out), 0, Cout, 1, 0, None)
    for _ in range(3):
        L.ytk_op_conv2d_f16(*args)
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True)
    e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        L.ytk_op_conv2d_f16(*args)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    fl = 2.0 * N * Ho * Wo * Cout * Cin * k * k
    r = {"case": "time conv N%d H%d W%d Cin%d Cout%d k%d s%d d%d" % (N, H, W, Cin, Cout, k, stride, dil), "ms": ms,
         "tflops": fl / ms / 1e9}
    results.append(r)
    print(json.dumps(r), flush=True)


def main():
    print(torch.cuda.get_device_name(0), flush=True)
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    try:
        run_linear(128, 64, 64, bias=False, out_f32=True)
        run_linear(128, 64, 64, bias=False)
        run_linear(128, 256, 64)
        run_linear(128, 1024, 64)
        run_linear(128, 64, 128, bias=False, out_f32=True)
        run_linear(128, 64, 256, bias=False, out_f32=True)
        run_linear(300, 128, 200)
        run_linear(1000, 768, 2304, act=2)
        run_linear(517, 768, 7119, out_f32=True)
        run_linear(640, 3072, 768, resid="f32", out_f32=True)
        run_linear(33, 192, 576, resid="f16", act=1)
        run_conv(1, 16, 24, 64, 64, 1, 1, 0, 1, bias=False, out_f32=True)
        run_conv(1, 16, 24, 64, 64, 3, 1, 1, 1)
        run_conv(2, 37, 50, 128, 256, 3, 1, 1, 1, act=1)
        run_conv(1, 37, 50, 128, 128, 3, 1, 2, 2, act=1, resid=True)
        run_conv(1, 38, 52, 64, 128, 3, 2, 1, 1, act=1)
        run_conv(1, 37, 51, 64, 128, 3, 2, 1, 1, act=1)
        run_conv(2, 38, 52, 256, 512, 1, 2, 0, 1)
        run_conv(1, 20, 28, 64, 256, 1, 1, 0, 1, mode=1, act=1)
        run_conv(1, 74, 100, 512, 512, 3, 1, 2, 2, act=1)
        run_conv(1, 296, 400, 256, 64, 3, 1, 1, 1, bias=False)
        if which == "all":
            timed_conv(1, 74, 100, 512, 512, 3, 1, 2, 2)
            timed_conv(1, 296, 400, 256, 64, 3, 1, 1, 1)
            timed_conv(1, 74, 100, 1024, 2048, 1, 1, 0, 1)
            timed_conv(1, 296, 400, 64, 64, 3, 1, 1, 1)
            timed_conv(8, 74, 100, 512, 512, 3, 1, 2, 2)
    except Exception as e:  # keep whatever we have
        results.append({"fatal": repr(e)})
        print("FATAL", repr(e), flush=True)
    out_dir = os.environ.get("YTK_REPORT_DIR", ".")
    os.makedirs(out_dir, exist_ok=True)
    json.dump(results, open(os.path.join(out_dir, "probe_gemm.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
