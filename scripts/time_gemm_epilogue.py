"""Times gemm_tc_kernel at the linear-layer shapes of one bench step with CUDA events: ms per launch, achieved TFLOP/s
and algorithmic GB/s (A once, W once, the result, the residual if any), and ms per bench step (x launches per step).

    python scripts/time_gemm_epilogue.py --lib build/parent/libytk_b200.so --out /tmp/gemm_parent.json
    python scripts/time_gemm_epilogue.py --out /tmp/gemm_new.json          # the in-tree library

--lib loads another build of the library (e.g. the parent commit's, kept under an ignored build/ directory), so that
two builds can alternate in one session.  The DBNet convolutions are timed per launch by bench.py's profiling window
(YTK_GEMM_DUMP=<csv>)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from yomitoku_b200 import _lib  # noqa: E402

D, F = 768, 3072
ENC_M, AR_M, REF_M = 424448, 3200, 323200   # bench step: 16 pages, 3200 crops, 101 decode steps
# name, M, K, N, act, residual ("f32": fp32 in place, the residual stream), fp32 output, launches per step
SHAPES = [
    ("enc.qkv", ENC_M, D, 3 * D, 0, None, False, 12),
    ("enc.proj", ENC_M, D, D, 0, "f32", True, 12),
    ("enc.fc1", ENC_M, D, F, 2, None, False, 12),
    ("enc.fc2", ENC_M, F, D, 0, "f32", True, 12),
    ("ar.lin", AR_M, D, D, 0, None, False, 101 * 3),
    ("ar.lin_resid", AR_M, D, D, 0, "f32", True, 101 * 2),
    ("ar.fc1", AR_M, D, F, 2, None, False, 101),
    ("ar.fc2", AR_M, F, D, 0, "f32", True, 101),
    ("ref.lin", REF_M, D, D, 0, None, False, 3),
    ("ref.lin_resid", REF_M, D, D, 0, "f32", True, 2),
    ("ref.fc1", REF_M, D, F, 2, None, False, 1),
    ("ref.fc2", REF_M, F, D, 0, "f32", True, 1),
]


def time_shape(L, M, K, N, act, resid, f32, iters, warmup):
    dev = "cuda:0"
    g = torch.Generator(device=dev).manual_seed(0)
    A = (torch.randn(M, K, device=dev, generator=g) * 0.5).half()
    W = (torch.randn(N, K, device=dev, generator=g) * 0.05).half()
    b = torch.randn(N, device=dev, generator=g)
    out = torch.randn(M, N, device=dev, generator=g) if f32 else torch.empty(M, N, device=dev, dtype=torch.float16)
    R = out if resid == "f32" else None

    def run():
        _lib.check(L.ytk_op_linear_f16(_lib.ptr(A), K, M, K, _lib.ptr(W), N, _lib.ptr(b), _lib.ptr(R),
                                        1 if resid == "f32" else 0, N, _lib.ptr(out), 1 if f32 else 0, N, act, None))
    for _ in range(warmup):
        run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    byt = M * K * 2 + N * K * 2 + M * N * (4 if f32 else 2) + (M * N * 4 if resid else 0)
    return ms, 2.0 * M * N * K / ms / 1e9, byt / ms / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="library to load instead of the in-tree build")
    ap.add_argument("--out", default=None, help="JSON result file")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_gemm_epilogue: needs a GPU")
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    L = _lib.lib()
    rows = []
    for name, M, K, N, act, resid, f32, per_step in SHAPES:
        iters = max(3, min(args.iters, int(args.iters * 3200 * 50 / M))) if M > 100000 else args.iters * 10
        ms, tf, gbs = time_shape(L, M, K, N, act, resid, f32, iters, args.warmup)
        rows.append({"shape": name, "M": M, "K": K, "N": N, "ms": round(ms, 4), "tflops": round(tf, 1),
                     "gb_per_s": round(gbs, 0), "per_step": per_step, "ms_per_step": round(ms * per_step, 3)})
        print("%-14s M=%7d K=%5d N=%5d  %8.4f ms  %6.1f TFLOP/s  %6.0f GB/s  x%4d = %8.3f ms/step" % (
            name, M, K, N, ms, tf, gbs, per_step, ms * per_step), flush=True)
    print("total %.3f ms per step" % sum(r["ms_per_step"] for r in rows))
    if args.out:
        json.dump({"lib": _lib.LIB_PATH, "gpu": torch.cuda.get_device_name(0), "rows": rows}, open(args.out, "w"),
                  indent=1)


if __name__ == "__main__":
    main()
