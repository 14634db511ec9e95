"""Aggregates a YTK_GEMM_DUMP file (one line per gemm_tc_kernel launch of a bench.py profiling window: shape, epilogue,
CUDA-event duration, epilogue path epi (1 = TMA, 0 = staged) and tile patch bw_log2) by shape: launches, total ms,
TFLOP/s, algorithmic operand + result bytes and the GB/s they imply.
    YTK_GEMM_DUMP=gpurun_out/gemm_dump.csv python bench.py --steps 1 --warmup 3 --no-e2e --no-cpu --no-extra
    python scripts/gemm_shape_table.py gpurun_out/gemm_dump.csv [out.json]"""
import csv
import json
import sys
from collections import OrderedDict

rows = [r for r in csv.DictReader(l for l in open(sys.argv[1]) if not l.startswith("pixels") or "cout" in l)
        if r["pixels"] != "pixels"]
agg = OrderedDict()
for r in rows:
    key = (int(r["pixels"]), int(r["cout"]), int(r["k"]), int(r["ntaps"]), int(r["block_n"]), int(r["epi"]),
           int(r["mode"]), int(r["act"]), int(r["resid"]), int(r["out_f32"]))
    a = agg.setdefault(key, {"n": 0, "ms": 0.0, "flops": 0.0})
    a["n"] += 1
    a["ms"] += float(r["ms"])
    a["flops"] += float(r["flops"])
total_ms = sum(a["ms"] for a in agg.values())
out = []
for key, a in sorted(agg.items(), key=lambda kv: -kv[1]["ms"]):
    pixels, cout, k, ntaps, bn, epi, mode, act, resid, of32 = key
    # algorithmic bytes per launch: the input once (for a conv: the un-expanded NHWC input of k channels), the weights,
    # the result (fp16 or fp32; mode 3 = row statistics only) and the residual if any
    in_b = pixels * k * 2
    w_b = cout * k * ntaps * 2
    out_b = 0 if mode == 3 else pixels * cout * (4 if of32 else 2)
    res_b = pixels * cout * (0, 2, 4)[resid]
    byt = in_b + w_b + out_b + res_b
    ms = a["ms"] / a["n"]
    out.append({"pixels": pixels, "cout": cout, "k": k, "taps": ntaps, "block_n": bn, "epi": epi, "mode": mode,
                "act": act, "resid": resid, "out_f32": of32, "launches": a["n"], "ms_total": round(a["ms"], 3),
                "share": round(a["ms"] / total_ms, 4), "ms_per_launch": round(ms, 4),
                "tflops": round(a["flops"] / a["n"] / ms / 1e9, 1), "alg_gb_per_s": round(byt / ms / 1e6, 0),
                "alg_mb": round(byt / 1e6, 1)})
print("%9s %5s %5s %4s %3s %2s %1s %1s %1s %1s | %4s %8s %6s %8s %7s %8s" % (
    "pixels", "cout", "k", "taps", "bn", "e", "m", "a", "r", "f", "n", "ms_tot", "share", "ms/launch", "TFLOP/s", "algGB/s"))
for o in out:
    print("%9d %5d %5d %4d %3d %2d %1d %1d %1d %1d | %4d %8.2f %6.3f %8.4f %7.0f %8.0f" % (
        o["pixels"], o["cout"], o["k"], o["taps"], o["block_n"], o["epi"], o["mode"], o["act"], o["resid"],
        o["out_f32"], o["launches"], o["ms_total"], o["share"], o["ms_per_launch"], o["tflops"], o["alg_gb_per_s"]))
print("total %.2f ms over %d launches" % (total_ms, len(rows)))
if len(sys.argv) > 2:
    json.dump({"total_ms": total_ms, "launches": len(rows), "shapes": out}, open(sys.argv[2], "w"), indent=1)
