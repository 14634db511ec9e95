"""Host pages vs pages already on the GPU, on one GPU: the same synthetic mixed-size pages given as numpy arrays (staged,
uploaded) and as CUDA uint8 tensors (packed in HBM by device_pages, no PCIe crossing), in two workloads:

  stream    BatchedOCR.stream over `--batches` batches of `--pages` pages of four sizes
  analyze   DocumentAnalyzer.analyze_pages on one such batch (OCR half and layout half)

plus the pack kernel on its own (device_pages of one batch, CUDA events over `--pack-iters` launches, bytes moved =
one read + one write of every page).  Detector: the seeded random DBNet with the trained binarize head
(tests/golden/dbnet_head_trained.npz); recognizer: parseq-tiny-dynw-v4 with peaked seeded weights; layout models:
seeded random.  Every arm is warmed up first, the two input forms alternate in each repetition, each timed run ends in
a device synchronise, and the device-input results must equal the host-input results.  Prints one JSON line with the
card name and its power limit.

    python scripts/time_device_pages.py --reps 3 --out /tmp/device_pages.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SIZES = [(1200, 1600), (900, 1200), (1000, 1000), (1600, 1200)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [v.strip() for v in out.split(",")[:2]]
        return name, limit
    except Exception as e:      # the numbers are still reported, marked as unattributed
        return "unknown (%s)" % e, "unknown"


def _words(results):
    return [[(w.points, w.content, w.det_score, w.rec_score) for w in r.words] for r in results]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--pages", type=int, default=16)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--pack-iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from oracle import parseq as ops
    from oracle import weights
    from trained_head import load_trained_head
    from yomitoku_b200 import DocumentAnalyzer, device_pages
    from yomitoku_b200.synth import synthetic_page

    if not torch.cuda.is_available():
        raise SystemExit("time_device_pages.py measures on a GPU; none is visible")
    cfg = {"ocr": {"text_detector": {"from_pretrained": False},
                   "text_recognizer": {"from_pretrained": False, "model_name": "parseq-tiny-dynw-v4",
                                       "dynamic_width": True, "batch_bucketing": True}},
           "layout_analyzer": {"layout_parser": {"from_pretrained": False},
                               "table_structure_recognizer": {"from_pretrained": False}}}
    an = DocumentAnalyzer(configs=cfg, device="cuda")
    an.text_recognizer.model.load_state_dict(weights.make_parseq_state_dict(ops.SPECS["parseq-tiny-dynw-v4"], seed=11,
                                                                            peaked=True))
    load_trained_head(an.text_detector.model)
    an.analyze_pages([synthetic_page(0, height=64, width=64)[0]])         # builds the BatchedOCR
    ocr = an._batched

    sizes = [SIZES[i % len(SIZES)] for i in range(args.pages)]
    batches = [[synthetic_page(1000 + b * args.pages + i, height=h, width=w)[0] for i, (h, w) in enumerate(sizes)]
               for b in range(args.batches)]
    dev_batches = [[torch.from_numpy(p).cuda() for p in pages] for pages in batches]
    n_pages = args.pages * args.batches

    def run_stream(device):
        return [r for res in ocr.stream(dev_batches if device else batches, lookahead=2) for r in res]

    def run_analyze(device):
        return an.analyze_pages(dev_batches[0] if device else batches[0])

    arms = {"stream": (run_stream, n_pages), "analyze": (run_analyze, args.pages)}
    times = {"%s_%s" % (a, f): [] for a in arms for f in ("host", "device")}
    for name, (fn, _) in arms.items():               # warm-up, and the results must not depend on the input form
        host, dev = fn(False), fn(True)
        if name == "stream":
            assert _words(host) == _words(dev), "stream: device input differs from host input"
        else:
            assert [r.model_dump() for r in host] == [r.model_dump() for r in dev], "analyze: results differ"
    for _ in range(args.reps):
        for name, (fn, _) in arms.items():
            for form in ("host", "device"):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(form == "device")
                torch.cuda.synchronize()
                times["%s_%s" % (name, form)].append(time.perf_counter() - t0)

    # the pack kernel alone, one batch
    views = dev_batches[0]
    device_pages(views)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.pack_iters):
        dp = device_pages(views)
    e1.record()
    torch.cuda.synchronize()
    pack_ms = e0.elapsed_time(e1) / args.pack_iters
    pack_bytes = 2 * dp.buf.numel()

    name, limit = card()
    res = {"card": name, "power_limit": limit, "pages_per_batch": args.pages, "batches": args.batches,
           "sizes": SIZES, "reps": args.reps,
           "pack": {"ms": round(pack_ms, 4), "bytes": pack_bytes, "GB_per_s": round(pack_bytes / pack_ms / 1e6, 1),
                    "note": "per device_pages call, host record preparation included"}}
    for key, ts in times.items():
        n = arms[key.split("_")[0]][1]
        med = float(np.median(ts))
        res[key] = {"pages_per_s": round(n / med, 2), "median_s": round(med, 4), "min_s": round(min(ts), 4),
                    "max_s": round(max(ts), 4)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    ocr.close()


if __name__ == "__main__":
    main()
