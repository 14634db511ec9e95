"""Throughput of the command line against the analysis it drives, on one GPU.  N synthetic 1200x1600 pages are written
as JPEG files into a temporary directory, then timed:

  decode        load_image of every file, one thread (what the CLI's decode thread does per batch)
  analyze       DocumentAnalyzer.analyze_pages on the already-decoded pages, --batch pages per call
  cli_json      cli.run over the directory, -f json
  cli_md_fig    cli.run over the directory, -f md --figure

Models: the seeded random DBNet with the trained binarize head (tests/golden/dbnet_head_trained.npz),
parseq-tiny-dynw-v4 with peaked seeded weights, the seeded random layout models (random layout weights find junk
regions, so that half dominates the time; `--no-layout` runs the OCR half alone).  Every arm is warmed up once, the arms
alternate in each repetition, and each timed run ends in a device synchronise.  Outputs go to a temporary directory.
Prints one JSON line with the card's name and power limit.

    python scripts/time_cli.py --pages 32 --batch 16 --reps 3 --out /tmp/time_cli.json
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from time_device_pages import card  # noqa: E402  (this script's directory is on the path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=32)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-layout", action="store_true", help="DocumentAnalyzer(layout_analyzer=False): OCR only")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import cv2
    import torch

    from oracle import parseq as ops
    from oracle import weights
    from trained_head import load_trained_head
    from yomitoku_b200 import DocumentAnalyzer, cli
    from yomitoku_b200.data import load_image
    from yomitoku_b200.synth import synthetic_page

    if not torch.cuda.is_available():
        raise SystemExit("time_cli.py measures on a GPU; none is visible")
    cfg = {"ocr": {"text_detector": {"from_pretrained": False},
                   "text_recognizer": {"from_pretrained": False, "model_name": "parseq-tiny-dynw-v4",
                                       "dynamic_width": True, "batch_bucketing": True}},
           "layout_analyzer": {"layout_parser": {"from_pretrained": False},
                               "table_structure_recognizer": {"from_pretrained": False}}}
    an = DocumentAnalyzer(configs=cfg, device="cuda", layout_analyzer=False if args.no_layout else None)
    an.text_recognizer.model.load_state_dict(weights.make_parseq_state_dict(ops.SPECS["parseq-tiny-dynw-v4"], seed=11,
                                                                            peaked=True))
    load_trained_head(an.text_detector.model)

    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "scans")
        os.makedirs(src)
        for i in range(args.pages):
            cv2.imwrite(os.path.join(src, "page%03d.jpg" % i), synthetic_page(2000 + i)[0])
        files = sorted(os.path.join(src, f) for f in os.listdir(src))
        decoded = [load_image(f)[0] for f in files]

        def decode():
            for f in files:
                load_image(f)

        def analyze():
            for k in range(0, len(decoded), args.batch):
                an.analyze_pages(decoded[k:k + args.batch])

        def run_cli(*fmt):
            out = tempfile.mkdtemp(dir=tmp)
            cli.run(cli.build_parser().parse_args([src, "-o", out, "--batch", str(args.batch), *fmt]), an)

        arms = {"decode": decode, "analyze": analyze, "cli_json": lambda: run_cli("-f", "json"),
                "cli_md_fig": lambda: run_cli("-f", "md", "--figure")}
        for fn in arms.values():          # warm-up: every shape and code path of the timed window
            fn()
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for name, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                times[name].append(time.perf_counter() - t0)

    name, limit = card()
    res = {"card": name, "power_limit": limit, "pages": args.pages, "batch": args.batch, "page_hw": [1200, 1600],
           "reps": args.reps, "layout": "none" if args.no_layout else "seeded random"}
    for key, ts in times.items():
        med = float(np.median(ts))
        res[key] = {"pages_per_s": round(args.pages / med, 2), "median_s": round(med, 4), "min_s": round(min(ts), 4),
                    "max_s": round(max(ts), 4)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    an._batched.close()


if __name__ == "__main__":
    main()
