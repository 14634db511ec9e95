"""One step of 16 pages of four sizes (four of each, interleaved) through the OCR path on one GPU, in three arms:

  mixed     one BatchedOCR call on the whole mixed batch (page table, one group per detector input size)
  grouped   the same pages sorted by size and sent as one same-size BatchedOCR call per size (what a caller had to do
            while batches had to be of one size)
  per_page  one OCR(page) call per page

Detector: the seeded random DBNet with the trained binarize head (tests/golden/dbnet_head_trained.npz), so its own maps
carry the synthetic pages' text lines; recognizer: parseq-tiny-dynw-v4 with peaked seeded weights.  Every arm is warmed
up on every shape first; each timed repetition ends in a device synchronise.  The arms are run alternately, and each
arm's result must equal the per-page calls (points and contents).  Prints and writes one JSON line with pages/s per
arm (median and spread over the repetitions), the card name and its power limit.

    python scripts/time_mixed_batch.py --reps 5 --out /tmp/mixed_batch.json
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

SIZES = [(1200, 1600), (900, 1200), (1000, 1000), (1600, 1200)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [v.strip() for v in out.split(",")[:2]]
        return name, limit
    except Exception as e:      # the numbers are still reported, marked as unattributed
        return "unknown (%s)" % e, "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--per-size", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from oracle import parseq as ops
    from oracle import weights
    from yomitoku_b200 import OCR
    from yomitoku_b200.pipeline import BatchedOCR
    from yomitoku_b200.synth import synthetic_page

    if not torch.cuda.is_available():
        raise SystemExit("time_mixed_batch.py measures on a GPU; none is visible")
    o = OCR(configs={"text_detector": {"from_pretrained": False},
                     "text_recognizer": {"from_pretrained": False, "model_name": "parseq-tiny-dynw-v4",
                                         "dynamic_width": True, "batch_bucketing": True}}, device="cuda")
    o.recognizer.model.load_state_dict(weights.make_parseq_state_dict(ops.SPECS["parseq-tiny-dynw-v4"], seed=11,
                                                                      peaked=True))
    z = np.load(os.path.join(ROOT, "tests", "golden", "dbnet_head_trained.npz"))
    o.detector.model.load_state_dict({k: torch.from_numpy(z[k]) for k in z.files}, strict=False)

    pages = [synthetic_page(500 + k, height=SIZES[k % len(SIZES)][0], width=SIZES[k % len(SIZES)][1])[0]
             for k in range(args.per_size * len(SIZES))]
    groups = [[p for p in pages if p.shape[:2] == s] for s in SIZES]
    b = BatchedOCR(o.detector, o.recognizer, det_batch=8)

    def run(arm):
        if arm == "mixed":
            res = b(pages)
            return res
        if arm == "grouped":
            by = {}
            for g in groups:
                for p, r in zip(g, b(g)):
                    by[id(p)] = r
            return [by[id(p)] for p in pages]
        return [o(p)[0] for p in pages]

    arms = ["mixed", "grouped", "per_page"]
    ref = None
    for arm in arms:            # warm-up: every shape, every engine, the worker pool
        res = run(arm)
        key = [[(w.points, w.content) for w in r.words] for r in res]
        if ref is None:
            ref = key
        assert key == ref, "arm %s differs from the mixed batch" % arm
    torch.cuda.synchronize()
    times = {a: [] for a in arms}
    for _ in range(args.reps):
        for arm in arms:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(arm)
            torch.cuda.synchronize()
            times[arm].append(time.perf_counter() - t0)
    b.close()
    name, limit = card()
    n = len(pages)
    result = {"metric": "pages_per_s", "pages": n, "sizes": SIZES, "reps": args.reps, "gpu": name,
              "power_limit": limit, "words": int(sum(len(r) for r in ref))}
    for arm in arms:
        t = np.asarray(times[arm])
        result[arm] = {"pages_per_s_median": round(n / float(np.median(t)), 2),
                       "pages_per_s_min": round(n / float(t.max()), 2), "pages_per_s_max": round(n / float(t.min()), 2)}
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
