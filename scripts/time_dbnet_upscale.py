"""Times text detection of small pages - pages the detector input (1280 on the short side, at most 1600 on the long one)
enlarges - on one GPU, and prints one JSON object.  For 16 synthetic pages of each of 900 x 1200 and 720 x 1280 (larger
synthetic pages shrunk with cv2 INTER_AREA, so that the detector input restores about the text size of the 1200 x 1600
pages the trained binarize head of tests/golden was fitted on; with it the maps hold the pages' text lines):

  * host_seam:  what TextDetector did with such pages before the device pre-processing took them - per page
                `preprocess` (cv2.resize INTER_AREA in fp32, float64 standardisation), one `model(x)` forward per
                chunk of 8 pages from the host fp32 tensor, the download of the maps and the OpenCV post-processing;
  * device:     TextDetector.detect_pages per chunk of 8 pages - the u8 pages go up, preprocess_kernel<AreaUpSampler>
                resizes them on the device, the post-processing front half runs there and only row runs come back;
  * batched:    BatchedOCR end to end (detection, host stage in the worker pool, recognition with a random-weight
                parseq-tiny-dynw-v4) on all 16 pages.

host_seam and device are alternated step by step in one run; every time is a host clock around work that ends in a
device synchronise, after warm-up, reported as the median per step and per page.  The card's name and power limit are
read in the same run.

Usage: python scripts/time_dbnet_upscale.py [--steps 5] [--warmup 2] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from trained_head import load_trained_head  # noqa: E402
from yomitoku_b200 import TextDetector, TextRecognizer  # noqa: E402
from yomitoku_b200.pipeline import BatchedOCR  # noqa: E402
from yomitoku_b200.synth import synthetic_page  # noqa: E402

N_PAGES, CHUNK = 16, 8
SIZES = {(900, 1200): (1200, 1600), (720, 1280): (900, 1600)}     # page -> the synthetic page it is shrunk from


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def host_seam(det, pages):
    out = []
    for s in range(0, len(pages), CHUNK):
        chunk = pages[s:s + CHUNK]
        x = torch.cat([det.preprocess(p) for p in chunk])
        with torch.inference_mode():
            prob = det.model(x)["binary"].cpu().numpy()
        out += [det.postprocess({"binary": prob[i:i + 1]}, p.shape[:2]) for i, p in enumerate(chunk)]
    return out


def device(det, pages):
    out = []
    for s in range(0, len(pages), CHUNK):
        out += [(r.points, r.scores) for r in det.detect_pages(pages[s:s + CHUNK])]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_dbnet_upscale: needs a GPU")
    det = TextDetector(from_pretrained=False, device="cuda")
    load_trained_head(det.model)
    rec = TextRecognizer(model_name="parseq-tiny-dynw-v4", from_pretrained=False, device="cuda")
    res = {"card": card(), "pages_per_size": N_PAGES, "detector_chunk": CHUNK, "cases": []}
    for hw, big in SIZES.items():
        pages = [cv2.resize(synthetic_page(200 + i, height=big[0], width=big[1])[0], (hw[1], hw[0]),
                            interpolation=cv2.INTER_AREA) for i in range(N_PAGES)]
        ms = {"host_seam": [], "device": [], "batched": []}
        for _ in range(a.warmup):
            host_seam(det, pages)
            device(det, pages)
        for _ in range(a.steps):
            t, ref = timed(lambda: host_seam(det, pages))
            ms["host_seam"].append(t)
            t, got = timed(lambda: device(det, pages))
            ms["device"].append(t)
        boxes = [len(q) for q, _ in got]
        same = sum(q == r[0] for (q, _), r in zip(got, ref))
        b = BatchedOCR(det, rec, det_batch=CHUNK)
        try:
            for _ in range(a.warmup):
                b(pages)
            for _ in range(a.steps):
                t, out = timed(lambda: b(pages))
                ms["batched"].append(t)
        finally:
            b.close()
        case = {"page": list(hw), "input": list(det.model.input_size(*hw)), "boxes_per_page": [min(boxes), max(boxes)],
                "pages_with_equal_quads_host_seam_vs_device": same, "words_per_page_batched": len(out[0].words)}
        for k, v in ms.items():
            case[k + "_ms_per_step"] = float(np.median(v))
            case[k + "_ms_per_page"] = float(np.median(v)) / N_PAGES
            case[k + "_steps_ms"] = [round(x, 2) for x in v]
        res["cases"].append(case)
    res["card_after"] = card()
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
