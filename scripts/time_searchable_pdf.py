"""Times the searchable PDF's page images on one GPU and prints one JSON object.  Cases: 16 seeded synthetic pages of
2480 x 3508 (A4 at 300 dpi) and of 1200 x 1600, each preset (high / middle / low).  Per case:

  * device_pages_ms: create_searchable_pdf from a DevicePages (the pages already in HBM, as after analyze_pages): the
    LANCZOS resize kernels, the batched nvJPEG encode, the JPEG download and the PDF write (empty text layer), host
    clock around the whole call (it ends with the JPEG bytes on the host);
  * numpy_pages_ms: the same from numpy pages (adds their upload);
  * host_pillow_ms: the reference's host approach per page: BGR -> RGB, Pillow LANCZOS resize when the preset shrinks
    the page, Pillow JPEG save at the preset's quality (no PDF write);
  * medians of three runs, the three paths alternated, after one warm-up of each; bytes per page of both encoders.
The card's name and power limit are read in the same run.  The PDFs go to a temporary directory.

Usage: python scripts/time_searchable_pdf.py [--runs 3] [--out FILE]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import cv2
import numpy as np
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from yomitoku_b200 import create_searchable_pdf, device_pages  # noqa: E402
from yomitoku_b200.schemas import DocumentAnalyzerSchema  # noqa: E402
from yomitoku_b200.searchable_pdf import PRESETS, target_size  # noqa: E402
from yomitoku_b200.synth import synthetic_page  # noqa: E402

N_PAGES = 16
SHAPES = {"a4_300dpi": (3508, 2480), "1200x1600": (1600, 1200)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def pages_of(H, W):
    return [np.ascontiguousarray(cv2.resize(synthetic_page(500 + k)[0], (W, H), interpolation=cv2.INTER_LINEAR))
            for k in range(N_PAGES)]


def host_pillow(pages, quality):
    mls, q = PRESETS[quality]
    sizes = []
    for p in pages:
        img = Image.fromarray(np.ascontiguousarray(p[:, :, ::-1]))
        w, h = img.size
        if mls is not None and max(w, h) > mls:
            s = mls / max(w, h)
            img = img.resize((int(w * s), int(h * s)), Image.LANCZOS)
        buf = io.BytesIO()
        img.save(buf, format="JPEG", quality=q)
        sizes.append(buf.tell())
    return sizes


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    out = {"card": card(), "pages_per_call": N_PAGES, "runs": a.runs, "cases": []}
    docs = [DocumentAnalyzerSchema() for _ in range(N_PAGES)]
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "out.pdf")
        for name, (H, W) in SHAPES.items():
            pages = pages_of(H, W)
            dp = device_pages([torch.from_numpy(p).cuda() for p in pages])
            torch.cuda.synchronize()
            for quality in PRESETS:
                paths = {
                    "device_pages_ms": lambda: create_searchable_pdf(dp, docs, path, image_quality=quality),
                    "numpy_pages_ms": lambda: create_searchable_pdf(pages, docs, path, image_quality=quality),
                    "host_pillow_ms": lambda: host_pillow(pages, quality),
                }
                times = {k: [] for k in paths}
                for k, fn in paths.items():  # warm-up
                    fn()
                pil_bytes = None
                for _ in range(a.runs):
                    for k, fn in paths.items():
                        ms, r = timed(fn)
                        times[k].append(ms)
                        if k == "host_pillow_ms":
                            pil_bytes = r
                create_searchable_pdf(dp, docs, path, image_quality=quality)
                pdf_bytes = os.path.getsize(path)
                case = {"pages": name, "quality": quality, "image": "%dx%d" % target_size(W, H, quality)}
                for k, v in times.items():
                    case[k] = round(float(np.median(v)), 2)
                    case[k.replace("_ms", "_ms_per_page")] = round(float(np.median(v)) / N_PAGES, 3)
                case["pdf_bytes_per_page"] = pdf_bytes // N_PAGES
                case["pillow_jpeg_bytes_per_page"] = int(np.mean(pil_bytes))
                out["cases"].append(case)
                print(json.dumps(case), flush=True)
            del dp
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
