"""Times schema extraction on one GPU and prints one JSON object:

  * TableSemanticParser.extract_pages and parse_pages in pages/s on the 16 synthetic form pages of
    scripts/time_table_semantic.py (mixed sizes, seeded weights, the detector's trained head, one fixed table per page,
    the cell detector's post-processing replaced by a 20 x 15 grid of 300 cells), alternated call by call, `--steps`
    timed calls of each after one warm-up, host clock around calls that end in a synchronise;
  * the host time of the extraction step alone (`extractor.extract` on the 16 parsed pages, `--reps` repetitions) next
    to the parse_pages call, for a form schema of key, cell, paragraph and regex fields and a three-column table;
  * the card's name and power limit, read in the same run.

Usage: python scripts/time_extract.py [--steps 3] [--reps 20] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

BOX = [40, 60, 835, 860]
ROWS, COLS = 20, 15
SCHEMA = {"fields": [
    {"name": "applicant", "description": "氏名", "normalize": "strip_spaces"},
    {"name": "phone", "description": "電話番号", "normalize": "phone_jp"},
    {"name": "postal", "description": "郵便番号", "normalize": "postal_code_jp"},
    {"name": "date", "description": "申込日", "normalize": "date_jp"},
    {"name": "first", "cell_id": "r1c0"},
    {"name": "boxed", "bbox": [BOX[0] + 60, BOX[1] + 50, BOX[0] + 100, BOX[1] + 70]},
    {"name": "number", "regex": r"\d{3,}", "normalize": "numeric"},
    {"name": "code", "regex": r"[A-Z]\d{6}"},
    {"name": "missing", "description": "存在しない項目", "regex": "ZZZ"},
    {"name": "items", "structure": "table",
     "columns": [{"name": "a", "cell_id": "r0c0"}, {"name": "b", "description": "品名"},
                 {"name": "c", "bbox": [BOX[0] + 106, BOX[1], BOX[0] + 158, BOX[1] + 40], "normalize": "numeric"}]},
]}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def form_parser():
    from test_gpu_table_semantic import _parser
    from yomitoku_b200.schemas import CellSchema, RegionSchema
    p, _ = _parser(tables=[BOX])
    cw, ch = (BOX[2] - BOX[0]) // COLS, (BOX[3] - BOX[1]) // ROWS

    def form_cells(preds, data, table_box):
        cells = [CellSchema(id="c%d" % (r * COLS + c), role="header" if r == 0 else "cell", contents=None, row=None,
                            col=None, row_span=None, col_span=None,
                            box=[BOX[0] + c * cw, BOX[1] + r * ch, BOX[0] + (c + 1) * cw, BOX[1] + (r + 1) * ch])
                 for r in range(ROWS) for c in range(COLS)]
        return cells, [], [RegionSchema(id=None, box=list(BOX), role="grid", score=0.9)]
    p.cell_detector.postprocess = form_cells
    return p


def timed(fn, steps):
    t = []
    for _ in range(steps):
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    return r, t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_extract.py measures on a GPU; none is visible")
    from test_gpu_table_semantic import _pages
    from yomitoku_b200.extractor import ExtractionSchema, extract
    schema = ExtractionSchema.model_validate(SCHEMA)
    pages = _pages(600, [(1200, 900), (1000, 1000), (900, 1200), (1600, 1200)] * 4)
    p = form_parser()
    try:
        parsed = p.parse_pages(pages)
        want = [extract(r, schema) for r in parsed]
        same = p.extract_pages(pages, schema) == want
        torch.cuda.synchronize()
        t_parse, t_extract = [], []
        for _ in range(a.steps):                  # alternated, so both see the same host and card
            t_parse += timed(lambda: p.parse_pages(pages), 1)[1]
            t_extract += timed(lambda: p.extract_pages(pages, schema), 1)[1]
    finally:
        if p._batched is not None:
            p._batched.close()
    host = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        for r in parsed:
            extract(r, schema)
        host.append(time.perf_counter() - t0)
    parse_s, extract_s, host_s = float(np.median(t_parse)), float(np.median(t_extract)), float(np.median(host))
    found = sum(f["source"] != "not_found" for w in want for f in w["fields"].values())
    out = {"card": card(), "pages": len(pages), "cells": sum(len(t.cells) for r in parsed for t in r.tables),
           "words": sum(len(r.words) for r in parsed), "schema_fields": len(schema.fields),
           "fields_found": found, "extract_pages_equals_parse_then_extract": same,
           "parse_pages": {"median_s": parse_s, "pages_per_s": len(pages) / parse_s},
           "extract_pages": {"median_s": extract_s, "pages_per_s": len(pages) / extract_s},
           "extraction_step_host": {"median_ms_16_pages": 1e3 * host_s, "ms_per_page": 1e3 * host_s / len(pages),
                                    "share_of_parse_pages": host_s / parse_s}}
    line = json.dumps(out, ensure_ascii=False)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
