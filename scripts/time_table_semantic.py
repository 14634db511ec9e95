"""Times the table semantic parser on one GPU and prints one JSON object:

  * the word-to-element assignment of TableSemanticParser.aggregate on synthetic form pages of 300 words and 300
    cells (a 20 x 15 grid table, words inside the cells, some across two) plus 10 paragraphs per page, for 1 and 16
    pages: the reference's Python loop (oracle/table_semantic.py, host clock, `--reps` repetitions) against the CUDA
    kernel - the whole `models.assign_best_overlap` call (uploads, one launch, download; CUDA events) and the launch
    alone on resident buffers (CUDA events around `--launches` launches) - after a warm-up, with the results compared;
  * TableSemanticParser.parse_pages in pages/s on 16 synthetic pages of mixed sizes (seeded weights, the detector's
    trained head, one fixed table per page in place of the layout model's as in the GPU tests, the cell detector's
    post-processing replaced by a 300-cell grid; `--steps` timed calls after one warm-up, host clock around calls that
    end in a synchronise), with the host time of the word assignment and of the grid / key-value stage;
  * the card's name and power limit, read in the same run.

Usage: python scripts/time_table_semantic.py [--reps 5] [--launches 200] [--steps 3] [--out FILE]
"""
import argparse
import ctypes
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
from oracle import table_semantic as ots  # noqa: E402
from yomitoku_b200 import _lib  # noqa: E402
from yomitoku_b200.models import OVERLAP_GROUP_DTYPE, assign_best_overlap  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def form_page(seed, n_rows=20, n_cols=15):
    """(word boxes, cell boxes, paragraph boxes) of one synthetic form page."""
    rng = np.random.default_rng(seed)
    cw, ch, x0, y0 = 100, 40, 50, 100
    cells = [[x0 + c * cw, y0 + r * ch, x0 + (c + 1) * cw, y0 + (r + 1) * ch] for r in range(n_rows) for c in range(n_cols)]
    words = []
    for x1, y1, x2, y2 in cells:
        if rng.random() < 0.9:
            w = int(rng.integers(20, 80))
            x = x1 + int(rng.integers(2, cw - w))
            words.append([x, y1 + 8, x + w, y2 - 8])
        else:
            words.append([x2 - 30, y1 + 8, x2 + 30, y2 - 8])          # across two cells
    paras = [[1600, 100 + 80 * i, 2300, 160 + 80 * i] for i in range(10)]
    words += [[p[0] + 10, p[1] + 5, p[2] - 10, p[3] - 5] for p in paras]
    return np.array(words, np.float64), np.array(cells, np.float64), np.array(paras, np.float64)


def batch_inputs(n_pages):
    words, elems, groups = [], [], []
    for i in range(n_pages):
        w, c, p = form_page(i)
        w0, e0 = sum(len(x) for x in words), sum(len(x) for x in elems)
        words.append(w)
        elems += [c, p]
        groups += [(w0, w0 + len(w), e0, e0 + len(c)), (w0, w0 + len(w), e0 + len(c), e0 + len(c) + len(p))]
    elems = np.concatenate(elems)
    return np.concatenate(words), elems, np.zeros(len(elems), np.uint8), np.array(groups, np.int32)


def event_ms(fn, n, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def assignment(n_pages, reps, launches):
    words, elems, skip, groups = batch_inputs(n_pages)
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        want = ots.assign_best_overlap(words, elems, skip, groups)
        t.append((time.perf_counter() - t0) * 1e3)
    got = assign_best_overlap(words, elems, skip, groups, 0.2, "cuda")
    same = got[0].tolist() == want[0] and got[1].tolist() == want[1]
    call_ms = event_ms(lambda: assign_best_overlap(words, elems, skip, groups, 0.2, "cuda"), reps * 10, 3)
    # the launch alone on resident buffers
    boxes = torch.from_numpy(np.concatenate([words, elems])).cuda()
    skip_d = torch.from_numpy(skip).cuda()
    total = int((groups[:, 1] - groups[:, 0]).sum())
    best = torch.empty(total, dtype=torch.int32, device="cuda")
    ratio = torch.empty(total, dtype=torch.float64, device="cuda")
    g = np.ascontiguousarray(groups).view(OVERLAP_GROUP_DTYPE).reshape(-1)
    L = _lib.lib()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def launch():
        _lib.check(L.ytk_op_assign_best_overlap_f64(boxes.data_ptr(), len(words), boxes[len(words):].data_ptr(),
                                                    skip_d.data_ptr(), len(elems), g.ctypes.data, len(g), 0.2,
                                                    best.data_ptr(), ratio.data_ptr(), total, stream))
    launch_ms = event_ms(launch, launches, 10)
    return {"pages": n_pages, "words": len(words), "cells_and_paragraphs": len(elems), "groups": len(groups),
            "python_loop_ms": {"median": float(np.median(t)), "min": float(np.min(t))},
            "kernel_call_ms": call_ms, "kernel_launch_only_ms": launch_ms, "identical_to_python_loop": same}


def parse_pages_rate(steps):
    """parse_pages on 16 pages; the cell detector's forward runs, its post-processing is replaced by a 20 x 15 grid of
    cells in one grid region (random weights find no cells), so the host structure stage sees a form-sized table."""
    from test_gpu_table_semantic import _pages, _parser
    from yomitoku_b200 import table_semantic_parser as tsp
    from yomitoku_b200.schemas import CellSchema, RegionSchema
    box = [40, 60, 835, 860]
    p, _ = _parser(tables=[box])
    cw, ch = (box[2] - box[0]) // 15, (box[3] - box[1]) // 20

    def form_cells(preds, data, table_box):
        cells = [CellSchema(id="c%d" % (r * 15 + c), role="header" if r == 0 else "cell", contents=None, row=None,
                            col=None, row_span=None, col_span=None,
                            box=[box[0] + c * cw, box[1] + r * ch, box[0] + (c + 1) * cw, box[1] + (r + 1) * ch])
                 for r in range(20) for c in range(15)]
        return cells, [], [RegionSchema(id=None, box=list(box), role="grid", score=0.9)]
    p.cell_detector.postprocess = form_cells
    stage = {"aggregate_pages": [], "semantic_page": []}
    for name in stage:
        fn = getattr(tsp, name)

        def timed(*a, _fn=fn, _name=name, **k):
            t0 = time.perf_counter()
            r = _fn(*a, **k)
            stage[_name].append(time.perf_counter() - t0)
            return r
        setattr(tsp, name, timed)
    shapes = [(1200, 900), (1000, 1000), (900, 1200), (1600, 1200)] * 4
    pages = _pages(600, shapes)
    try:
        p.parse_pages(pages)
        torch.cuda.synchronize()
        t = []
        for v in stage.values():
            del v[:]
        for _ in range(steps):
            t0 = time.perf_counter()
            res = p.parse_pages(pages)
            torch.cuda.synchronize()
            t.append(time.perf_counter() - t0)
    finally:
        if p._batched is not None:
            p._batched.close()
    s = float(np.median(t))
    return {"pages": len(pages), "median_s": s, "pages_per_s": len(pages) / s,
            "words": sum(len(r.words) for r in res), "tables": sum(len(r.tables) for r in res),
            "cells": sum(len(t.cells) for r in res for t in r.tables),
            "host_ms_per_call": {"word_assignment": 1e3 * sum(stage["aggregate_pages"]) / steps,
                                 "grid_kv_structure": 1e3 * sum(stage["semantic_page"]) / steps}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_table_semantic.py measures on a GPU; none is visible")
    out = {"card": card(), "assignment": [assignment(n, a.reps, a.launches) for n in (1, 16)]}
    print(json.dumps(out), flush=True)           # the assignment figures stand even if the parser run fails
    out["parse_pages"] = parse_pages_rate(a.steps)
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
