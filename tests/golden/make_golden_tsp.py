"""Generates tests/golden/tsp_ref.json from the reference's OWN files, executed from /root/reference by path (build
container only): table_semantic_parser.py (TableSemanticParser.__call__ and everything it calls after the models),
grid_parser.py, kv_parser.py, schemas/table_semantic_parser.py, schemas/document_analyzer.py, reading_order.py,
utils/misc.py, utils/graph.py and utils/union_find.py.  The four models are stand-ins that return the seeded synthetic
outputs of each case (text detector / recognizer: the words; layout parser: tables and paragraphs; cell detector:
cells, kv_item and grid regions); the modules the flow imports but never executes (base, export, visualizers, model
wrappers, ocr) are stubs.

Each case stores its inputs and the reference's `model_dump()`.  The reference orders key-value items whose values
share a top edge by the iteration order of a Python set of cell ids, which follows the per-process string hash; the
generator runs the reference under three hash seeds and requires the outputs to agree after
oracle.table_semantic.canonical_kv (that order, and the kv ids that follow it, normalised).
Usage: python tests/golden/make_golden_tsp.py
"""
import importlib.machinery
import json
import logging
import os
import subprocess
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import refcheck as rc  # noqa: E402
from oracle.table_semantic import canonical_kv  # noqa: E402


# ------------------------------------------------------------------------------------------------ synthetic cases
def _word(rng, x1, y1, x2, y2, vertical=False):
    text = "".join(rng.choice(list("abcdefghijklmnopqrstuvwxyz0123456789"), int(rng.integers(1, 6))))
    return {"points": [[x1, y1], [x2, y1], [x2, y2], [x1, y2]], "content": text,
            "direction": "vertical" if vertical else "horizontal", "rec_score": 0.9, "det_score": 0.8}


def _words_in(rng, box, n):
    x1, y1, x2, y2 = box
    out = []
    for _ in range(n):
        w, h = int(rng.integers(8, max(9, (x2 - x1) // 2))), int(rng.integers(6, max(7, (y2 - y1) // 2)))
        x = int(rng.integers(x1 + 1, max(x1 + 2, x2 - w)))
        y = int(rng.integers(y1 + 1, max(y1 + 2, y2 - h)))
        out.append(_word(rng, x, y, x + w, y + h, vertical=h > 2 * w))
    return out


def _grid_cells(rng, x0, y0, n_rows, n_cols, cw, ch, header_rows=1, span=True, jitter=2):
    """A grid of cells with `header_rows` header rows; a header spanning two columns and a cell spanning two rows."""
    cells, skip = [], set()
    if span and n_cols >= 3 and n_rows >= header_rows + 2:
        cells.append(("header", (x0, y0, x0 + 2 * cw, y0 + ch)))
        skip |= {(0, 0), (0, 1)}
        cells.append(("cell", (x0 + cw, y0 + (header_rows) * ch, x0 + 2 * cw, y0 + (header_rows + 2) * ch)))
        skip |= {(header_rows, 1), (header_rows + 1, 1)}
    for r in range(n_rows):
        for c in range(n_cols):
            if (r, c) in skip:
                continue
            j = rng.integers(-jitter, jitter + 1, 4) if jitter else np.zeros(4, int)
            box = (x0 + c * cw + j[0], y0 + r * ch + j[1], x0 + (c + 1) * cw + j[2], y0 + (r + 1) * ch + j[3])
            role = "header" if r < header_rows else ("empty" if rng.random() < 0.12 else "cell")
            cells.append((role, tuple(int(v) for v in box)))
    return cells


def _kv_cells(rng, x0, y0, n_rows, kw, vw, ch, vertical=False):
    """Key-value rows: a header key left of a value (or above it when vertical)."""
    cells = []
    for r in range(n_rows):
        if vertical:
            cells.append(("header", (x0 + r * vw, y0, x0 + (r + 1) * vw, y0 + ch)))
            cells.append(("cell", (x0 + r * vw, y0 + ch, x0 + (r + 1) * vw, y0 + 2 * ch)))
        else:
            cells.append(("header", (x0, y0 + r * ch, x0 + kw, y0 + (r + 1) * ch)))
            cells.append(("cell" if rng.random() > 0.15 else "empty", (x0 + kw, y0 + r * ch, x0 + kw + vw,
                                                                        y0 + (r + 1) * ch)))
    return cells


def _table(cells, box, kv_regions=(), grid_regions=()):
    return {"box": [int(v) for v in box], "role": None,
            "cells": [{"id": "c%d" % i, "box": [int(v) for v in b], "role": r} for i, (r, b) in enumerate(cells)],
            "kv_regions": [{"box": [int(v) for v in b], "score": float(s)} for b, s in kv_regions],
            "grid_regions": [{"box": [int(v) for v in b], "score": float(s)} for b, s in grid_regions]}


def _hull(cells, pad=2):
    bs = [b for _, b in cells]
    return (min(b[0] for b in bs) - pad, min(b[1] for b in bs) - pad, max(b[2] for b in bs) + pad,
            max(b[3] for b in bs) + pad)


def make_case(seed, kind):
    rng = np.random.default_rng(seed)
    tables, paragraphs, words = [], [], []
    if kind in ("grid", "mixed", "overlap", "ties"):
        g = _grid_cells(rng, 60, 80, int(rng.integers(4, 7)), int(rng.integers(3, 6)), 110, 40,
                        header_rows=1 + int(kind == "grid"), jitter=0 if kind == "ties" else 2)
        cells, regions = list(g), [(_hull(g), 0.9)]
        kv_regions = []
        if kind in ("mixed", "overlap"):
            k = _kv_cells(rng, 60, _hull(g)[3] + 20, 4, 120, 220, 36)
            cells += k
            kv_regions.append((_hull(k), 0.8))
        if kind == "overlap":
            kv_regions.append((_hull(g[:len(g) // 2 + 2]), 0.7))      # a kv region over half the grid
            regions.append((_hull(g, pad=6), 0.6))                    # the grid predicted twice
        tables.append(_table(cells, _hull(cells, 8), kv_regions, regions))
    if kind in ("kv", "mixed", "empty_small"):
        y0 = 700 if kind == "mixed" else 60
        k = _kv_cells(rng, 80, y0, int(rng.integers(3, 6)), 140, 260, 38)
        v = _kv_cells(rng, 560, y0, 3, 0, 120, 36, vertical=True)
        orphan = [("header", (80, y0 - 40, 480, y0)), ("cell", (80 + 400, y0 + 10, 540, y0 + 48))]
        cells = k + v + orphan
        tables.append(_table(cells, _hull(cells, 8), [(_hull(k), 0.9), (_hull(v), 0.85)], []))
    if kind == "empty_small":
        tables.append(_table([("cell", (900, 900, 1000, 940))], (890, 890, 1010, 950)))           # one cell: paragraph
        tables.append(_table([("empty", (700, 1000, 800, 1040)), ("empty", (800, 1000, 900, 1040)),
                              ("group", (700, 990, 900, 1050)), ("cell", (700, 1040, 800, 1080)),
                              ("cell", (800, 1040, 900, 1080))],
                             (690, 980, 910, 1090), [], [((690, 980, 910, 1090), 0.9)]))
    for t in tables:
        for c in t["cells"]:
            if c["role"] != "group" and rng.random() < 0.85:
                words += _words_in(rng, c["box"], int(rng.integers(1, 4)))
        # a word straddling two cells
        if len(t["cells"]) > 1:
            a, b = t["cells"][0]["box"], t["cells"][1]["box"]
            words.append(_word(rng, a[0] + 3, a[1] + 3, b[2] - 3, min(a[3], b[3]) - 3))
    if kind == "ties" and tables:
        cs = [c for c in tables[0]["cells"] if c["role"] != "header"]
        for a, b in zip(cs, cs[1:]):
            if a["box"][1] == b["box"][1] and a["box"][3] == b["box"][3] and a["box"][2] == b["box"][0]:
                x = a["box"][2]
                words.append(_word(rng, x - 10, a["box"][1] + 5, x + 10, a["box"][1] + 15))   # half in each
    for i in range(int(rng.integers(2, 5))):
        box = [1100 + 10 * i, 100 + 150 * i, 1400, 100 + 150 * i + 80]
        paragraphs.append({"box": box, "role": "section_headings" if i == 0 else None, "score": 0.9})
        words += _words_in(rng, box, int(rng.integers(1, 4)))
    words.append(_word(rng, 1500, 1500, 1540, 1520))                                         # outside everything
    order = rng.permutation(len(words))
    return {"tables": tables, "paragraphs": paragraphs, "words": [words[i] for i in order]}


CASES = [  # (seed, kind, grid_only, kv_only)
    (400, "grid", False, False), (401, "grid", False, False), (402, "kv", False, False), (403, "kv", False, False),
    (404, "mixed", False, False), (405, "mixed", True, False), (406, "mixed", False, True),
    (407, "overlap", False, False), (408, "overlap", False, False), (409, "empty_small", False, False),
    (410, "ties", False, False), (411, "ties", False, False),
]


# ------------------------------------------------------------------------------------------------ the reference
def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, None)
    m.__path__ = []
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


def load_reference_tsp():
    from pydantic import BaseModel, ConfigDict
    rc._pkg("ytk_ref")
    rc._pkg("ytk_ref.utils")

    class BaseSchema(BaseModel):                     # reference base.py:51-57 without its omegaconf-based module
        model_config = ConfigDict(extra="forbid", validate_assignment=True)

    _stub("ytk_ref.base", BaseSchema=BaseSchema)
    _stub("ytk_ref.export", export_csv=None, export_html=None, export_markdown=None, export_json=None)
    _stub("ytk_ref.utils.logger", set_logger=lambda name, level="INFO": logging.getLogger(name))
    _stub("ytk_ref.utils.visualizer", cell_detector_visualizer=None)
    rc._load("ytk_ref.utils.misc", "utils/misc.py", "ytk_ref.utils")
    rc._load("ytk_ref.utils.graph", "utils/graph.py", "ytk_ref.utils")
    rc._load("ytk_ref.utils.union_find", "utils/union_find.py", "ytk_ref.utils")
    schemas = rc._pkg("ytk_ref.schemas")
    da = rc._load("ytk_ref.schemas.document_analyzer", "schemas/document_analyzer.py", "ytk_ref.schemas")
    for k in dir(da):
        if k.endswith("Schema") or k in ("Element", "WordPrediction"):
            setattr(schemas, k, getattr(da, k))
    rc._load("ytk_ref.reading_order", "reading_order.py", "ytk_ref")
    rc._load("ytk_ref.schemas.table_semantic_parser", "schemas/table_semantic_parser.py", "ytk_ref.schemas")
    _stub("ytk_ref.ocr", OCRSchema=da.OCRSchema, ocr_aggregate=lambda det, rec: det.words)
    for mod, cls in (("layout_parser", "LayoutParser"), ("table_cell_detector", "CellDetector"),
                     ("text_detector", "TextDetector"), ("text_recognizer", "TextRecognizer")):
        _stub("ytk_ref." + mod, **{cls: None})
    rc._load("ytk_ref.grid_parser", "grid_parser.py", "ytk_ref")
    rc._load("ytk_ref.kv_parser", "kv_parser.py", "ytk_ref")
    return rc._load("ytk_ref.table_semantic_parser", "table_semantic_parser.py", "ytk_ref")


def reference_parse(mod, case, grid_only, kv_only):
    da = sys.modules["ytk_ref.schemas.document_analyzer"]
    ts = sys.modules["ytk_ref.schemas.table_semantic_parser"]

    class Det:
        words = case["words"]
        points = [w["points"] for w in case["words"]]

    tables = [da.Element(id=None, box=t["box"], score=0.9, role=None, contents=None) for t in case["tables"]]
    layout = da.LayoutParserSchema(paragraphs=[da.Element(id=None, contents=None, **p) for p in case["paragraphs"]],
                                   tables=tables, figures=[])

    def cells_of(img, bordered):
        assert len(bordered) == len(case["tables"])
        return [ts.TableDetectorSchema(
            id=None, box=t["box"], role=t["role"],
            cells=[ts.CellSchema(id=c["id"], box=c["box"], role=c["role"], contents=None, row=None, col=None,
                                 row_span=None, col_span=None) for c in t["cells"]],
            kv_regions=[ts.RegionSchema(id=None, role="kv_item", **r) for r in t["kv_regions"]],
            grid_regions=[ts.RegionSchema(id=None, role="grid", **r) for r in t["grid_regions"]]) for t in case["tables"]]

    p = object.__new__(mod.TableSemanticParser)
    p.text_detector = lambda img: (Det, None)
    p.layout_parser = lambda img: (layout, None)
    p.cell_detector = cells_of
    p.text_recognizer = lambda img, points: (None, None)
    p.visualize, p.merge_same_column_values = False, False
    res, _, _ = p(np.zeros((4, 4, 3), np.uint8), grid_only=grid_only, kv_only=kv_only)
    return res.model_dump()


def child():
    mod = load_reference_tsp()
    out = []
    for seed, kind, grid_only, kv_only in CASES:
        case = make_case(seed, kind)
        out.append({"seed": seed, "kind": kind, "grid_only": grid_only, "kv_only": kv_only, "input": case,
                    "output": reference_parse(mod, case, grid_only, kv_only)})
    json.dump(out, sys.stdout)


def main():
    runs = []
    for hs in ("0", "1", "2"):
        env = dict(os.environ, PYTHONHASHSEED=hs, YTK_TSP_CHILD="1")
        r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=env, capture_output=True, text=True)
        if r.returncode:
            raise SystemExit(r.stderr)
        runs.append(json.loads(r.stdout))
    for case_runs in zip(*runs):
        canon = [json.dumps(canonical_kv(c["output"]), sort_keys=True) for c in case_runs]
        assert len(set(canon)) == 1, "case %d depends on the string hash beyond the kv order" % case_runs[0]["seed"]
    with open(os.path.join(HERE, "tsp_ref.json"), "w") as f:
        json.dump({"cases": runs[0]}, f)
    n_kv = sum(len(t["kv_items"]) for c in runs[0] for t in c["output"]["tables"])
    n_grid = sum(len(t["grids"]) for c in runs[0] for t in c["output"]["tables"])
    print("wrote tsp_ref.json: %d cases, %d kv items, %d grids" % (len(runs[0]), n_kv, n_grid))


if __name__ == "__main__":
    child() if os.environ.get("YTK_TSP_CHILD") == "1" else main()
