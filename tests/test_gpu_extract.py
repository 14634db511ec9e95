"""Fields out of forms on the GPU: `TableSemanticParser.extract_pages` on a batch of pages of mixed sizes, on the host
and on the device, against `extract(parser(page)[0], schema)` page by page, and the command line
(`python -m yomitoku_b200.extract`) over a directory of PNGs against the same.  The parser has seeded weights, the
detector's trained head, fixed tables in place of the layout model's, and the cell detector's post-processing replaced
by a known layout per table (a grid with a header row above key-value rows), so that the grid and key-value parsers
and every kind of field have something to find."""
import importlib
import json
import os

import cv2
import numpy as np
import pytest
import torch

from test_gpu_table_semantic import _pages, _parser
from yomitoku_b200 import extract
from yomitoku_b200.data import load_image
from yomitoku_b200.schemas import CellSchema, RegionSchema

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TABLES = [[40, 60, 700, 420], [100, 480, 760, 760]]
CW, CH, GRID_ROWS, GRID_COLS, KV_ROWS = 120, 30, 4, 3, 3


def _cell(role, x1, y1, x2, y2):
    return CellSchema(id=None, role=role, contents=None, row=None, col=None, row_span=None, col_span=None,
                      box=[int(x1), int(y1), int(x2), int(y2)])


def form_layout(preds, data, table_box):
    """A grid of GRID_ROWS x GRID_COLS cells (row 0 headers) at the table's top left, KV_ROWS key | value rows below."""
    x0, y0 = table_box[0] + 5, table_box[1] + 5
    cells = [_cell("header" if r == 0 else "cell", x0 + c * CW, y0 + r * CH, x0 + (c + 1) * CW, y0 + (r + 1) * CH)
             for r in range(GRID_ROWS) for c in range(GRID_COLS)]
    grid = [x0 - 2, y0 - 2, x0 + GRID_COLS * CW + 2, y0 + GRID_ROWS * CH + 2]
    k0 = y0 + GRID_ROWS * CH + 20
    for r in range(KV_ROWS):
        cells.append(_cell("header", x0, k0 + r * CH, x0 + CW, k0 + (r + 1) * CH))
        cells.append(_cell("cell", x0 + CW, k0 + r * CH, x0 + 3 * CW, k0 + (r + 1) * CH))
    for i, c in enumerate(cells):
        c.id = "c%d" % i
    kv = [x0 - 2, k0 - 2, x0 + 3 * CW + 2, k0 + KV_ROWS * CH + 2]
    return (cells, [RegionSchema(id=None, box=kv, role="kv_item", score=0.8)],
            [RegionSchema(id=None, box=grid, role="grid", score=0.9)])


X0, Y0 = TABLES[0][0] + 5, TABLES[0][1] + 5
SCHEMA = {"fields": [
    {"name": "first_header", "cell_id": "r0c0"},
    {"name": "by_bbox", "bbox": [X0 + CW, Y0 + CH, X0 + 2 * CW, Y0 + 2 * CH]},
    {"name": "any_text", "regex": r"\S{2,}", "normalize": "alphanumeric"},
    {"name": "missing", "description": "存在しない項目"},
    {"name": "grid", "structure": "table",
     "columns": [{"name": "first", "cell_id": "r0c0"}, {"name": "second", "bbox": [X0 + CW, Y0, X0 + 2 * CW, Y0 + CH]},
                 {"name": "third", "cell_id": "r0c2", "normalize": "numeric"}]},
]}


def _layout_parser():
    p, forwards = _parser(TABLES)
    p.cell_detector.postprocess = form_layout
    return p, forwards


def _key_field(results):
    """A kv field whose description is the text of a key cell the parser found (skipped if the model read none)."""
    for r in results:
        for t in r.tables:
            for kv in t.kv_items:
                text = "".join(t.cells[k].contents or "" for k in kv.key)
                if text.strip():
                    return {"name": "by_key", "description": text.strip()}
    return None


def test_extract_pages_equals_per_page_extract():
    p, forwards = _layout_parser()
    pages = _pages(700, [(1200, 900), (900, 1000), (800, 800), (1000, 1200)])
    try:
        per_page = [p(pg)[0] for pg in pages]
        assert all(len(r.tables) == 2 and all(t.grids and t.kv_items for t in r.tables) for r in per_page)
        schema = dict(SCHEMA, fields=SCHEMA["fields"] + [f for f in [_key_field(per_page)] if f])
        for simple in (False, True):
            want = [extract(r, schema, simple=simple) for r in per_page]
            del forwards[:]
            assert p.extract_pages(pages, schema, simple=simple) == want
            assert len(forwards) == 1
            assert p.extract_pages([torch.from_numpy(pg).to(DEV) for pg in pages], schema, simple=simple) == want
        want = [extract(r, schema, normalize=False) for r in per_page]
        assert p.extract_pages(pages, schema, normalize=False) == want
        fields = want[0]["fields"]
        assert fields["first_header"]["source"] == "cell_id" and fields["by_bbox"]["source"] == "bbox"
        assert fields["missing"]["source"] == "not_found"
        assert fields["grid"]["source"] == "grid" and len(fields["grid"]["records"]) == 2 * (GRID_ROWS - 1)
        assert any(w["fields"]["any_text"]["source"] == "regex" for w in want)
    finally:
        if p._batched is not None:
            p._batched.close()


def test_command_line_over_a_directory(tmp_path):
    cli = importlib.import_module("yomitoku_b200.extract")
    p, forwards = _layout_parser()
    pages = _pages(720, [(1100, 900), (800, 1000), (900, 900)])
    src = tmp_path / "forms"
    src.mkdir()
    for i, pg in enumerate(pages):
        cv2.imwrite(str(src / ("form%d.png" % i)), pg)
    schema_path = tmp_path / "schema.json.yaml"
    schema_path.write_text(json.dumps(SCHEMA, ensure_ascii=False), encoding="utf-8")      # JSON is YAML
    try:
        for simple in (False, True):
            out = tmp_path / ("out_simple" if simple else "out")
            argv = [str(src), "-s", str(schema_path), "-o", str(out), "--batch", "2"] + (["--simple"] if simple else [])
            del forwards[:]
            written = cli.run(cli.build_parser().parse_args(argv), p)
            assert len(forwards) == 2
            assert sorted(os.path.basename(w) for w in written) == ["form%d_p1_extract.json" % i for i in range(3)]
            for i in range(3):
                page = load_image(src / ("form%d.png" % i))[0]
                assert np.array_equal(page, pages[i])
                want = extract(p(page)[0], SCHEMA, simple=simple)
                text = (out / ("form%d_p1_extract.json" % i)).read_text(encoding="utf-8")
                assert text == json.dumps(want, ensure_ascii=False, indent=2)
    finally:
        if p._batched is not None:
            p._batched.close()
