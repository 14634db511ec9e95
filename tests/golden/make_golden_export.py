"""Generates tests/golden/export_ref.json from the reference's OWN exporters, executed by path from the reference
checkout oracle.refcheck points at (the tests do not need it): export/export_{markdown,html,csv,json}.py,
schemas/document_analyzer.py (the result types the exporters read) and data/functions.py (load_image).

Stand-ins:
  * utils.misc.save_image records each figure write (path, crop shape, sha256 of the crop's pixels) instead of
    writing; the figure file is cv2.imencode(".jpg", crop) of that crop, which the test recomputes;
  * lxml: identity `html.fromstring` / `etree.tostring`, so that the golden HTML is the reference's element string
    before lxml re-indents it;
  * the modules the loaded files import but these paths never execute (base, utils.logger, pypdfium2) are stubs.

Cases are synthetic DocumentAnalyzerSchema results (Markdown specials, <, &, URLs, multi-line text, headings, page
headers / footers, tables with spans / empty cells / None contents, figures with and without paragraphs); each runs
under every combination of ignore_line_break, export_figure, export_figure_letter, figure_width and figure_dir that
the format takes, plus a few runs in other encodings and one export_figure run without an image.  The golden keeps
those axes and, per run, the sha256 prefix of the file's bytes (or the exception the reference raised) and the figure
writes.  load_image runs on a small PNG and a 3-frame TIFF written from seeded arrays, a page under 32 px, a PDF and
an unsupported suffix.
Usage: python tests/golden/make_golden_export.py
"""
import hashlib
import importlib.machinery
import itertools
import json
import logging
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import refcheck as rc  # noqa: E402


# ------------------------------------------------------------------------------------------------ synthetic cases
def _para(box, contents, order, role=None, direction="horizontal"):
    return {"box": box, "contents": contents, "direction": direction, "order": order, "role": role}


def _word(box, content):
    x1, y1, x2, y2 = box
    return {"points": [[x1, y1], [x2, y1], [x2, y2], [x1, y2]], "content": content, "direction": "horizontal",
            "rec_score": 0.875, "det_score": 0.5}


def _table(box, n_row, n_col, cells, order):
    """cells: (row, col, row_span, col_span, contents), 1-based like the table recogniser's."""
    x1, y1, x2, y2 = box
    return {"box": box, "n_row": n_row, "n_col": n_col,
            "rows": [{"box": [x1, y1 + 10 * r, x2, y1 + 10 * r + 10], "score": 0.9} for r in range(n_row)],
            "cols": [{"box": [x1 + 10 * c, y1, x1 + 10 * c + 10, y2], "score": 0.9} for c in range(n_col)],
            "spans": [],
            "cells": [{"row": r, "col": c, "row_span": rs, "col_span": cs, "contents": t,
                       "box": [x1 + 10 * c, y1 + 10 * r, x1 + 10 * (c + cs), y1 + 10 * (r + rs)]}
                      for r, c, rs, cs, t in cells],
            "order": order}


def _figure(box, order, paragraphs, direction="horizontal"):
    return {"box": box, "order": order, "paragraphs": paragraphs, "direction": direction}


CASES = {
    "text": {
        "paragraphs": [
            _para([10, 5, 290, 15], "Page header #1", 0, "page_header"),
            _para([10, 20, 290, 40], "1. Introduction", 1, "section_headings"),
            _para([10, 45, 290, 80], "a*b_c `code` [link](x) {x} #tag +1 !bang ~tilde| pipe - dash\nsecond line", 2),
            _para([10, 85, 290, 100], "x < y & z > w \"quoted\" 'single'", 3),
            _para([10, 105, 290, 120], "see https://example.com/a?b=1&c=2 and http://&amp; or https://<x>", 4),
            _para([10, 125, 290, 140], "日本語の段落\n改行あり ① 😀", 5, direction="vertical"),
            _para([10, 185, 290, 195], "footer - 3", 6, "page_footer"),
        ],
        "tables": [], "figures": [],
        "words": [_word([10, 20, 100, 40], "Introduction"), _word([10, 125, 60, 140], "日本語")],
    },
    "table": {
        "paragraphs": [_para([10, 150, 200, 170], "after the table", 2), _para([10, 2, 200, 12], "Title", 0,
                                                                               "section_headings")],
        "tables": [_table([5, 20, 295, 140], 4, 4, [
            (1, 1, 1, 2, "head | spans two"), (1, 3, 1, 1, "C"), (1, 4, 1, 1, "D&<E>"),
            (2, 1, 2, 1, "rows\n2-3"), (2, 2, 1, 1, ""), (2, 3, 1, 2, "x*y"),
            (3, 2, 1, 1, "line1\nline2"), (3, 3, 1, 1, "https://a.b/c?d&e"), (3, 4, 1, 1, ""),
            (4, 1, 1, 4, "bottom, with comma and \"quotes\""),
        ], 1)],
        "figures": [], "words": [],
    },
    "table_none": {
        "paragraphs": [_para([10, 150, 200, 170], "p", 1)],
        "tables": [_table([5, 20, 295, 140], 2, 2, [(1, 1, 1, 1, "a"), (1, 2, 1, 1, None), (2, 1, 1, 2, "b\nc")], 0)],
        "figures": [], "words": [],
    },
    "figures": {
        "paragraphs": [_para([10, 2, 200, 12], "before", 0), _para([10, 150, 200, 170], "between\nfigures", 2),
                       _para([10, 180, 200, 195], "last", 5)],
        "tables": [_table([5, 120, 100, 140], 1, 2, [(1, 1, 1, 1, "t1"), (1, 2, 1, 1, "t2")], 4)],
        "figures": [
            _figure([10, 20, 110, 90], 1, [_para([20, 30, 100, 40], "fig *b* 2", 2), _para([20, 50, 100, 60],
                                                                                          "fig a\n1", 1)]),
            _figure([150, 100, 320, 210], 3, []),             # reaches past the page's right and bottom edges
        ],
        "words": [_word([20, 30, 100, 40], "fig")],
    },
    "empty": {"paragraphs": [], "tables": [], "figures": [], "words": []},
}
IMAGE = {"seed": 7, "shape": [200, 300, 3]}      # the page the figures are cut from


def page_image():
    return np.random.default_rng(IMAGE["seed"]).integers(0, 256, IMAGE["shape"], dtype=np.uint8)


AXES = {
    "options": {   # the options each exporter takes besides ignore_line_break / encoding / img
        "md": ["export_figure", "export_figure_letter", "figure_width", "figure_dir"],
        "html": ["export_figure", "export_figure_letter", "figure_width", "figure_dir"],
        "csv": ["export_figure", "export_figure_letter", "figure_dir"],
        "json": ["export_figure", "figure_dir"],
    },
    "values": {"ignore_line_break": [False, True], "export_figure": [False, True],
               "export_figure_letter": [False, True], "figure_width": [200, 512], "figure_dir": ["figures", "img/fig"]},
    "encoding_runs": [["text", "shift-jis"], ["text", "cp932"], ["text", "utf-8-sig"], ["text", "euc-jp"]],
}


def expand_runs(g):
    """(case, format, kwargs, with image) of every run, in the order of the golden's results; tests/test_export_host.py
    expands the golden's axes the same way."""
    out = []
    for case, (fmt, names) in itertools.product(g["cases"], g["options"].items()):
        names = ["ignore_line_break"] + names
        for values in itertools.product(*(g["values"][n] for n in names)):
            out.append((case, fmt, dict(zip(names, values), encoding="utf-8"), True))
    for (case, enc), fmt in itertools.product(g["encoding_runs"], g["options"]):
        out.append((case, fmt, {"encoding": enc, "export_figure": False}, False))
    for fmt in g["options"]:      # export_figure without an image
        out.append(("figures", fmt, {"export_figure": True, "encoding": "utf-8"}, False))
    return out


def sha16(data):
    return hashlib.sha256(data).hexdigest()[:16]


# ------------------------------------------------------------------------------------------------ the reference
def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, None)
    m.__path__ = []
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


SAVED = []


def _record_save_image(img, path):
    crop = np.ascontiguousarray(img)
    SAVED.append((path, list(crop.shape), sha16(crop.tobytes())))


def load_reference():
    from pydantic import BaseModel, ConfigDict
    rc._pkg("ytk_ref")
    rc._pkg("ytk_ref.utils")

    class BaseSchema(BaseModel):                     # reference base.py:51-57 without its omegaconf-based module
        model_config = ConfigDict(extra="forbid", validate_assignment=True)

    _stub("ytk_ref.base", BaseSchema=BaseSchema)
    _stub("ytk_ref.utils.misc", save_image=_record_save_image)
    _stub("ytk_ref.utils.logger", set_logger=lambda name, level="INFO": logging.getLogger(name))
    _stub("pypdfium2")
    identity = types.SimpleNamespace(fromstring=lambda s: s, tostring=lambda s, **kw: s)
    _stub("lxml", etree=identity, html=identity)
    _stub("lxml.etree", fromstring=identity.fromstring, tostring=identity.tostring)
    _stub("lxml.html", fromstring=identity.fromstring, tostring=identity.tostring)
    exp = rc._pkg("ytk_ref.export")
    mods = {}
    for fmt, name in (("md", "export_markdown"), ("html", "export_html"), ("csv", "export_csv"),
                      ("json", "export_json")):
        mods[fmt] = rc._load("ytk_ref.export." + name, "export/%s.py" % name, "ytk_ref.export")
        setattr(exp, name, getattr(mods[fmt], name))
    rc._pkg("ytk_ref.schemas")
    da = rc._load("ytk_ref.schemas.document_analyzer", "schemas/document_analyzer.py", "ytk_ref.schemas")
    _stub("yomitoku")                                # export_json.convert_json imports the result type from here
    _stub("yomitoku.document_analyzer", DocumentAnalyzerSchema=da.DocumentAnalyzerSchema)
    rc._load("ytk_ref.constants", "constants.py", "ytk_ref")
    rc._pkg("ytk_ref.data")
    fn = rc._load("ytk_ref.data.functions", "data/functions.py", "ytk_ref.data")
    return mods, da.DocumentAnalyzerSchema, fn.load_image


def run_export(mods, schema_cls, run, tmp):
    """The run's result ("!<exception name>" or the sha256 prefix of the file's bytes) and its figure writes."""
    case, fmt, kwargs, with_img = run
    inputs = schema_cls.model_validate(CASES[case])
    out_path = os.path.join(tmp, "out", "doc_p1.%s" % fmt)
    os.makedirs(os.path.dirname(out_path), exist_ok=True)
    if os.path.exists(out_path):
        os.remove(out_path)
    fn = getattr(mods[fmt], {"md": "export_markdown", "html": "export_html", "csv": "export_csv",
                             "json": "export_json"}[fmt])
    SAVED.clear()
    try:
        fn(inputs, out_path, img=page_image() if with_img else None, **kwargs)
    except Exception as e:          # the reference's own failure on this input (e.g. None contents in Markdown)
        assert not os.path.exists(out_path)
        return "!" + type(e).__name__, []
    with open(out_path, "rb") as f:
        return sha16(f.read()), [[os.path.relpath(p, tmp), shape, h] for p, shape, h in SAVED]


def _page_record(p):
    p = np.ascontiguousarray(p)
    return [list(p.shape), str(p.dtype), sha16(p.tobytes())]


LOAD_FILES = {   # name -> list of (mode, h, w, seed) frames
    "page.png": [("RGBA", 40, 50, 1)],
    "scan.tiff": [("RGB", 40, 60, 2), ("L", 50, 35, 3), ("RGB", 33, 90, 4)],
    "tiny.png": [("RGB", 20, 40, 5)],
}


def write_load_files(tmp):
    """The load_image inputs, written from seeded arrays (the test writes the same files)."""
    from PIL import Image
    for name, frames in LOAD_FILES.items():
        imgs = []
        for mode, h, w, seed in frames:
            c = {"RGBA": 4, "RGB": 3, "L": 1}[mode]
            a = np.random.default_rng(seed).integers(0, 256, (h, w, c), dtype=np.uint8)
            imgs.append(Image.fromarray(a[:, :, 0] if c == 1 else a, mode))
        imgs[0].save(os.path.join(tmp, name), save_all=len(imgs) > 1, append_images=imgs[1:])
    with open(os.path.join(tmp, "doc.pdf"), "wb") as f:
        f.write(b"%PDF-1.4\n%%EOF\n")
    with open(os.path.join(tmp, "anim.gif"), "wb") as f:
        f.write(b"GIF89a")


def main():
    mods, schema_cls, load_image = load_reference()
    golden = dict(cases=CASES, image=IMAGE, **AXES)
    with tempfile.TemporaryDirectory() as tmp:
        results = [run_export(mods, schema_cls, r, tmp) for r in expand_runs(golden)]
        write_load_files(tmp)
        loads = {}
        for name in list(LOAD_FILES) + ["doc.pdf", "anim.gif"]:
            try:
                loads[name] = {"pages": [_page_record(p) for p in load_image(os.path.join(tmp, name))]}
            except Exception as e:
                loads[name] = {"error": type(e).__name__, "message": str(e)}
    golden.update(results=[r for r, _ in results], figures={str(i): f for i, (_, f) in enumerate(results) if f},
                  load_files=LOAD_FILES, load_image=loads)
    with open(os.path.join(HERE, "export_ref.json"), "w", encoding="utf-8") as f:     # one line per key
        f.write("{\n%s\n}\n" % ",\n".join("%s: %s" % (json.dumps(k), json.dumps(v, ensure_ascii=False))
                                         for k, v in golden.items()))
    n_err = sum(r.startswith("!") for r, _ in results)
    print("wrote export_ref.json: %d runs (%d raise in the reference), %d figure writes"
          % (len(results), n_err, sum(len(f) for _, f in results)))


if __name__ == "__main__":
    main()
