"""Generates tests/golden/pdf_ref.json from the reference's OWN create_searchable_pdf (utils/searchable_pdf.py, with
utils/misc.py for is_contained), executed by path from the reference checkout oracle.refcheck points at (the tests do
not need it).

Stand-ins: reportlab's canvas records, per word the reference draws, the strings of its drawString calls (one per
character of a vertical word, between saveState / rotate / restoreState) and whether it rotated; `_calc_font_size`
records the words the reference considers, in its order, with the text and box extents it is called with (a word whose
font size comes out 0 is skipped by the reference); stringWidth is len(text) * size / 2; jaconv.h2z is the identity, so
a vertical word's recorded text is the recognised text (the cases keep the characters the reference's extra full-width
table maps - space, U+00A5, U+00B7 - out of vertical words).

Cases are synthetic DocumentAnalyzerSchema pages given as plain attribute objects: horizontal and vertical paragraphs,
tables with their cells listed out of order, figure paragraphs, a word inside two containers, words inside none, float
quads, empty words, zero-height and zero-width words, characters outside the BMP, plus seeded random pages.
Usage: python tests/golden/make_golden_pdf.py
"""
import importlib.util
import json
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import refcheck as rc  # noqa: E402


def _quad(x1, y1, x2, y2):
    return [[x1, y1], [x2, y1], [x2, y2], [x1, y2]]


def _word(box, content, direction="horizontal"):
    return {"points": _quad(*box), "content": content, "direction": direction, "rec_score": 0.9, "det_score": 0.9}


def _para(box, order, direction="horizontal"):
    return {"box": box, "contents": None, "direction": direction, "order": order, "role": None}


def _table(order, cells):
    return {"box": [0, 0, 1, 1], "n_row": 1, "n_col": 1, "rows": [], "cols": [], "spans": [], "order": order,
            "cells": [{"row": r, "col": c, "row_span": 1, "col_span": 1, "box": box, "contents": None}
                      for r, c, box in cells]}


def _figure(order, paragraphs):
    return {"box": [0, 0, 1, 1], "order": order, "paragraphs": paragraphs, "direction": None}


def fixed_pages():
    page1 = {
        "paragraphs": [_para([50, 50, 400, 200], 0), _para([500, 50, 700, 600], 1, "vertical"),
                       _para([40, 700, 300, 760], 4)],
        "tables": [_table(2, [(1, 1, [300, 300, 400, 350]), (0, 0, [200, 250, 300, 300]), (1, 0, [200, 300, 300, 350]),
                              (0, 1, [300, 250, 400, 300])])],
        "figures": [_figure(3, [_para([60, 400, 180, 600], 5, "vertical"), _para([200, 420, 480, 480], 6)])],
        "words": [
            _word([220, 120, 380, 160], "二行目の右"), _word([60, 60, 200, 100], "見出し"),
            _word([60, 120, 200, 160], "二行目"), _word([210, 60, 390, 100], "𠮷野家 AB"),
            _word([640, 60, 680, 400], "縦書き一列目", "vertical"), _word([580, 60, 620, 300], "二列目", "vertical"),
            _word([520, 70, 560, 560], "三列目𩸽", "vertical"),
            _word([310, 260, 390, 290], "セルB"), _word([210, 260, 290, 290], "セルA"),
            _word([210, 310, 290, 340], "セルC"), _word([310, 310, 390, 340], "セルD"),
            _word([70, 410, 110, 590], "図の縦", "vertical"), _word([120, 410, 170, 500], "図二", "vertical"),
            _word([210, 430, 470, 470], "図の横書き"),
            {"points": [[50.7, 705.2], [150.9, 705.2], [150.9, 745.8], [50.7, 745.8]], "content": "float quad",
             "direction": "horizontal", "rec_score": 0.9, "det_score": 0.9},
            _word([160, 705, 290, 745], ""),
            _word([700, 900, 780, 950], "どこにもない"),
            _word([70, 170, 150, 170], "高さ0"), _word([300, 130, 300, 150], "幅0"),
            _word([150, 60, 150, 80], "縦幅0", "vertical"),
        ],
    }
    # a word inside two containers: a paragraph drawn over a table cell
    page2 = {
        "paragraphs": [_para([0, 0, 500, 100], 1), _para([0, 150, 250, 300], 2)],
        "tables": [_table(0, [(0, 0, [0, 150, 250, 300]), (0, 1, [250, 150, 500, 300])])],
        "figures": [],
        "words": [_word([10, 160, 100, 200], "両方"), _word([300, 160, 400, 200], "右セル"),
                  _word([10, 10, 100, 50], "上"), _word([200, 10, 300, 50], "上二"), _word([110, 10, 190, 50], "上一"),
                  _word([10, 210, 100, 250], "同じ行"), _word([10, 210, 100, 250], "同じ箱")],
    }
    return [({"H": 1000, "W": 800}, page1), ({"H": 400, "W": 600}, page2)]


def random_page(rng, H=900, W=700):
    chars = "あいうえおカキクケコ漢字表図ABCxyz0123𠀋😀"
    n_el = int(rng.integers(2, 7))
    orders = [int(o) for o in rng.permutation(n_el)]
    doc = {"paragraphs": [], "tables": [], "figures": [], "words": []}

    def box():
        x1, y1 = int(rng.integers(0, W - 60)), int(rng.integers(0, H - 60))
        return [x1, y1, x1 + int(rng.integers(30, 300)), y1 + int(rng.integers(30, 300))]

    for o in orders:
        kind = rng.integers(0, 3)
        if kind == 0:
            doc["paragraphs"].append(_para(box(), o, "vertical" if rng.random() < 0.4 else "horizontal"))
        elif kind == 1:
            cells = []
            for r in range(int(rng.integers(1, 3))):
                for c in range(int(rng.integers(1, 3))):
                    cells.append((r, c, box()))
            rng.shuffle(cells)
            doc["tables"].append(_table(o, cells))
        else:
            doc["figures"].append(_figure(o, [_para(box(), None, "vertical" if rng.random() < 0.4 else "horizontal")
                                              for _ in range(int(rng.integers(0, 3)))]))
    for _ in range(int(rng.integers(10, 25))):
        x1, y1 = rng.uniform(0, W - 40), rng.uniform(0, H - 40)
        x2, y2 = x1 + rng.uniform(5, 120), y1 + rng.uniform(5, 120)
        text = "".join(rng.choice(list(chars), int(rng.integers(1, 6))))
        doc["words"].append({"points": [[x1, y1], [x2, y1], [x2, y2], [x1, y2]], "content": text,
                             "direction": "vertical" if rng.random() < 0.3 else "horizontal",
                             "rec_score": 0.9, "det_score": 0.9})
    return {"H": H, "W": W}, doc


def _ns(v):
    if isinstance(v, dict):
        return types.SimpleNamespace(**{k: _ns(x) for k, x in v.items()})
    if isinstance(v, list) and v and isinstance(v[0], dict):
        return [_ns(x) for x in v]
    return v


class _Recorder:
    def __init__(self):
        self.pages = [[]]
        self.considered = [[]]


REC = _Recorder()


class _Canvas:
    def __init__(self, *a, **k):
        self.rotated = False

    def setPageSize(self, size):
        pass

    def drawImage(self, *a, **k):
        pass

    def setFillColor(self, c):
        pass

    def setFont(self, name, size):
        REC.pages[-1].append({"strings": [], "rotated": False})

    def saveState(self):
        pass

    def restoreState(self):
        pass

    def translate(self, x, y):
        pass

    def rotate(self, a):
        REC.pages[-1][-1]["rotated"] = True

    def drawString(self, x, y, s):
        REC.pages[-1][-1]["strings"].append(s)

    def showPage(self):
        REC.pages.append([])
        REC.considered.append([])

    def save(self):
        pass


def _install_standins():
    rl = types.ModuleType("reportlab")
    for name in ("lib", "lib.colors", "pdfbase", "pdfbase.pdfmetrics", "pdfbase.ttfonts", "pdfgen", "pdfgen.canvas"):
        sys.modules["reportlab." + name] = types.ModuleType("reportlab." + name)
    sys.modules["reportlab"] = rl
    sys.modules["reportlab.lib.colors"].Color = lambda *a, **k: None
    pm = sys.modules["reportlab.pdfbase.pdfmetrics"]
    pm.registerFont = lambda f: None
    pm.stringWidth = lambda text, font, size: len(text) * size / 2
    sys.modules["reportlab.pdfbase"].pdfmetrics = pm
    sys.modules["reportlab.pdfbase.ttfonts"].TTFont = lambda *a, **k: None
    sys.modules["reportlab.pdfgen.canvas"].Canvas = _Canvas
    sys.modules["reportlab.pdfgen"].canvas = sys.modules["reportlab.pdfgen.canvas"]
    jc = types.ModuleType("jaconv")
    jc.h2z = lambda text, **k: text
    sys.modules["jaconv"] = jc
    pkg = types.ModuleType("yomitoku_ref")
    pkg.__path__ = []
    sys.modules["yomitoku_ref"] = pkg
    const = types.ModuleType("yomitoku_ref.constants")
    const.ROOT_DIR = ""
    sys.modules["yomitoku_ref.constants"] = const
    schemas = types.ModuleType("yomitoku_ref.schemas")
    schemas.DocumentAnalyzerSchema = object
    sys.modules["yomitoku_ref.schemas"] = schemas
    utils = types.ModuleType("yomitoku_ref.utils")
    utils.__path__ = []
    sys.modules["yomitoku_ref.utils"] = utils


def _load(modname, relpath):
    spec = importlib.util.spec_from_file_location(modname, os.path.join(rc.SRC, relpath))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[modname] = mod
    spec.loader.exec_module(mod)
    return mod


def main():
    from PIL import Image

    _install_standins()
    _load("yomitoku_ref.utils.misc", "utils/misc.py")
    sp = _load("yomitoku_ref.utils.searchable_pdf", "utils/searchable_pdf.py")
    calc = sp._calc_font_size

    def recording_calc(content, a, b):
        REC.considered[-1].append({"text": content, "extents": [int(a), int(b)]})
        return calc(content, a, b)

    sp._calc_font_size = recording_calc
    rng = np.random.default_rng(7)
    pages = fixed_pages() + [random_page(rng) for _ in range(3)]
    out = {"pages": []}
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)  # the reference writes its tmp_<i>.png page files into the working directory
        try:
            images = [Image.new("RGB", (shape["W"], shape["H"]), (255, 255, 255)) for shape, _ in pages]
            sp.create_searchable_pdf(images, [_ns(doc) for _, doc in pages], os.path.join(tmp, "out.pdf"))
        finally:
            os.chdir(cwd)
    for (shape, doc), drawn, considered in zip(pages, REC.pages, REC.considered):
        out["pages"].append({"shape": shape, "doc": doc, "considered": considered,
                             "drawn": [{"text": "".join(d["strings"]), "vertical": d["rotated"]} for d in drawn]})
    path = os.path.join(HERE, "pdf_ref.json")
    with open(path, "w", encoding="utf-8") as f:   # one page a line
        f.write('{"pages": [\n' + ",\n".join(json.dumps(p, ensure_ascii=False) for p in out["pages"]) + "\n]}\n")
    print("wrote", path, sum(len(p["considered"]) for p in out["pages"]), "words considered")


if __name__ == "__main__":
    main()
