"""The command line (yomitoku_b200/cli.py) on the CPU: `run` with a stub analyzer whose `analyze_pages` returns a
canned result per page, so that file naming, --combine, --pages, --batch and the error paths are checked without a
GPU.  Every file must be what the exporters write for that page's result alone."""
import json
import os

import cv2
import numpy as np
import pytest

from yomitoku_b200 import cli, export
from yomitoku_b200.data import load_image
from yomitoku_b200.schemas import DocumentAnalyzerSchema


def canned(page):
    """A result that depends on the page's pixels: a heading, a paragraph, a table and a figure."""
    h, w = page.shape[:2]
    m = float(page.mean())
    return DocumentAnalyzerSchema.model_validate({
        "paragraphs": [{"box": [0, 0, w, 8], "contents": "page %dx%d" % (h, w), "direction": "horizontal",
                        "order": 0, "role": "section_headings"},
                       {"box": [0, 10, w, 20], "contents": "mean %.4f\n*next* line" % m, "direction": "horizontal",
                        "order": 2, "role": None}],
        "tables": [{"box": [0, 20, w, 30], "n_row": 1, "n_col": 2, "rows": [], "cols": [], "spans": [], "order": 1,
                    "cells": [{"row": 1, "col": 1, "row_span": 1, "col_span": 1, "box": [0, 20, 5, 30],
                               "contents": "a,b"},
                              {"row": 1, "col": 2, "row_span": 1, "col_span": 1, "box": [5, 20, 10, 30],
                               "contents": "%d" % h}]}],
        "figures": [{"box": [2, 3, min(w, 30), min(h, 25)], "order": 3, "direction": "horizontal",
                     "paragraphs": [{"box": [2, 3, 9, 9], "contents": "in figure", "direction": "horizontal",
                                     "order": 0, "role": None}]}],
        "words": []})


class StubAnalyzer:
    def __init__(self):
        self.calls = []

    def analyze_pages(self, pages):
        self.calls.append(len(pages))
        return [canned(p) for p in pages]


def _page(seed, h, w):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _tiff(path, pages):
    from PIL import Image
    imgs = [Image.fromarray(p[:, :, ::-1].copy()) for p in pages]
    imgs[0].save(str(path), save_all=True, append_images=imgs[1:])


@pytest.fixture
def tree(tmp_path):
    """in/c.png (48x64), in/.hidden/a.png (40x50), in/sub/scan.tiff (3 frames of different sizes)."""
    root = tmp_path / "in"
    (root / ".hidden").mkdir(parents=True)
    (root / "sub").mkdir()
    cv2.imwrite(str(root / "c.png"), _page(1, 48, 64))
    cv2.imwrite(str(root / ".hidden" / "a.png"), _page(2, 40, 50))
    _tiff(root / "sub" / "scan.tiff", [_page(3, 40, 60), _page(4, 56, 36), _page(5, 33, 70)])
    return root


def _args(*argv):
    return cli.build_parser().parse_args([str(a) for a in argv])


def _expected_page(fmt, page, out_path, **kw):
    """What the exporter writes for this page alone (into a scratch copy of out_path's directory)."""
    res = canned(page)
    if fmt == "json":
        export.export_json(res, out_path, img=page, **kw)
    elif fmt == "csv":
        export.export_csv(res, out_path, img=page, **kw)
    elif fmt == "html":
        export.export_html(res, out_path, img=page, **kw)
    else:
        export.export_markdown(res, out_path, img=page, **kw)


def _files(d):
    return sorted(str(p.relative_to(d)) for p in d.rglob("*") if p.is_file())


@pytest.mark.parametrize("fmt", ["json", "csv", "html", "md"])
def test_one_file_per_page(tree, tmp_path, fmt):
    out = tmp_path / "out"
    an = StubAnalyzer()
    written = cli.run(_args(tree, "-f", fmt, "-o", out, "--figure", "--figure_letter", "--batch", 2), an)
    names = ["_hidden_a_p1", "in_c_p1", "sub_scan_p1", "sub_scan_p2", "sub_scan_p3"]
    assert sorted(os.path.basename(w) for w in written) == ["%s.%s" % (n, fmt) for n in names]
    assert an.calls == [2, 2, 1]
    # byte-equal to the exporter on each page alone, figures included
    ref = tmp_path / "ref"
    ref.mkdir()
    kw = dict(export_figure=True)
    if fmt != "json":
        kw["export_figure_letter"] = True
    pages = {"_hidden_a_p1": load_image(tree / ".hidden" / "a.png")[0], "in_c_p1": load_image(tree / "c.png")[0]}
    for i, p in enumerate(load_image(tree / "sub" / "scan.tiff")):
        pages["sub_scan_p%d" % (i + 1)] = p
    for name, page in pages.items():
        _expected_page(fmt, page, str(ref / ("%s.%s" % (name, fmt))), **kw)
    assert _files(out) == _files(ref)
    for f in _files(ref):
        assert (out / f).read_bytes() == (ref / f).read_bytes(), f
    assert len([f for f in _files(out) if f.startswith("figures/")]) == 5


@pytest.mark.parametrize("fmt", ["json", "csv", "html", "md"])
def test_combine(tree, tmp_path, fmt):
    out = tmp_path / "out"
    an = StubAnalyzer()
    written = cli.run(_args(tree / "sub" / "scan.tiff", "-f", fmt, "-o", out, "--combine", "--figure", "--batch", 2),
                      an)
    assert [os.path.basename(w) for w in written] == ["sub_scan.%s" % fmt]
    assert an.calls == [2, 1]
    pages = load_image(tree / "sub" / "scan.tiff")
    ref = tmp_path / "ref"
    ref.mkdir()
    parts = []
    for i, p in enumerate(pages):
        page_path = str(ref / ("sub_scan_p%d.%s" % (i + 1, fmt)))
        res = canned(p)
        if fmt == "json":
            parts.append(export.convert_json(res, page_path, False, p, True, "figures").model_dump())
        elif fmt == "csv":
            parts.extend(export.convert_csv(res, page_path, False, img=p))
        elif fmt == "html":
            parts.append(export.convert_html(res, page_path, False, True, False, img=p)[0])
        else:
            parts.append(export.convert_markdown(res, page_path, img=p)[0])
    merged = ref / ("sub_scan.%s" % fmt)
    save = {"json": export.save_json, "csv": export.save_csv, "html": export.save_html, "md": export.save_markdown}
    save[fmt](parts if fmt in ("json", "csv") else "\n".join(parts), str(merged), "utf-8")
    assert _files(out) == _files(ref)
    for f in _files(ref):
        assert (out / f).read_bytes() == (ref / f).read_bytes(), f
    if fmt == "json":
        assert len(json.loads(merged.read_text(encoding="utf-8"))) == 3


def test_combine_across_batches_and_files(tree, tmp_path):
    """A file whose pages straddle two batches is written once, when its last page is done."""
    out = tmp_path / "out"
    an = StubAnalyzer()
    written = cli.run(_args(tree, "-f", "md", "-o", out, "--combine", "--batch", 3), an)
    assert sorted(os.path.basename(w) for w in written) == ["_hidden_a.md", "in_c.md", "sub_scan.md"]
    assert an.calls == [3, 2]
    text = (out / "sub_scan.md").read_text(encoding="utf-8")
    assert text.count("\\# page") == 0 and text.count("# page") == 3


def test_pages_selects_tiff_frames(tree, tmp_path):
    out = tmp_path / "out"
    an = StubAnalyzer()
    written = cli.run(_args(tree / "sub" / "scan.tiff", "-o", out, "--pages", "1,3-5"), an)
    assert [os.path.basename(w) for w in written] == ["sub_scan_p1.json", "sub_scan_p3.json"]
    assert an.calls == [2]
    assert cli.parse_pages("1,2,5-7,2") == [1, 2, 5, 6, 7]


def test_markdown_is_md_and_names_are_sanitised(tmp_path):
    d = tmp_path / "..dots"
    d.mkdir()
    cv2.imwrite(str(d / "x.y.png"), _page(9, 40, 40))
    written = cli.run(_args(d / "x.y.png", "-f", "markdown", "-o", tmp_path / "o"), StubAnalyzer())
    assert [os.path.basename(w) for w in written] == ["__dots_x.y_p1.md"]
    assert cli._sanitize_path_component(".a.b") == "_a.b" and cli._sanitize_path_component("") == ""


def test_bad_options(tree, tmp_path):
    an = StubAnalyzer()
    with pytest.raises(ValueError, match="Invalid output format"):
        cli.run(_args(tree, "-f", "docx", "-o", tmp_path / "o"), an)
    with pytest.raises(ValueError, match="Invalid encoding"):
        cli.run(_args(tree, "--encoding", "latin-1", "-o", tmp_path / "o"), an)
    with pytest.raises(ValueError, match="PDF output"):
        cli.run(_args(tree, "-f", "pdf", "-o", tmp_path / "o"), an)
    with pytest.raises(ValueError, match="--batch"):
        cli.run(_args(tree, "--batch", "0", "-o", tmp_path / "o"), an)
    for argv in (["-v"], ["--font_path", "f.ttf"], ["--pdf_quality", "high"], ["--dpi", "300"]):
        with pytest.raises(SystemExit):
            _args(tree, *argv)
    pdf = tmp_path / "doc.pdf"
    pdf.write_bytes(b"%PDF-1.4\n%%EOF\n")
    with pytest.raises(ValueError, match="PDF input is not supported"):
        cli.run(_args(pdf, "-o", tmp_path / "o"), an)
    with pytest.raises(FileNotFoundError):
        cli.run(_args(tmp_path / "missing", "-o", tmp_path / "o"), an)
    with pytest.raises(ValueError, match="PDF input is not supported"):
        cli.main([str(pdf), "-o", str(tmp_path / "o")])     # refused before any model is built
    assert an.calls == []


def test_unreadable_files_are_skipped(tree, tmp_path):
    (tree / "broken.png").write_bytes(b"not an image")
    (tree / "notes.txt").write_text("hello")
    (tree / "doc.pdf").write_bytes(b"%PDF-1.4\n%%EOF\n")
    cv2.imwrite(str(tree / "tiny.png"), _page(7, 20, 20))
    an = StubAnalyzer()
    written = cli.run(_args(tree, "-o", tmp_path / "out", "--batch", 16), an)
    assert sorted(os.path.basename(w) for w in written) == [
        "_hidden_a_p1.json", "in_c_p1.json", "sub_scan_p1.json", "sub_scan_p2.json", "sub_scan_p3.json"]
    assert an.calls == [5]


def test_analyzer_configs():
    lite = cli.analyzer_configs(_args("x", "--lite", "--enable-rec-orientation-fallback",
                                      "--rec-orientation-fallback-thresh", "0.5", "--tr_cfg", "r.yaml"))
    rec = lite["ocr"]["text_recognizer"]
    assert rec == {"path_cfg": "r.yaml", "model_name": "parseq-tiny-dynw-v4", "dynamic_width": True,
                   "batch_bucketing": True, "source_downscale": True, "rec_orientation_fallback": True,
                   "rec_orientation_fallback_thresh": 0.5}
    full = cli.analyzer_configs(_args("x", "--td_name", "dbnet", "--lp_cfg", "lp.yaml"))
    assert full["ocr"]["text_detector"] == {"path_cfg": None, "model_name": "dbnet"}
    assert full["ocr"]["text_recognizer"]["model_name"] == "parseq-large-v4_1"
    assert full["layout_analyzer"]["layout_parser"] == {"path_cfg": "lp.yaml"}
    a = _args("x")
    assert (a.format, a.outdir, a.device, a.batch, a.figure_width, a.figure_dir, a.reading_order) == \
        ("json", "results", "cuda", 16, 200, "figures", "auto")


def test_module_entry_point():
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "yomitoku_b200", "--help"], cwd=root, capture_output=True, text=True)
    assert r.returncode == 0 and "--batch" in r.stdout and "--combine" in r.stdout
