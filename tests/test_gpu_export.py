"""GPU: the command line end to end with seeded models (DBNet with the trained binarize head, parseq-tiny-dynw-v4 with
peaked seeded weights) over a folder of synthetic pages of two sizes, and the exporters fed a CUDA page."""
import json

import cv2
import numpy as np
import pytest
import torch

from oracle import parseq as ops
from oracle import weights
from trained_head import load_trained_head
from yomitoku_b200 import DocumentAnalyzer, cli, export
from yomitoku_b200 import schemas as S
from yomitoku_b200.data import load_image
from yomitoku_b200.synth import synthetic_page

pytestmark = pytest.mark.gpu

REC = {"from_pretrained": False, "model_name": "parseq-tiny-dynw-v4", "dynamic_width": True, "batch_bucketing": True}
NOP = {"from_pretrained": False}
WRITERS = {"md": export.export_markdown, "html": export.export_html, "csv": export.export_csv,
           "json": export.export_json}


def stub_layout(img):
    """A table over the first text rows, a paragraph region and a figure over part of the text, scaled to the page."""
    h, w = img.shape[:2]
    cw, ch = (w - 40) // 3, 58
    cells = [S.TableCellSchema(col=c + 1, row=r + 1, col_span=1, row_span=1,
                               box=[20 + cw * c, 10 + ch * r, 20 + cw * (c + 1), 10 + ch * (r + 1)], contents=None)
             for r in range(3) for c in range(3)]
    table = S.TableStructureRecognizerSchema(box=[20, 10, 20 + 3 * cw, 10 + 3 * ch], n_row=3, n_col=3, rows=[],
                                             cols=[], spans=[], cells=cells, order=0)
    para = S.Element(id=None, box=[0, h // 3, w, h // 2], score=0.9, role="section_headings", contents=None)
    fig = S.Element(id=None, box=[w // 2, h // 2 + 20, w - 10, h - 30], score=0.9, role=None, contents=None)
    return S.LayoutAnalyzerSchema(paragraphs=[para], tables=[table], figures=[fig]), None


def _analyzer(layout_analyzer=None):
    cfg = {"ocr": {"text_detector": NOP, "text_recognizer": REC},
           "layout_analyzer": {"layout_parser": NOP, "table_structure_recognizer": NOP}}
    an = DocumentAnalyzer(configs=cfg, device="cuda", layout_analyzer=layout_analyzer)
    an.text_recognizer.model.load_state_dict(weights.make_parseq_state_dict(ops.SPECS["parseq-tiny-dynw-v4"], seed=11,
                                                                            peaked=True))
    load_trained_head(an.text_detector.model)
    return an


def _write_pages(d):
    """Four PNG pages of two sizes (1200x1600 and 1600x1200) in two folders; returns {output stem: page}."""
    (d / "a").mkdir(parents=True)
    (d / "b").mkdir()
    pages = {}
    for i, (sub, portrait) in enumerate([("a", False), ("a", True), ("b", False), ("b", True)]):
        page = synthetic_page(300 + i, portrait=portrait)[0]
        cv2.imwrite(str(d / sub / ("page%d.png" % i)), page)
        pages["%s_page%d_p1" % (sub, i)] = load_image(d / sub / ("page%d.png" % i))[0]
    return pages


def _floats_close(a, b):
    """JSON values equal, floats (the recognition scores) to 1e-6: analyze_pages and the one-page call agree on
    every word, box and text, and on the scores to that tolerance."""
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_floats_close(a[k], b[k]) for k in a)
    if isinstance(a, list):
        return len(a) == len(b) and all(_floats_close(x, y) for x, y in zip(a, b))
    if isinstance(a, float) or isinstance(b, float):
        return abs(a - b) <= 1e-6
    return a == b


def _check_run_equals_single_pages(an, tmp_path, fmt, extra=()):
    src = tmp_path / "in"
    pages = _write_pages(src)
    out, ref = tmp_path / ("out_" + fmt), tmp_path / ("ref_" + fmt)
    ref.mkdir()
    calls = []
    batched = an.analyze_pages

    def counting(pages_):
        calls.append(len(pages_))
        return batched(pages_)
    an.analyze_pages = counting
    written = cli.run(cli.build_parser().parse_args([str(src), "-f", fmt, "-o", str(out), "--batch", "3", "--figure",
                                                     *extra]), an)
    del an.analyze_pages
    assert calls == [3, 1]
    assert sorted(p.name for p in out.glob("*.%s" % fmt)) == sorted("%s.%s" % (k, fmt) for k in pages)
    assert len(written) == 4
    kw = dict(export_figure=True)
    if fmt in ("md", "html"):
        kw["export_figure_letter"] = "--figure_letter" in extra
    n_fig = 0
    for stem, page in pages.items():
        res = an(page)[0]
        n_fig += len(res.figures)
        WRITERS[fmt](res, str(ref / ("%s.%s" % (stem, fmt))), img=page, **kw)
    got = sorted(p.relative_to(out) for p in out.rglob("*") if p.is_file())
    assert got == sorted(p.relative_to(ref) for p in ref.rglob("*") if p.is_file())
    for f in got:
        if f.suffix == ".json":
            assert _floats_close(json.loads((out / f).read_text(encoding="utf-8")),
                                 json.loads((ref / f).read_text(encoding="utf-8"))), f
        else:
            assert (out / f).read_bytes() == (ref / f).read_bytes(), f
    return n_fig


@pytest.mark.parametrize("fmt", ["md", "json"])
def test_run_equals_per_page_export(tmp_path, fmt):
    """run() over mixed-size pages in batches of 3 writes, page by page, what the exporter writes for analyzer(page)
    alone - figure crops included."""
    an = _analyzer(stub_layout)
    n_fig = _check_run_equals_single_pages(an, tmp_path, fmt, extra=("--figure_letter",) if fmt == "md" else ())
    assert n_fig == 4
    an._batched.close()


def test_run_with_default_layout_models(tmp_path):
    """The same with the built-in layout analyzer (seeded RT-DETRv2 layout parser and table recogniser)."""
    an = _analyzer()
    _check_run_equals_single_pages(an, tmp_path, "html")
    an._batched.close()


def test_cuda_page_exports_equal_numpy_page(tmp_path):
    page = synthetic_page(7)[0]
    res = S.DocumentAnalyzerSchema.model_validate({
        "paragraphs": [{"box": [0, 0, 100, 20], "contents": "x", "direction": "horizontal", "order": 0, "role": None}],
        "tables": [], "words": [],
        "figures": [{"box": [10, 20, 410, 333], "order": 1, "paragraphs": [], "direction": "horizontal"},
                    {"box": [1500, 1100, 1700, 1300], "order": 2, "paragraphs": [], "direction": "horizontal"}]})
    dev = torch.from_numpy(page).cuda()
    for fmt, write in WRITERS.items():
        a, b = tmp_path / "np" / ("p.%s" % fmt), tmp_path / "cuda" / ("p.%s" % fmt)
        a.parent.mkdir(exist_ok=True)
        b.parent.mkdir(exist_ok=True)
        write(res, str(a), img=page, export_figure=True)
        write(res, str(b), img=dev, export_figure=True)
        assert a.read_bytes() == b.read_bytes()
    for i in range(2):
        fa = tmp_path / "np" / "figures" / ("p_figure_%d.png" % i)
        fb = tmp_path / "cuda" / "figures" / ("p_figure_%d.png" % i)
        assert fa.read_bytes() == fb.read_bytes()
    crop = cv2.imdecode(np.frombuffer(fb.read_bytes(), np.uint8), cv2.IMREAD_COLOR)
    assert crop.shape == (100, 100, 3)          # the second figure is clipped at the page's corner
