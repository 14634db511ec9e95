"""The exporters (yomitoku_b200/export.py), the schema methods that call them and data.load_image against what
yomitoku's own exporters and load_image give (tests/golden/export_ref.json, made by make_golden_export.py)."""
import hashlib
import itertools
import json
import os

import cv2
import numpy as np
import pytest

from yomitoku_b200 import export
from yomitoku_b200.data import load_image
from yomitoku_b200.schemas import DocumentAnalyzerSchema

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "export_ref.json")
with open(GOLDEN, encoding="utf-8") as _f:
    REF = json.load(_f)
WRITERS = {"md": export.export_markdown, "html": export.export_html, "csv": export.export_csv,
           "json": export.export_json}
# yomitoku asserts that an image is given for export_figure; here that is a ValueError
ERROR_TYPES = {"!AssertionError": ValueError, "!TypeError": TypeError, "!AttributeError": AttributeError}


def sha16(data):
    return hashlib.sha256(data).hexdigest()[:16]


def expand_runs(g):
    """(case, format, kwargs, with image) of every run, in the order of the golden's results (as the generator
    expands the same axes)."""
    out = []
    for case, (fmt, names) in itertools.product(g["cases"], g["options"].items()):
        names = ["ignore_line_break"] + names
        for values in itertools.product(*(g["values"][n] for n in names)):
            out.append((case, fmt, dict(zip(names, values), encoding="utf-8"), True))
    for (case, enc), fmt in itertools.product(g["encoding_runs"], g["options"]):
        out.append((case, fmt, {"encoding": enc, "export_figure": False}, False))
    for fmt in g["options"]:
        out.append(("figures", fmt, {"export_figure": True, "encoding": "utf-8"}, False))
    return out


RUNS = expand_runs(REF)
assert len(RUNS) == len(REF["results"])


def page_image():
    return np.random.default_rng(REF["image"]["seed"]).integers(0, 256, REF["image"]["shape"], dtype=np.uint8)


def _schema(case):
    return DocumentAnalyzerSchema.model_validate(REF["cases"][case])


def _run_id(run):
    case, fmt, kwargs, with_img = run
    return "%s-%s-%s%s" % (case, fmt, "-".join("%s=%s" % kv for kv in sorted(kwargs.items())),
                           "" if with_img else "-noimg")


@pytest.mark.parametrize("i", range(len(RUNS)), ids=[_run_id(r) for r in RUNS])
def test_export_matches_reference(i, tmp_path):
    case, fmt, kwargs, with_img = RUNS[i]
    want, want_figs = REF["results"][i], REF["figures"].get(str(i), [])
    inputs = _schema(case)
    before = inputs.model_dump()
    img = page_image() if with_img else None
    out_path = tmp_path / "out" / ("doc_p1.%s" % fmt)
    out_path.parent.mkdir()
    if want.startswith("!"):
        with pytest.raises(ERROR_TYPES[want]):
            WRITERS[fmt](inputs, str(out_path), img=img, **kwargs)
        assert not out_path.exists()
    else:
        WRITERS[fmt](inputs, str(out_path), img=img, **kwargs)
        data = out_path.read_bytes()
        assert sha16(data) == want, data.decode(kwargs["encoding"], errors="replace")
    # figure files: same paths, JPEG bytes of the same crop
    figs = sorted(str(p.relative_to(tmp_path)) for p in tmp_path.rglob("*_figure_*"))
    assert figs == sorted(f[0] for f in want_figs)
    for path, shape, crop_sha in want_figs:
        data = (tmp_path / path).read_bytes()
        assert list(cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR).shape) == shape
        k = int(path.rsplit("_figure_", 1)[1].split(".")[0])
        x1, y1, x2, y2 = REF["cases"][case]["figures"][k]["box"]
        crop = page_image()[y1:y2, x1:x2, :]
        assert sha16(np.ascontiguousarray(crop).tobytes()) == crop_sha
        assert data == cv2.imencode(".jpg", crop)[1].tobytes()
    assert inputs.model_dump() == before          # the caller's result is untouched


def test_convert_returns_what_export_writes(tmp_path):
    inputs, img = _schema("figures"), page_image()
    out = str(tmp_path / "a.md")
    md, elements = export.convert_markdown(inputs, out, img=img, export_figure_letter=True)
    assert md == export.export_markdown(inputs, out, img=img, export_figure_letter=True)
    assert [e["order"] for e in elements] == sorted(e["order"] for e in elements)
    out = str(tmp_path / "a.html")
    html, _ = export.convert_html(inputs, out, False, True, True, img=img)
    assert html == export.export_html(inputs, out, img=img, export_figure_letter=True)
    out = str(tmp_path / "a.json")
    copy = export.convert_json(inputs, out, True, img, True, "figures")
    assert [f.figure_path for f in copy.figures] == [os.path.join("figures", "a_figure_%d.png" % i) for i in range(2)]
    assert all(f.figure_path is None for f in inputs.figures)


def test_schema_methods(tmp_path):
    inputs, img = _schema("figures"), page_image()
    kw = dict(img=img, export_figure_letter=True, figure_dir="figs")
    cases = (("to_markdown", export.export_markdown, "md"), ("to_html", export.export_html, "html"),
             ("to_csv", export.export_csv, "csv"))
    for method, fn, ext in cases:
        a, b = tmp_path / "method" / ("p.%s" % ext), tmp_path / "function" / ("p.%s" % ext)
        a.parent.mkdir(exist_ok=True)
        b.parent.mkdir(exist_ok=True)
        getattr(inputs, method)(str(a), **kw)
        fn(inputs, str(b), **kw)
        assert a.read_bytes() == b.read_bytes()
        for i in range(2):
            name = "p_figure_%d.png" % i
            assert (a.parent / "figs" / name).read_bytes() == (b.parent / "figs" / name).read_bytes()
    with pytest.raises(ValueError, match="img is required"):
        inputs.to_markdown(str(tmp_path / "x.md"))      # export_figure is on by default, as in yomitoku
    # to_json stays the generic schema dump; export_json is yomitoku's file
    inputs.to_json(str(tmp_path / "g.json"))
    assert json.loads((tmp_path / "g.json").read_text(encoding="utf-8")) == inputs.model_dump()


def _write_load_files(tmp):
    from PIL import Image
    for name, frames in REF["load_files"].items():
        imgs = []
        for mode, h, w, seed in frames:
            c = {"RGBA": 4, "RGB": 3, "L": 1}[mode]
            a = np.random.default_rng(seed).integers(0, 256, (h, w, c), dtype=np.uint8)
            imgs.append(Image.fromarray(a[:, :, 0] if c == 1 else a, mode))
        imgs[0].save(os.path.join(tmp, name), save_all=len(imgs) > 1, append_images=imgs[1:])
    (tmp / "doc.pdf").write_bytes(b"%PDF-1.4\n%%EOF\n")
    (tmp / "anim.gif").write_bytes(b"GIF89a")


def test_load_image_matches_reference(tmp_path):
    _write_load_files(tmp_path)
    for name, want in REF["load_image"].items():
        if "pages" in want:
            pages = load_image(tmp_path / name)
            got = [[list(p.shape), str(p.dtype), sha16(np.ascontiguousarray(p).tobytes())] for p in pages]
            assert got == want["pages"], name
            continue
        with pytest.raises(ValueError) as e:
            load_image(tmp_path / name)
        if name == "doc.pdf":
            assert "PDF" in str(e.value) and "not part of this package" in str(e.value)
        else:
            assert str(e.value) == want["message"].replace(", 'pdf'", "")
    assert len(REF["load_image"]["scan.tiff"]["pages"]) == 3
    with pytest.raises(FileNotFoundError):
        load_image(tmp_path / "missing.png")


def test_load_image_warns_on_small_pages(tmp_path, caplog):
    import logging
    _write_load_files(tmp_path)
    logging.getLogger("yomitoku_b200.data").propagate = True
    with caplog.at_level(logging.WARNING, logger="yomitoku_b200.data"):
        load_image(tmp_path / "page.png")
    assert any("image size is small" in r.getMessage() for r in caplog.records)
    big = tmp_path / "big.png"
    cv2.imwrite(str(big), np.zeros((720, 800, 3), np.uint8))
    caplog.clear()
    with caplog.at_level(logging.WARNING, logger="yomitoku_b200.data"):
        pages = load_image(big)
    assert not caplog.records and pages[0].shape == (720, 800, 3)
