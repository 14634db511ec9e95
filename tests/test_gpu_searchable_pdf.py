"""GPU: the searchable PDF's device path (yomitoku_b200/searchable_pdf.py).

  * the device resize (ytk_resize_pages_u8, LANCZOS) equals Pillow's Image.resize((w, h), LANCZOS) byte for byte on a
    mixed-size batch for every preset; `high` is the plain BGR -> RGB transpose;
  * nvJPEG pages decode (cv2.imdecode) to the target size, within 1 dB of Pillow's own JPEG's PSNR at the same quality;
  * numpy pages, CUDA pages and a DevicePages give byte-identical files;
  * end to end: DocumentAnalyzer.analyze_pages(dp), then create_searchable_pdf(dp, results): the text layer read back
    holds the words the order rules select from those results."""
import io

import cv2
import numpy as np
import pytest
import torch
from PIL import Image

from test_gpu_export import _analyzer, stub_layout
from test_searchable_pdf_host import Pdf, jpeg_size, text_layer
from yomitoku_b200 import create_searchable_pdf, device_pages
from yomitoku_b200.searchable_pdf import PRESETS, _poly2rect, encode_pages, resize_pages, target_size, text_layer_words
from yomitoku_b200.synth import synthetic_page

pytestmark = pytest.mark.gpu

SHAPES = [(3508, 2480), (1600, 1200), (1200, 1600), (2101, 1499), (777, 513), (2400, 61)]


def pages_of(shapes, seed=0):
    out = []
    for k, (H, W) in enumerate(shapes):
        page = synthetic_page(seed + k)[0]
        out.append(np.ascontiguousarray(cv2.resize(page, (W, H), interpolation=cv2.INTER_LINEAR)))
    return out


def pil_resize(page_bgr, size):
    img = Image.fromarray(np.ascontiguousarray(page_bgr[:, :, ::-1]))
    return np.asarray(img if img.size == size else img.resize(size, Image.LANCZOS))


@pytest.mark.parametrize("quality", list(PRESETS))
def test_device_resize_equals_pillow(quality):
    pages = pages_of(SHAPES)
    dp = device_pages([torch.from_numpy(p).cuda() for p in pages])
    sizes = [target_size(W, H, quality) for H, W in dp.shapes]
    dp.ready(torch.cuda.current_stream())
    out = resize_pages(dp.buf, [int(o) for o in dp.table["page_off"]], dp.shapes, sizes)
    torch.cuda.synchronize()
    for page, size, planar in zip(pages, sizes, out):
        got = planar.permute(1, 2, 0).cpu().numpy()
        if quality == "high":
            np.testing.assert_array_equal(got, page[:, :, ::-1])
        np.testing.assert_array_equal(got, pil_resize(page, size), err_msg="%s %s" % (page.shape, size))


def psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return 10 * np.log10(255.0 ** 2 / mse)


@pytest.mark.parametrize("quality", list(PRESETS))
def test_jpeg_quality(quality):
    pages = pages_of(SHAPES[:4], seed=20)
    q = PRESETS[quality][1]
    report = []
    for (data, (w, h), (W, H)), page in zip(encode_pages(pages, quality), pages):
        assert (W, H) == (page.shape[1], page.shape[0])
        ref = pil_resize(page, (w, h))
        dec = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)
        assert dec.shape == (h, w, 3) and jpeg_size(data) == (w, h, 3)
        buf = io.BytesIO()
        Image.fromarray(ref).save(buf, format="JPEG", quality=q)
        pil_dec = np.asarray(Image.open(io.BytesIO(buf.getvalue())).convert("RGB"))
        ours, theirs = psnr(dec[:, :, ::-1], ref), psnr(pil_dec, ref)
        report.append("%dx%d nvJPEG %d B %.2f dB, Pillow %d B %.2f dB" % (w, h, len(data), ours, buf.tell(), theirs))
        assert ours >= theirs - 1.0, report[-1]
    print("\n[%s q%d] " % (quality, q) + "; ".join(report))


def _doc():
    from yomitoku_b200 import schemas as S
    words = [S.WordPrediction(points=[[100, 100], [300, 100], [300, 140], [100, 140]], content="検索できる",
                              direction="horizontal", rec_score=0.9, det_score=0.9),
             S.WordPrediction(points=[[500, 100], [540, 100], [540, 400], [500, 400]], content="縦書き",
                              direction="vertical", rec_score=0.9, det_score=0.9)]
    paras = [S.ParagraphSchema(box=[90, 90, 310, 150], contents=None, direction="horizontal", order=0, role=None),
             S.ParagraphSchema(box=[490, 90, 550, 410], contents=None, direction="vertical", order=1, role=None)]
    return S.DocumentAnalyzerSchema(paragraphs=paras, tables=[], words=words, figures=[])


@pytest.mark.parametrize("quality", ["high", "low"])
def test_page_forms_give_identical_files(tmp_path, quality):
    pages = pages_of([(1600, 1200), (2101, 1499), (777, 513)], seed=40)
    docs = [_doc() for _ in pages]
    forms = {"numpy": pages, "cuda": [torch.from_numpy(p).cuda() for p in pages]}
    forms["device_pages"] = device_pages(forms["cuda"])
    data = {}
    for name, imgs in forms.items():
        path = tmp_path / ("%s.pdf" % name)
        create_searchable_pdf(imgs, docs, str(path), image_quality=quality)
        data[name] = path.read_bytes()
    assert data["numpy"] == data["cuda"] == data["device_pages"]
    words = text_layer(Pdf(data["numpy"]))
    assert [[t for t, _, _ in p] for p in words] == [["検索できる", "縦書き"]] * 3


def test_end_to_end_from_analyze_pages(tmp_path):
    an = _analyzer(stub_layout)
    pages = [synthetic_page(60)[0], synthetic_page(61, portrait=True)[0]]
    dp = device_pages([torch.from_numpy(p).cuda() for p in pages])
    results = an.analyze_pages(dp)
    path = tmp_path / "doc.pdf"
    create_searchable_pdf(dp, results, str(path), image_quality="middle")
    layer = text_layer(Pdf(path.read_bytes()))
    total = 0
    for res, words, page in zip(results, layer, pages):
        want = [w.content for w in text_layer_words(res)
                if w.content and (lambda r: r[2] > r[0] and r[3] > r[1])(_poly2rect(w.points))]
        assert [t for t, _, _ in words] == want
        total += len(want)
    assert total > 0
