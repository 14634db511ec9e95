"""GPU: batches of pages of different sizes, from the page-table kernels up to the public API.

  op level      the page-table entries against the same-size entries page by page, bit for bit: detector
                pre-processing (ytk_op_dbnet_preprocess_table_u8 vs ytk_op_dbnet_preprocess_u8 / _up_u8), crop extraction
                (ytk_extract_crops_table_u8 vs ytk_extract_crops_u8, records from data.crop_records), pyramid halving
                (ytk_halve_pages_table_u8 vs cv2.resize(fx=fy=0.5, INTER_AREA), odd sizes) and the DBNet forward
                (ytk_dbnet_forward_table_u8 vs detect_pages_u8 of each page alone); invalid records are an error and
                launch nothing.
  module level  BatchedOCR / TextDetector.detect_pages / DocumentAnalyzer.analyze_pages over a mixed batch equal the
                one-page calls, with the trained detector head so that the detector's own maps carry the lines.
"""
import ctypes

import cv2
import numpy as np
import pytest
import torch

from oracle import parseq as ops
from oracle import weights
from trained_head import load_trained_head
from yomitoku_b200 import OCR, DocumentAnalyzer, TextDetector, _lib
from yomitoku_b200 import data as D
from yomitoku_b200.models import extract_crops_device, halve_pages_device
from yomitoku_b200.pipeline import BatchedOCR
from yomitoku_b200.synth import synthetic_page

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# page size -> detector input (shortest 1280, limit 1600)
SHAPES = [((1200, 1600), (1184, 1600)), ((900, 1200), (1184, 1600)), ((600, 800), (1184, 1600)),
          ((1500, 2000), (1184, 1600)), ((1600, 1200), (1600, 1184)), ((1000, 1000), (1280, 1280)),
          ((2339, 1654), (1600, 1120)), ((480, 3000), (256, 1600))]
MIXED = [(1200, 1600), (900, 1200), (1000, 1000), (600, 800), (1600, 1200), (1199, 1597)]


def _fp(t):
    return ctypes.c_void_p(t.data_ptr())


def _flat(pages):
    table, total = D.page_table([p.shape[:2] for p in pages])
    flat = torch.from_numpy(np.concatenate([p.reshape(-1) for p in pages])).to(DEV)
    assert flat.numel() == total
    return flat, table


def _random_pages(shapes, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]


def test_shapes_map_to_the_listed_detector_inputs():
    for (h, w), hnwn in SHAPES:
        assert D.shortest_edge_size(h, w, 1280, 1600) == hnwn


def test_preprocess_table_equals_same_size_op_per_page():
    pages = _random_pages([s for s, _ in SHAPES], 0)
    flat, table = _flat(pages)
    L = _lib.lib()
    for Hn, Wn in sorted({hw for _, hw in SHAPES}):
        idx = [i for i, (_, hw) in enumerate(SHAPES) if hw == (Hn, Wn)]
        n = len(idx)
        got = torch.full((n + 1, Hn + 6, Wn + 8, 8), float("nan"), dtype=torch.float16, device=DEV)
        _lib.check(L.ytk_op_dbnet_preprocess_table_u8(_fp(flat), flat.numel(), table[idx].ctypes.data, n, Hn, Wn,
                                                      _fp(got), None))
        for j, i in enumerate(idx):
            H0, W0 = pages[i].shape[:2]
            ref = torch.empty((1, Hn + 6, Wn + 8, 8), dtype=torch.float16, device=DEV)
            src = torch.from_numpy(pages[i]).to(DEV)
            op = L.ytk_op_dbnet_preprocess_u8 if (Hn <= H0 and Wn <= W0) else L.ytk_op_dbnet_preprocess_up_u8
            _lib.check(op(_fp(src), 1, H0, W0, Hn, Wn, _fp(ref), None))
            torch.cuda.synchronize()
            assert torch.equal(got[j].view(torch.int16), ref[0].view(torch.int16)), (SHAPES[i], j)
        assert torch.isnan(got[n]).all()          # nothing written past the last page


def test_dbnet_table_forward_equals_per_page_forward():
    det = TextDetector(from_pretrained=False, device="cuda")
    load_trained_head(det.model)
    pages = [synthetic_page(200 + i, height=h, width=w)[0] for i, ((h, w), hw) in enumerate(SHAPES)
             if hw == (1184, 1600)]
    flat, table = _flat(pages)
    got = det.model.detect_pages_table(flat, table)
    for i, p in enumerate(pages):
        ref = det.model.detect_pages_u8(torch.from_numpy(p).to(DEV)[None])
        assert torch.equal(got[i], ref[0]), i
    host = det.model.detect_pages_table(flat.cpu(), table)        # pages on the host: the entry copies them
    assert torch.equal(host.to(DEV), got)


def test_extract_crops_table_equals_same_size_entry_per_page():
    pages, quads = [], []
    for k, (h, w) in enumerate(MIXED):
        p, q = synthetic_page(220 + k, height=h, width=w)
        pages.append(p)
        quads.append(q[:40] + [[[30, 40], [60, 40], [60, 400], [30, 400]]])      # + one vertical line
    geoms = []
    for i, (p, q) in enumerate(zip(pages, quads)):
        g, _, _ = D.crop_records(p.shape, q, (32, 800), True, False, page=i)
        geoms.append(g)
    allg = np.ascontiguousarray(np.concatenate(geoms))
    allg[len(allg) // 2]["rot"] |= 2                                             # one 180-degree second look
    flat, table = _flat(pages)
    canv, total = extract_crops_device((flat, table), allg)
    got = canv[:total].cpu().numpy()
    base = 0
    for i, p in enumerate(pages):
        mine = allg[base:base + len(geoms[i])]
        base += len(geoms[i])
        g = mine.copy()
        g["page"] = 0
        ref_c, ref_total = extract_crops_device(torch.from_numpy(p).to(DEV)[None], g)
        ref = ref_c[:ref_total].cpu().numpy()
        for r, a in zip(g, mine):
            nb = int(r["canvas_w"]) * int(r["canvas_h"]) * 3
            assert np.array_equal(got[int(a["pix_off"]):int(a["pix_off"]) + nb],
                                  ref[int(r["pix_off"]):int(r["pix_off"]) + nb])


def test_halve_table_equals_opencv_per_page():
    pages = _random_pages([(1199, 1597), (901, 1201), (600, 799), (33, 47), (7, 5)], 1)
    level = _flat(pages)
    expect = pages
    for _ in range(2):
        level = halve_pages_device(level)
        expect = [cv2.resize(p, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_AREA) for p in expect]
        flat, table = level
        got = flat.cpu().numpy()
        assert [(int(t["H"]), int(t["W"])) for t in table] == [e.shape[:2] for e in expect]
        for t, e in zip(table, expect):
            o = int(t["page_off"])
            assert np.array_equal(got[o:o + e.size].reshape(e.shape), e)


def _err(status):
    assert status != 0
    return _lib.lib().ytk_last_error().decode()


def test_invalid_page_tables_are_errors_not_launches():
    L = _lib.lib()
    pages = _random_pages([(64, 96), (80, 64)], 2)
    flat, table = _flat(pages)
    canvas = torch.zeros((2, 64 + 6, 96 + 8, 8), dtype=torch.float16, device=DEV)
    det = TextDetector(from_pretrained=False, device="cuda")
    h = det.model._ensure()
    prob = torch.zeros((2, 1280, 1920), dtype=torch.float32, device=DEV)
    page, quads = synthetic_page(240, height=300, width=400)
    geoms, _, _ = D.crop_records(page.shape, quads[:4], (32, 800), True, False)
    geoms = np.ascontiguousarray(geoms)
    scratch_b, canv_b = D.layout_crop_buffers(geoms)
    scratch_b = scratch_b + 16 + geoms.nbytes + table.nbytes
    scratch = torch.zeros(scratch_b, dtype=torch.uint8, device=DEV)
    canv = torch.zeros(max(canv_b, 1), dtype=torch.uint8, device=DEV)
    one, _ = _flat([page])

    def variants():
        t = table.copy()
        t[1]["page_off"] = flat.numel() - 10                      # page beyond pages_bytes
        yield "beyond", t
        t = table.copy()
        t[0]["H"] = 0                                               # empty page
        yield "empty", t
        t = table.copy()
        t[1]["x1"] -= 1                                             # not the whole page
        yield "part", t

    torch.cuda.synchronize()
    launches = L.ytk_launch_count()
    for name, t in variants():
        assert "page 1" in _err(L.ytk_op_dbnet_preprocess_table_u8(_fp(flat), flat.numel(), t.ctypes.data, 2, 64, 96,
                                                                   _fp(canvas), None)) or name == "empty"
        _err(L.ytk_dbnet_forward_table_u8(h, _fp(flat), 1, flat.numel(), t.ctypes.data, 2, _fp(prob), 1, None))
        _err(L.ytk_halve_pages_table_u8(_fp(flat), flat.numel(), t.ctypes.data, 2, _fp(canvas), canvas.numel() * 2,
                                        D.page_table([(32, 48), (40, 32)])[0].ctypes.data, _fp(scratch),
                                        scratch.numel(), None))
        if name != "part":       # the crop extraction reads pages, not rectangles: a partial rectangle is valid there
            _err(L.ytk_extract_crops_table_u8(_fp(flat), flat.numel(), t.ctypes.data, 2, geoms.ctypes.data, len(geoms),
                                              _fp(scratch), scratch.numel(), _fp(canv), canv.numel(), None))
    # pages of one DBNet call that map to different network inputs: the message names both shapes
    t2, _ = D.page_table([(900, 1200), (1000, 1000)])
    big = torch.zeros(900 * 1200 * 3 + 1000 * 1000 * 3, dtype=torch.uint8, device=DEV)
    msg = _err(L.ytk_dbnet_forward_table_u8(h, _fp(big), 1, big.numel(), t2.ctypes.data, 2, _fp(prob), 1, None))
    assert "900x1200" in msg and "1184x1600" in msg and "1000x1000" in msg and "1280x1280" in msg, msg
    # crop records: page index outside the table, ROI outside its own page
    t1, _ = D.page_table([page.shape[:2]])
    for field, value in (("page", 1), ("page", -1), ("x0", 400 - int(geoms[0]["rw"]) + 1),
                         ("y0", 300 - int(geoms[0]["rh"]) + 1)):
        g = geoms.copy()
        g[0][field] = value
        assert "record 0" in _err(L.ytk_extract_crops_table_u8(_fp(one), one.numel(), t1.ctypes.data, 1, g.ctypes.data,
                                                               len(g), _fp(scratch), scratch.numel(), _fp(canv),
                                                               canv.numel(), None))
    # halving to a wrong size
    bad = D.page_table([(32, 48), (41, 32)])[0]
    assert "expected" in _err(L.ytk_halve_pages_table_u8(_fp(flat), flat.numel(), table.ctypes.data, 2, _fp(canvas),
                                                         canvas.numel() * 2, bad.ctypes.data, _fp(scratch),
                                                         scratch.numel(), None))
    # scratch too small for the records + the page table
    assert "scratch" in _err(L.ytk_extract_crops_table_u8(_fp(one), one.numel(), t1.ctypes.data, 1, geoms.ctypes.data,
                                                          len(geoms), _fp(scratch), scratch_b - table.nbytes - 16 -
                                                          geoms.nbytes, _fp(canv), canv.numel(), None))
    assert L.ytk_launch_count() == launches


# ------------------------------------------------------------------------------------------------------ module level
def _ocr(**rec):
    o = OCR(configs={"text_detector": {"from_pretrained": False},
                     "text_recognizer": {"from_pretrained": False, "model_name": "parseq-tiny-dynw-v4",
                                         "dynamic_width": True, "batch_bucketing": True, **rec}}, device="cuda")
    spec = ops.SPECS["parseq-tiny-dynw-v4"]
    o.recognizer.model.load_state_dict(weights.make_parseq_state_dict(spec, seed=11, peaked=True))
    load_trained_head(o.detector.model)
    return o


def _mixed(first=300, shapes=MIXED):
    return [synthetic_page(first + i, height=h, width=w)[0] for i, (h, w) in enumerate(shapes)]


def _same(got, ref):
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        assert len(r.words) > 10
        assert [w.points for w in g.words] == [w.points for w in r.words]
        assert [w.content for w in g.words] == [w.content for w in r.words]
        assert [w.det_score for w in g.words] == [w.det_score for w in r.words]
        assert np.allclose([w.rec_score for w in g.words], [w.rec_score for w in r.words], atol=1e-6)


@pytest.mark.parametrize("mode", ["device-crops", "host-crops", "no-pool", "fallback", "source-downscale"])
def test_batched_ocr_mixed_batch_equals_per_page_ocr(mode):
    rec = {"fallback": {"rec_orientation_fallback": True, "rec_orientation_fallback_thresh": 0.9},
           "source-downscale": {"source_downscale": True}}.get(mode, {})
    o = _ocr(**rec)
    pages = _mixed()
    ref = [o(p)[0] for p in pages]
    b = BatchedOCR(o.detector, o.recognizer, workers=1 if mode == "no-pool" else 3, det_batch=2,
                   device_crops=mode != "host-crops")
    try:
        got = b(pages)
    finally:
        b.close()
    _same(got, ref)


def test_stream_over_mixed_batches_equals_per_batch_calls():
    o = _ocr()
    pages = _mixed(320, MIXED + [(900, 1200), (1000, 1000)])
    batches = [pages[0:3], pages[3:8], pages[1:2], pages[2:6]]          # totals differ from batch to batch
    b = BatchedOCR(o.detector, o.recognizer, workers=3, det_batch=2)
    try:
        ref = [b(pg) for pg in batches]
        got = list(b.stream(batches, lookahead=2))
    finally:
        b.close()
    assert len(got) == len(batches)
    for g, r in zip(got, ref):
        _same(g, r)


def test_text_detector_detect_pages_mixed_equals_per_page_calls():
    o = _ocr()
    pages = _mixed(340)
    got = o.detector.detect_pages(pages)
    for g, p in zip(got, pages):
        r, _ = o.detector(p)
        assert g.points == r.points and g.scores == r.scores and len(r.points) > 10


def test_more_detector_shapes_than_cached_engines(monkeypatch):
    monkeypatch.setenv("YTK_DBNET_MAX_ENGINES", "2")          # read when the handle is created
    o = _ocr()
    pages = _mixed(360)
    assert len({D.shortest_edge_size(h, w, 1280, 1600) for h, w in MIXED}) > 2
    ref = [o(p)[0] for p in pages]
    b = BatchedOCR(o.detector, o.recognizer, workers=2, det_batch=2)
    try:
        got = b(pages)
    finally:
        b.close()
    _same(got, ref)


def _stub_layout(img):
    from yomitoku_b200 import schemas as S
    h, w = img.shape[:2]
    cells = [S.TableCellSchema(col=c + 1, row=r + 1, col_span=1, row_span=1,
                               box=[20 + 200 * c, 10 + 58 * r, 20 + 200 * (c + 1), 10 + 58 * (r + 1)], contents=None)
             for r in range(3) for c in range(3)]
    rows = [S.TableLineSchema(box=[20, 10 + 58 * r, 620, 68 + 58 * r], score=0.9) for r in range(3)]
    cols = [S.TableLineSchema(box=[20 + 200 * c, 10, 220 + 200 * c, 184], score=0.9) for c in range(3)]
    table = S.TableStructureRecognizerSchema(box=[20, 10, 620, 184], n_row=3, n_col=3, rows=rows, cols=cols, spans=[],
                                             cells=cells, order=0)
    para = S.Element(id=None, box=[0, h // 2, w, h - 10], score=0.9, role=None, contents=None)
    return S.LayoutAnalyzerSchema(paragraphs=[para], tables=[table], figures=[]), None


@pytest.mark.parametrize("layout", ["stub", "default"])
def test_document_analyzer_mixed_batch_equals_per_page_calls(layout):
    cfg = {"ocr": {"text_detector": {"from_pretrained": False},
                   "text_recognizer": {"from_pretrained": False, "model_name": "parseq-tiny-dynw-v4",
                                       "dynamic_width": True, "batch_bucketing": True}},
           "layout_analyzer": {"layout_parser": {"from_pretrained": False},
                               "table_structure_recognizer": {"from_pretrained": False}}}
    pages = _mixed(380, MIXED[:4])
    for split in (False, True):
        an = DocumentAnalyzer(configs=cfg, device="cuda", split_text_across_cells=split,
                              layout_analyzer=_stub_layout if layout == "stub" else None)
        load_trained_head(an.text_detector.model)
        single = [an(p)[0] for p in pages]
        batched = an.analyze_pages(pages)
        assert len(batched) == len(pages)
        for a, b in zip(single, batched):
            assert len(a.words) > 10
            assert [w.points for w in a.words] == [w.points for w in b.words]
            assert [w.content for w in a.words] == [w.content for w in b.words]
            assert [p.contents for p in a.paragraphs] == [p.contents for p in b.paragraphs]
            assert [[c.contents for c in t.cells] for t in a.tables] == [[c.contents for c in t.cells] for t in b.tables]
            assert np.allclose([w.rec_score for w in a.words], [w.rec_score for w in b.words], atol=1e-6)
        an._batched.close()
