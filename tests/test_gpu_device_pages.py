"""GPU: pages that are already on the device (yomitoku_b200/device_pages.py, ytk_pack_pages_u8 in csrc/page_ops.cu).

  pack kernel   the packed buffer equals a torch gather (flip / permute / contiguous) byte for byte: contiguous BGR, RGB,
                CHW permute views, crops and step-2 views, widths 1 / 7 / 4000, batches of 1 to 64 mixed-size pages;
                invalid records are an error and launch nothing.
  modules       a page passed on the device gives exactly the result of the same pixels as a numpy array: TextDetector,
                OCR, BatchedOCR (call and stream, orientation fallback, source_downscale), LayoutAnalyzer, CellDetector,
                DocumentAnalyzer; with device input nothing is staged or uploaded and both halves of analyze_pages read
                one buffer; pages written on a side stream the caller made current; an nvJPEG decode in RGB.
"""
import numpy as np
import pytest
import torch

from oracle import parseq as ops
from oracle import rtdetr as R
from oracle import weights
from trained_head import load_trained_head
from yomitoku_b200 import OCR, CellDetector, DocumentAnalyzer, LayoutAnalyzer, TextRecognizer, _lib, device_pages
from yomitoku_b200 import data as D
from yomitoku_b200.device_pages import PAGE_SRC_DTYPE
from yomitoku_b200.pipeline import BatchedOCR
from yomitoku_b200.synth import synthetic_page

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MIXED = [(1200, 1600), (900, 1200), (1000, 1000), (600, 800)]


def _rand(*shape, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(0, 256, shape, dtype=torch.uint8, device=DEV, generator=g)


def _check_pack(views, order):
    dp = device_pages(views, order)
    torch.cuda.synchronize()
    shapes = [tuple(v.shape[:2]) for v in views]
    table, total = D.page_table(shapes)
    assert dp.shapes == shapes and dp.buf.numel() == total and np.array_equal(dp.table, table)
    for i, v in enumerate(views):
        expect = (v.flip(-1) if order == "rgb" else v).contiguous().reshape(-1)
        o = int(table["page_off"][i])
        assert torch.equal(dp.buf[o:o + expect.numel()], expect), (i, tuple(v.shape), v.stride())


def _cases():
    base = _rand(301, 517, 3, seed=1)
    chw = _rand(3, 257, 193, seed=2)
    return {"contiguous": [base], "chw-permute": [chw.permute(1, 2, 0)],
            "crop-step2": [base[10:200, 33:301], base[::2, ::2], base[1::2, ::3], chw.permute(1, 2, 0)[::2, 5:100]],
            "widths": [_rand(5, 1, 3, seed=3), _rand(9, 7, 3, seed=4), _rand(33, 4000, 3, seed=5)],
            "stack": _rand(4, 64, 80, 3, seed=6)}


@pytest.mark.parametrize("order", ["bgr", "rgb"])
@pytest.mark.parametrize("case", ["contiguous", "chw-permute", "crop-step2", "widths", "stack"])
def test_pack_equals_torch_gather(case, order):
    views = _cases()[case]
    if isinstance(views, torch.Tensor):
        dp = device_pages(views, order)
        torch.cuda.synchronize()
        expect = (views.flip(-1) if order == "rgb" else views).contiguous().reshape(-1)
        assert torch.equal(dp.buf, expect)
        return
    _check_pack(views, order)


@pytest.mark.parametrize("n", [1, 2, 17, 64])
def test_pack_batches_of_mixed_sizes(n):
    rng = np.random.default_rng(n)
    views = []
    for i in range(n):
        h, w = (int(v) for v in rng.integers(1, 400, 2))
        kind = i % 3
        if kind == 0:
            views.append(_rand(h, w, 3, seed=i))
        elif kind == 1:
            views.append(_rand(3, h, w, seed=i).permute(1, 2, 0))
        else:
            views.append(_rand(2 * h, 2 * w + 1, 3, seed=i)[::2, 1::2])
    _check_pack(views, "rgb" if n % 2 else "bgr")


def test_invalid_pack_records_are_errors_not_launches():
    L = _lib.lib()
    page = _rand(20, 30, 3, seed=7)
    table, total = D.page_table([(20, 30)])
    dst = torch.zeros(total, dtype=torch.uint8, device=DEV)
    scratch = torch.zeros(PAGE_SRC_DTYPE.itemsize + table.nbytes, dtype=torch.uint8, device=DEV)
    good = np.zeros(1, PAGE_SRC_DTYPE)
    good[0] = (page.data_ptr(), 90, 3, 1, 20, 30, 0, 0)
    host = torch.zeros(10, dtype=torch.uint8)

    def call(srcs, t=table, dst_bytes=total, scratch_bytes=scratch.numel()):
        return L.ytk_pack_pages_u8(srcs.ctypes.data, len(srcs), dst.data_ptr(), dst_bytes, t.ctypes.data,
                                   scratch.data_ptr(), scratch_bytes, None)

    torch.cuda.synchronize()
    launches = L.ytk_launch_count()
    for field, value, reason in (("H", 0, "empty"), ("sw", -3, "negative"), ("rgb", 2, "channel order"),
                                 ("H", 21, "page record"), ("data", host.data_ptr(), "device memory"),
                                 ("data", 0, "empty")):
        s = good.copy()
        s[0][field] = value
        assert call(s) != 0
        assert reason in L.ytk_last_error().decode(), (field, value)
    assert call(good, dst_bytes=total - 1) != 0                     # the page overruns the buffer
    assert call(good, scratch_bytes=scratch.numel() - 1) != 0
    assert "scratch" in L.ytk_last_error().decode()
    assert L.ytk_launch_count() == launches
    _lib.check(call(good))
    torch.cuda.synchronize()
    assert torch.equal(dst, page.reshape(-1))


# ------------------------------------------------------------------------------------------------------ module level
def _ocr(**rec):
    o = OCR(configs={"text_detector": {"from_pretrained": False},
                     "text_recognizer": {"from_pretrained": False, "model_name": "parseq-tiny-dynw-v4",
                                         "dynamic_width": True, "batch_bucketing": True, **rec}}, device="cuda")
    spec = ops.SPECS["parseq-tiny-dynw-v4"]
    o.recognizer.model.load_state_dict(weights.make_parseq_state_dict(spec, seed=11, peaked=True))
    load_trained_head(o.detector.model)
    return o


def _mixed(first, shapes=MIXED):
    return [synthetic_page(first + i, height=h, width=w)[0] for i, (h, w) in enumerate(shapes)]


def _dev(pages):
    return [torch.from_numpy(p).to(DEV) for p in pages]


def _words(r):
    return [(w.points, w.content, w.det_score, w.rec_score, w.direction) for w in r.words]


def _same_ocr(got, ref):
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        assert len(r.words) > 10
        assert _words(g) == _words(r)


def test_text_detector_device_page_equals_host_page():
    o = _ocr()
    pages = _mixed(400, MIXED[:3])
    det = o.detector
    for device_post in (True, False):
        det.device_post = device_post
        for p in pages:
            ref, _ = det(p)
            got, _ = det(torch.from_numpy(p).to(DEV))
            assert len(ref.points) > 10 and got.points == ref.points and got.scores == ref.scores
        ref = det.detect_pages(pages)
        got = det.detect_pages(device_pages(_dev(pages)))
        assert [g.points for g in got] == [r.points for r in ref] and [g.scores for g in got] == [r.scores for r in ref]


def test_ocr_device_page_equals_host_page():
    o = _ocr()
    for p in _mixed(410, MIXED[1:3]):
        _same_ocr([o(torch.from_numpy(p).to(DEV))[0]], [o(p)[0]])


@pytest.mark.parametrize("mode", ["plain", "fallback", "source-downscale"])
def test_batched_ocr_device_pages_equal_host_pages(mode):
    rec = {"fallback": {"rec_orientation_fallback": True, "rec_orientation_fallback_thresh": 0.9},
           "source-downscale": {"source_downscale": True}}.get(mode, {})
    o = _ocr(**rec)
    pages = _mixed(420)
    b = BatchedOCR(o.detector, o.recognizer, workers=2, det_batch=2)
    try:
        ref = b(pages)
        _same_ocr(b(_dev(pages)), ref)
        batches = [pages[0:2], pages[1:4]]
        ref_s = [b(pg) for pg in batches]
        got_s = list(b.stream([_dev(batches[0]), device_pages(_dev(batches[1]))]))
    finally:
        b.close()
    for g, r in zip(got_s, ref_s):
        _same_ocr(g, r)


def test_text_recognizer_host_crop_path_rejects_device_pages(monkeypatch):
    monkeypatch.setenv("YTK_DEVICE_CROPS", "0")
    rec = TextRecognizer(model_name="parseq-tiny-dynw-v4", from_pretrained=False, device="cuda")
    with pytest.raises(ValueError, match="device crop extraction"):
        rec(_rand(64, 96, 3, seed=8), [[[0, 0], [40, 0], [40, 20], [0, 20]]])


class _Table:
    def __init__(self, box, role=None):
        self.box, self.role = box, role


def _layout_analyzer():
    nop = {"from_pretrained": False}
    an = LayoutAnalyzer(configs={"layout_parser": nop, "table_structure_recognizer": nop}, device="cuda")
    an.layout_parser.model.load_state_dict(R.make_state_dict(R.SPECS["layout"], seed=11))
    an.table_structure_recognizer.model.load_state_dict(R.make_state_dict(R.SPECS["table"], seed=12))
    return an


def _dump(items):
    return [x.model_dump() for x in items]


def test_layout_analyzer_and_cell_detector_device_pages_equal_host_pages():
    an = _layout_analyzer()
    pages = _mixed(430, MIXED[1:4])
    assert _dump(an.analyze_pages(_dev(pages))) == _dump(an.analyze_pages(pages))
    assert an(torch.from_numpy(pages[0]).to(DEV))[0].model_dump() == an(pages[0])[0].model_dump()
    tables = [_Table([20, 10, 620, 184]), _Table([100, 300, 700, 560])]
    assert _dump(an.table_structure_recognizer(torch.from_numpy(pages[0]).to(DEV), [t.box for t in tables])[0]) == \
        _dump(an.table_structure_recognizer(pages[0], [t.box for t in tables])[0])
    cell = CellDetector(from_pretrained=False, device="cuda")
    assert _dump(cell(torch.from_numpy(pages[0]).to(DEV), tables)) == _dump(cell(pages[0], tables))


def _document_analyzer(**kw):
    cfg = {"ocr": {"text_detector": {"from_pretrained": False},
                   "text_recognizer": {"from_pretrained": False, "model_name": "parseq-tiny-dynw-v4",
                                       "dynamic_width": True, "batch_bucketing": True}},
           "layout_analyzer": {"layout_parser": {"from_pretrained": False},
                               "table_structure_recognizer": {"from_pretrained": False}}}
    an = DocumentAnalyzer(configs=cfg, device="cuda", **kw)
    load_trained_head(an.text_detector.model)
    return an


def test_document_analyzer_device_pages_equal_host_pages():
    an = _document_analyzer()
    pages = _mixed(440, MIXED[:3])
    try:
        assert an(torch.from_numpy(pages[1]).to(DEV))[0].model_dump() == an(pages[1])[0].model_dump()
        ref = an.analyze_pages(pages)
        assert all(len(r.words) > 10 for r in ref)
        assert _dump(an.analyze_pages(_dev(pages))) == _dump(ref)
    finally:
        an._batched.close()


def test_device_input_is_not_staged_or_uploaded(monkeypatch):
    from yomitoku_b200 import layout_analyzer, layout_parser
    from yomitoku_b200.models import RTDETRv2
    an = _document_analyzer()
    pages = _mixed(450, MIXED[1:3])
    ref = an.analyze_pages(pages)

    def forbidden(*a, **k):
        raise AssertionError("device input must not be staged or uploaded")
    for owner, name in ((BatchedOCR, "_stage"), (BatchedOCR, "_upload_pages"), (layout_parser, "upload_pages"),
                        (layout_analyzer, "upload_pages")):
        monkeypatch.setattr(owner, name, forbidden)
    seen = {"ocr": set(), "layout": set()}
    detect_chunk, forward_u8 = BatchedOCR._detect_chunk, RTDETRv2.forward_u8

    def spy_detect(self, stage, *a, **k):
        seen["ocr"].add(stage.data_ptr())
        return detect_chunk(self, stage, *a, **k)

    def spy_forward(self, pages, *a, **k):
        if self is an.layout.layout_parser.model:
            seen["layout"].add(pages.data_ptr())
        return forward_u8(self, pages, *a, **k)
    monkeypatch.setattr(BatchedOCR, "_detect_chunk", spy_detect)
    monkeypatch.setattr(RTDETRv2, "forward_u8", spy_forward)
    dp = device_pages(_dev(pages))
    try:
        got = an.analyze_pages(dp)
    finally:
        an._batched.close()
    assert _dump(got) == _dump(ref)
    assert seen["ocr"] == seen["layout"] == {dp.buf.data_ptr()}


def test_pages_written_on_a_side_stream():
    o = _ocr()
    pages = _mixed(460, MIXED[1:3])
    ref = [o.detector.detect_pages(pages), None]
    b = BatchedOCR(o.detector, o.recognizer, workers=2, det_batch=2)
    try:
        ref[1] = b(pages)
        host = [torch.from_numpy(p).pin_memory() for p in pages]
        side = torch.cuda.Stream()
        for k in range(2):
            with torch.cuda.stream(side):
                busy = torch.randn(8192, 8192, device=DEV)
                for _ in range(8):          # keeps the side stream busy while the host goes on
                    busy = torch.tanh(busy @ busy)
                dev = [torch.empty(p.shape, dtype=torch.uint8, device=DEV) for p in pages]
                for d, h in zip(dev, host):
                    d.copy_(h, non_blocking=True)
                if k == 0:
                    dp = device_pages(dev)
                    del dev                     # the caller may drop its tensors right away
                else:
                    got_s = list(b.stream([dev]))[0]
            if k == 0:
                got = o.detector.detect_pages(dp)
                assert [g.points for g in got] == [r.points for r in ref[0]]
                _same_ocr(b(dp), ref[1])
            else:
                _same_ocr(got_s, ref[1])
    finally:
        b.close()


def test_nvjpeg_decode_in_rgb_equals_host_path():
    tv = pytest.importorskip("torchvision.io")
    page = _mixed(470, [(900, 1200)])[0]
    data = tv.encode_jpeg(torch.from_numpy(np.ascontiguousarray(page[:, :, ::-1])).permute(2, 0, 1), quality=95)
    try:
        img = tv.decode_jpeg(data, device="cuda")
        torch.cuda.synchronize()
    except Exception as e:                       # no nvJPEG on this machine
        pytest.skip("decode_jpeg(device='cuda') unavailable: %s" % e)
    o = _ocr()
    host = np.ascontiguousarray(img.permute(1, 2, 0).cpu().numpy()[:, :, ::-1])
    got = o(device_pages([img.permute(1, 2, 0)], channel_order="rgb"))[0]
    _same_ocr([got], [o(host)[0]])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_pages_on_another_gpu_than_the_model():
    o = _ocr()
    page = torch.from_numpy(_mixed(480, [(600, 800)])[0]).to("cuda:1")
    for call in (lambda: o.detector(page), lambda: o.recognizer(page, [[[0, 0], [40, 0], [40, 20], [0, 20]]])):
        with pytest.raises(ValueError, match="cuda:1"):
            call()
