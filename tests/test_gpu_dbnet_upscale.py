"""GPU: pages that grow to the detector input, from the op up to the public API.

  op level   ytk_op_dbnet_preprocess_table_u8 (preprocess_kernel, AreaUpSampler) vs OpenCV's up-scaling tables of
             cv2.resize(INTER_AREA) (tests/test_dbnet_upscale_host.py: up_matrix, equal to cv2 within 1e-4 on the 0..255
             scale) applied in float64 as two separable matrices, / 255, mean / std by position.  The device value must
             be fp16(r) for some r within e of the reference.  Derivation of e (u = 2^-24): the kernel's weights (1 - f,
             f) are the reference's fp32 weights, so only the arithmetic errs.  The horizontal pass a p0 + b p1 over
             values <= 255 with a + b <= 1 + u costs at most 2 u 255; the vertical pass over two such values adds its
             own 2 u 255 and carries theirs, so the sum is off by at most 4 u 255, i.e. 4 u / 0.224 after / 255 and the
             division by std >= 0.224.  The normalisation in double with fp32 mean / std adds u 0.485 / 0.224 < 3 u
             and u |ref| for the rounded std, the cast to fp32 u |ref|.  So |d| <= 4 u / 0.224 + 2 u (|ref| + 3)
             (nx = ny = 2 taps in the decimation test's bound), and e takes twice that:
                 e = 2 ((nx + ny + 4) u / 0.224 + 2 u (|ref| + 3)),  nx = ny = 2.
             Away from the fp16 rounding midpoints only got == fp16(ref) passes.  Canvases are NaN-filled with one
             canvas more than the call writes, which must come back untouched; the border ring and channels 3..7 must
             be exactly 0.  Wrong variants the kernel must miss by >= 10x the tolerance: scale = s / n, INTER_LINEAR's
             half-pixel centres (each where its tables differ from OpenCV's; s / n differs on the two trap shapes) and
             mean / std applied to true RGB.
  engine     detect_pages_u8 on small pages (trained head) vs forward(preprocess(page)): the canvases may differ only
             next to fp16 rounding midpoints, and the engine's map is bitwise the seam's map of the op's own canvas;
             maps and quads are equal where the canvases are, else the boxes match as in test_gpu_dbnet.py (IoU >= 0.9
             and corners within 2 px for >= 95 % of the clear-score boxes, IoU >= 0.5 for >= 99 %, box counts within
             3 %).  TextDetector's entries never take the host seam.
  API        BatchedOCR (__call__ with and without device crops, stream) and DocumentAnalyzer.analyze_pages accept
             900x1200 and 720x1280 pages and equal the one-page calls.
"""
import cv2
import numpy as np
import pytest
import torch

from oracle import parseq as ops
from oracle import weights
from test_dbnet_upscale_host import SHAPE_IDS, SHAPES, TRAPS, same_tables, up_resize
from test_gpu_dbnet_kernels import U, _fp16_match, _normalise, _page, preprocess_pages
from yomitoku_b200 import OCR, DocumentAnalyzer, TextDetector
from yomitoku_b200.pipeline import BatchedOCR
from yomitoku_b200.synth import synthetic_page, synthetic_prob_map

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SMALL = [(900, 1200), (720, 1280)]


def _canvas_up(pages, Hn, Wn):
    """the op's canvases for pages [n, H0, W0, 3] u8, plus one NaN canvas past them -> numpy fp16 [n + 1, ...]"""
    canvas = torch.full((len(pages) + 1, Hn + 6, Wn + 8, 8), float("nan"), dtype=torch.float16, device=DEV)
    preprocess_pages(pages, Hn, Wn, canvas)
    return canvas.cpu().numpy()


def _e(ref):
    return 2 * ((2 + 2 + 4) * U / 0.224 + 2 * U * (np.abs(ref) + 3))


# ======================================================================================================== op level
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("hw,size", SHAPES, ids=SHAPE_IDS)
def test_preprocess_table_up_vs_float64(hw, size, n):
    (H0, W0), (Hn, Wn) = hw, size
    kinds = ("random",) if n == 1 else ("random", "gradient", "bright")
    pages = np.stack([_page(k, H0, W0, seed=H0 * 7 + W0 + i) for i, k in enumerate(kinds)])
    out = _canvas_up(pages, Hn, Wn)
    assert np.isnan(out[n]).all()                                 # nothing past the n canvases
    inner = np.zeros(out.shape[:3], dtype=bool)
    inner[:, 3:3 + Hn, 3:3 + Wn] = True
    assert (out[:n][~inner[:n]] == 0).all()                       # exactly zero border ring
    assert (out[:n, :, :, 3:] == 0).all()                         # exactly zero channels 3..7
    got = out[:n, 3:3 + Hn, 3:3 + Wn, :3]
    variants = [v for v in ("s_over_n", "linear") if not same_tables(H0, W0, Hn, Wn, v)]
    if (hw, size) in TRAPS:
        assert "s_over_n" in variants
    n_nb, misses = 0, {"true RGB": float("inf")}
    for i in range(n):
        area = up_resize(pages[i], Hn, Wn)
        ref = _normalise(area)
        e = _e(ref)
        ok, nb = _fp16_match(got[i], ref, e)
        n_nb += nb
        assert ok.all(), (i, kinds[i], int((~ok).sum()), np.argwhere(~ok)[:5])
        tol = 2.0 ** -11 * np.abs(ref) + e
        misses["true RGB"] = min(misses["true RGB"], float((np.abs(got[i] - _normalise(area, true_rgb=True)) / tol).max()))
        if kinds[i] == "random":
            for v in variants:
                misses[v] = float((np.abs(got[i] - _normalise(up_resize(pages[i], Hn, Wn, v))) / tol).max())
    print("[preprocess up] %dx%d -> %dx%d n %d: fp16(ref) exact except %d values next to a midpoint; wrong variants: %s"
          % (H0, W0, Hn, Wn, n, n_nb, ", ".join("%s %.0f x tol" % kv for kv in misses.items())))
    for v, m in misses.items():
        assert m >= 10.0, (v, m)


# ======================================================================================================== engine
@pytest.fixture(scope="module")
def det():
    from trained_head import load_trained_head
    d = TextDetector(from_pretrained=False, device="cuda")
    load_trained_head(d.model)
    return d


def _rects(qs):
    a = np.asarray(qs, dtype=np.float64).reshape(len(qs), 4, 2)
    return np.stack([a[:, :, 0].min(1), a[:, :, 1].min(1), a[:, :, 0].max(1), a[:, :, 1].max(1)], 1)


def _match(q_from, q_to):
    """For every box of q_from: (best IoU, max corner distance of the axis-aligned hulls) among q_to."""
    A, B = _rects(q_from), _rects(q_to)
    out = []
    for r in A:
        ix = np.clip(np.minimum(B[:, 2], r[2]) - np.maximum(B[:, 0], r[0]), 0, None)
        iy = np.clip(np.minimum(B[:, 3], r[3]) - np.maximum(B[:, 1], r[1]), 0, None)
        inter = ix * iy
        iou = inter / ((B[:, 2] - B[:, 0]) * (B[:, 3] - B[:, 1]) + (r[2] - r[0]) * (r[3] - r[1]) - inter)
        j = int(np.argmax(iou))
        out.append((iou[j], np.abs(B[j] - r).max()))
    return np.asarray(out)


def _small_page(seed, hw):
    """A synthetic page of the given small size whose text, once the detector input enlarges it, has about the size of
    the 1200 x 1600 pages the trained head was fitted on: a larger synthetic page shrunk with cv2 INTER_AREA."""
    big = {(900, 1200): (1200, 1600), (720, 1280): (900, 1600)}[hw]
    page, _ = synthetic_page(seed, height=big[0], width=big[1])
    return cv2.resize(page, (hw[1], hw[0]), interpolation=cv2.INTER_AREA)


@pytest.mark.parametrize("hw", SMALL, ids=["%dx%d" % hw for hw in SMALL])
def test_engine_u8_path_equals_host_seam_of_table_op(det, hw):
    """detect_pages_u8 (the engine runs the op's kernel on the same arguments) against the reference's way: the host
    resize + standardisation of TextDetector.preprocess through the model-level seam."""
    page = _small_page(70, hw)
    Hn, Wn = det.model.input_size(*hw)
    x = det.preprocess(page)                                      # (1, 3, Hn, Wn) fp32
    assert x.shape == (1, 3, Hn, Wn)
    host = x[0].permute(1, 2, 0).double().numpy()
    got = _canvas_up(page[None], Hn, Wn)[0, 3:3 + Hn, 3:3 + Wn, :3]
    # the host value is cv2's fp32 resize (within 1e-4 of the tables on the 0..255 scale) standardised in float64 and
    # rounded to fp32
    e = _e(host) + 1e-4 / 255 / 0.224 + U * np.abs(host)
    ok, _ = _fp16_match(got, host, e)
    n_diff = int((got != host.astype(np.float16)).sum())
    print("[engine up] %dx%d -> %dx%d: %d of %d canvas values differ from fp16(host preprocess), all next to a midpoint"
          % (hw[0], hw[1], Hn, Wn, n_diff, got.size))
    assert ok.all(), int((~ok).sum())
    prob_u8 = det.model.detect_pages_u8(page)[0].numpy()
    q_u8, s_u8 = det.postprocess({"binary": prob_u8[None, None]}, hw)
    # the engine reads exactly the op's canvas: the seam fed with the canvas values (the seam rounds its fp32 input to
    # the same fp16 canvas) returns the same bits
    x_op = torch.from_numpy(got.astype(np.float32)).permute(2, 0, 1)[None].contiguous()
    assert np.array_equal(prob_u8, det.model(x_op)["binary"][0, 0].numpy())
    prob_seam = det.model(x)["binary"][0, 0].numpy()
    q_seam, s_seam = det.postprocess({"binary": prob_seam[None, None]}, hw)
    pp = det.post_processor
    clear = np.asarray(s_seam) >= pp.box_thresh + 0.05
    m = _match(q_seam, q_u8) if len(q_u8) else np.zeros((len(q_seam), 2))
    good = (m[:, 0] >= 0.9) & (m[:, 1] <= 2)
    print("[engine up] host seam vs u8 path: map max |d| %.3g; %d / %d boxes; %d of %d clear-score boxes found (IoU >= "
          "0.9, 2 px), %d with IoU >= 0.5" % (np.abs(prob_u8 - prob_seam).max(), len(q_u8), len(q_seam),
                                              int((good & clear).sum()), int(clear.sum()),
                                              int(((m[:, 0] >= 0.5) & clear).sum())))
    assert len(q_seam) >= 100                                     # the map holds the page's text lines
    if n_diff == 0:
        assert np.array_equal(prob_u8, prob_seam)
        assert q_u8 == q_seam and s_u8 == s_seam
    else:
        # the matching of test_gpu_dbnet.py: a map difference near the threshold moves a blob edge by a pixel, which
        # the unclip step scales up to a few pixels of the box
        assert abs(len(q_u8) - len(q_seam)) <= 0.03 * len(q_seam), (len(q_u8), len(q_seam))
        assert (good & clear).sum() >= 0.95 * clear.sum()
        assert ((m[:, 0] >= 0.5) & clear).sum() >= 0.99 * clear.sum()
    # the public entries: the same boxes, with and without the device front half of the post-processing
    for device_post in (True, False):
        det.device_post = device_post
        try:
            res, _ = det(page)
            two = det.detect_pages([page, page])
        finally:
            det.device_post = True
        assert np.array_equal(np.asarray(res.points).reshape(-1, 4, 2), np.asarray(q_u8).reshape(-1, 4, 2))
        assert np.allclose(res.scores, s_u8)
        assert two[0].points == two[1].points == res.points


def test_detector_entries_skip_the_host_seam(det, monkeypatch):
    """TextDetector.__call__ and detect_pages on a small page run the device pre-processing: the host resize and the
    model-level seam are never called."""
    def boom(*a, **k):
        raise AssertionError("host seam called")
    page, _ = synthetic_page(71, height=720, width=1280)
    monkeypatch.setattr(det, "preprocess", boom)
    monkeypatch.setattr(det.model, "forward", boom)
    for device_post in (True, False):
        monkeypatch.setattr(det, "device_post", device_post)
        res, _ = det(page)
        assert len(res.points) == len(res.scores)
        assert len(det.detect_pages([page, page])) == 2


# ======================================================================================================== API
def _ocr():
    o = OCR(configs={"text_detector": {"from_pretrained": False},
                     "text_recognizer": {"from_pretrained": False, "model_name": "parseq-tiny-dynw-v4",
                                         "dynamic_width": True, "batch_bucketing": True}}, device="cuda")
    spec = ops.SPECS["parseq-tiny-dynw-v4"]
    o.recognizer.model.load_state_dict(weights.make_parseq_state_dict(spec, seed=11, peaked=True))
    return o


def _small_batch(o, hw, first, n):
    """n synthetic pages of size hw, their quads and stand-in probability maps at the up-scaled detector input"""
    size = o.detector.model.input_size(*hw)
    assert size[0] > hw[0] and size[1] > hw[1]
    pages, quads, probs = [], [], []
    for i in range(n):
        p, q = synthetic_page(first + i, height=hw[0], width=hw[1])
        pages.append(p)
        quads.append(q)
        probs.append(synthetic_prob_map(q, size, hw))
    return pages, quads, probs


@pytest.mark.parametrize("device_crops", [True, False], ids=["device-crops", "host-crops"])
@pytest.mark.parametrize("hw", SMALL, ids=["%dx%d" % hw for hw in SMALL])
def test_batched_ocr_small_pages_equal_per_page_calls(hw, device_crops):
    o = _ocr()
    pages, quads, probs = _small_batch(o, hw, 90, 3)
    b = BatchedOCR(o.detector, o.recognizer, workers=2, det_batch=2, device_crops=device_crops)
    try:
        res = b(pages, prob_override=probs)
    finally:
        b.close()
    assert len(res) == 3
    for i in range(3):
        assert len(res[i].words) == len(quads[i])
        det_points = [w.points for w in res[i].words]
        single, _ = o.recognizer(pages[i], det_points)
        assert [w.content for w in res[i].words] == single.contents
        assert np.allclose([w.rec_score for w in res[i].words], single.scores, atol=1e-6)


def test_stream_small_pages_equals_batched_calls():
    o = _ocr()
    batches, overrides = [], []
    for k in range(4):
        pages, _, probs = _small_batch(o, SMALL[k % 2], 100 + 2 * k, 2)
        batches.append(pages)
        overrides.append(probs)
    b = BatchedOCR(o.detector, o.recognizer, workers=3, det_batch=1)
    try:
        ref = [b(pg, prob_override=po) for pg, po in zip(batches, overrides)]
        got = list(b.stream(batches, lookahead=2, prob_override=overrides))
    finally:
        b.close()
    assert len(got) == len(ref) == 4
    for g, r in zip(got, ref):
        assert [[w.content for w in page.words] for page in g] == [[w.content for w in page.words] for page in r]
        assert [[w.points for w in page.words] for page in g] == [[w.points for w in page.words] for page in r]


def test_document_analyzer_small_pages():
    """analyze_pages on 900 x 1200 pages (one result per page, equal to the one-page calls); a stub layout analyzer
    without regions keeps the layout models out of it."""
    from trained_head import load_trained_head
    from yomitoku_b200 import schemas as S

    def layout(img):
        return S.LayoutAnalyzerSchema(paragraphs=[], tables=[], figures=[]), None

    cfg = {"ocr": {"text_detector": {"from_pretrained": False},
                   "text_recognizer": {"from_pretrained": False, "model_name": "parseq-tiny-dynw-v4",
                                       "dynamic_width": True, "batch_bucketing": True}}}
    an = DocumentAnalyzer(configs=cfg, device="cuda", layout_analyzer=layout)
    load_trained_head(an.text_detector.model)
    pages = [synthetic_page(110 + i, height=900, width=1200)[0] for i in range(2)]
    try:
        batched = an.analyze_pages(pages)
        single = [an(p)[0] for p in pages]
    finally:
        if an._batched is not None:
            an._batched.close()
    assert len(batched) == 2
    for a, b in zip(single, batched):
        assert len(b.words) > 0
        assert [w.points for w in a.words] == [w.points for w in b.words]
        assert [w.content for w in a.words] == [w.content for w in b.words]
