"""GPU: the side paths of the device-side crop extraction - the orientation fallback's 180-degree second look (record
bit `rot & 2`) and the source_downscale pyramid (ytk_halve_pages_table_u8) - against OpenCV and against the host-crop path of
TextRecognizer / BatchedOCR.  (Sorted after the other GPU test files on purpose: these kernels' arithmetic is pinned on
the CPU by tests/test_crop_math.py; this file adds the end-to-end equalities.)"""
import os
import sys

import cv2
import numpy as np
import pytest
import torch

from yomitoku_b200 import data as D

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_crop_math import random_quad  # noqa: E402
from test_gpu_crops import CFG, _ocr, device_extract  # noqa: E402

pytestmark = pytest.mark.gpu


def test_device_orientation_fallback_crops_match_opencv():
    """Record bit `rot & 2` (the orientation fallback's 180-degree second look on the fixed canvas)."""
    cv2.setNumThreads(1)
    rng = np.random.default_rng(78)
    H, W = 900, 1400
    page = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    quads = [random_quad(rng, H, W, k % 6) for k in range(36)]
    ds = D.ParseqDataset(CFG, page, quads, num_workers=1, dynamic_width=True)
    geoms, keep = D.crop_geometry(page.shape, quads, CFG.data.img_size, True)
    geoms["rot"] |= 2
    geoms["canvas_w"] = CFG.data.img_size[1]
    for got, roi in zip(device_extract(page[None], geoms), ds.roi_images):
        assert np.array_equal(got, D.resize_with_padding(cv2.rotate(roi, cv2.ROTATE_180), CFG.data.img_size))


def test_pyramid_levels_match_opencv_through_tables():
    """ytk_halve_pages_table_u8 == cv2.resize(page, None, fx=0.5, fy=0.5, INTER_AREA), level after level, odd sizes
    included; the first level from a same-size (2, H, W, 3) batch, the next ones from the returned page table."""
    from yomitoku_b200.models import halve_pages_device
    cv2.setNumThreads(1)
    rng = np.random.default_rng(31)
    for H, W in ((1200, 1600), (1199, 1597), (37, 53), (2, 3)):
        pages = rng.integers(0, 256, (2, H, W, 3), dtype=np.uint8)
        dev = torch.from_numpy(pages).cuda()
        host = [pages[0], pages[1]]
        for level in range(3):
            if min(host[0].shape[:2]) < 2:
                break
            dev = halve_pages_device(dev)
            host = [cv2.resize(h, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_AREA) for h in host]
            flat, table = dev
            got = flat.cpu().numpy()
            assert [(int(t["H"]), int(t["W"])) for t in table] == [h.shape[:2] for h in host]
            for t, h in zip(table, host):
                o = int(t["page_off"])
                assert np.array_equal(got[o:o + h.size].reshape(h.shape), h)


def test_recognizer_side_paths_device_crops_equal_host_crops():
    from yomitoku_b200.synth import synthetic_page
    o = _ocr()
    page, quads = synthetic_page(3)
    rec = o.recognizer
    # orientation fallback: every crop scoring below the threshold takes the 180-degree second look on both paths;
    # identical canvases -> identical decisions and results
    rec.rec_orientation_fallback, rec.rec_orientation_fallback_thresh = True, 0.9
    rec.device_crops = False
    e, _ = rec(page, quads[:40])
    rec.device_crops = True
    f, _ = rec(page, quads[:40])
    rec.rec_orientation_fallback, rec.device_crops = False, False
    assert e.contents == f.contents and np.allclose(e.scores, f.scores, atol=1e-6)
    # source_downscale: big lines are cut from pyramid levels 2 / 1 / 1 (the last one is vertical text), odd page size
    big = [[[100, 100], [900, 100], [900, 240], [100, 240]], [[50, 300], [700, 300], [700, 370], [50, 370]],
           [[1000, 100], [1100, 100], [1100, 900], [1000, 900]]]
    odd = np.ascontiguousarray(page[:1199, :1597])
    rec.source_downscale = True
    g, _ = rec(odd, quads[:20] + big)
    rec.device_crops = True
    h, _ = rec(odd, quads[:20] + big)
    rec.source_downscale, rec.device_crops = False, False
    assert g.contents == h.contents and np.allclose(g.scores, h.scores, atol=1e-6)


def test_batched_ocr_device_crops_with_source_downscale():
    """BatchedOCR with source_downscale: big lines come from pyramid levels built on the GPU for the whole batch; the
    result must equal the host-crop path (OpenCV pyramid in the workers)."""
    from yomitoku_b200.pipeline import BatchedOCR
    from yomitoku_b200.synth import synthetic_page
    o = _ocr()
    o.recognizer.source_downscale = True
    big = [[[100, 100], [900, 100], [900, 240], [100, 240]], [[50, 300], [700, 300], [700, 370], [50, 370]],
           [[1000, 100], [1100, 100], [1100, 900], [1000, 900]]]
    pages, quads = [], []
    for i in range(3):
        p, q = synthetic_page(160 + i)
        pages.append(p)
        quads.append(q[:25] + big[i:] + q[25:40])
    host = BatchedOCR(o.detector, o.recognizer, workers=2, det_batch=2, device_crops=False)
    dev = BatchedOCR(o.detector, o.recognizer, workers=2, det_batch=2, device_crops=True)
    try:
        ref = host(pages, quads_override=quads)
        got = dev(pages, quads_override=quads)
    finally:
        host.close()
        dev.close()
        o.recognizer.source_downscale = False
    for r, g, q in zip(ref, got, quads):
        assert len(r.words) == len(g.words) == len(q)
        assert [w.content for w in r.words] == [w.content for w in g.words]
        assert np.allclose([w.rec_score for w in r.words], [w.rec_score for w in g.words], atol=1e-6)


def test_batched_ocr_orientation_fallback_equals_per_page_calls():
    """BatchedOCR honours rec_orientation_fallback (the batch takes the device-crops path, the second look is the same
    record with `rot |= 2`): per page identical to TextRecognizer.__call__ on the host path with the fallback on."""
    from yomitoku_b200.pipeline import BatchedOCR
    from yomitoku_b200.synth import synthetic_page
    o = _ocr()
    rec = o.recognizer
    rec.rec_orientation_fallback, rec.rec_orientation_fallback_thresh = True, 0.9
    pages, quads = [], []
    for i in range(2):
        p, q = synthetic_page(170 + i)
        pages.append(p)
        quads.append(q[:60])
    b = BatchedOCR(o.detector, rec, workers=2, det_batch=2)
    try:
        got = b(pages, quads_override=quads)
    finally:
        b.close()
    for i in range(2):
        rec.device_crops = False
        single, _ = rec(pages[i], quads[i])
        assert [w.content for w in got[i].words] == single.contents
        assert np.allclose([w.rec_score for w in got[i].words], single.scores, atol=1e-6)
    rec.rec_orientation_fallback = False
