"""GPU: the device-side crop extraction (csrc/crop_ops.cu behind ytk_extract_crops_table_u8) - bit-exact against the crops the
reference's own data/functions.py cut (tests/golden/crops_ref.npz), against OpenCV through the host mirror
(yomitoku_b200.data.ParseqDataset), against the same arithmetic compiled for the host (oracle/crop_host.cpp), and end
to end: BatchedOCR / TextRecognizer with device_crops must return exactly what the host-crop path returns."""
import ctypes
import os
import sys
from types import SimpleNamespace as NS

import cv2
import numpy as np
import pytest
import torch

from yomitoku_b200 import data as D
from yomitoku_b200.models import extract_crops_device

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_crop_math import host_extract, random_quad  # noqa: E402

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CFG = NS(data=NS(img_size=[32, 800]))


def device_extract(pages_bgr, geoms):
    """pages_bgr: (n, H, W, 3) uint8; returns the canvases as host arrays (poison-filled buffer first)."""
    dev = torch.from_numpy(np.ascontiguousarray(pages_bgr)).cuda()
    canv, total = extract_crops_device(dev, geoms)
    torch.cuda.synchronize()
    host = canv.cpu().numpy()
    return [host[g["pix_off"]:g["pix_off"] + int(g["canvas_w"]) * int(g["canvas_h"]) * 3]
            .reshape(g["canvas_h"], g["canvas_w"], 3) for g in geoms]


def test_device_crops_match_reference_generated_crops():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden import crops_ref_page
    z = np.load(os.path.join(HERE, "golden", "crops_ref.npz"))
    page_bgr = np.ascontiguousarray(crops_ref_page()[:, :, ::-1])
    quads = z["quads"].tolist()
    n = 0
    for dyn, prefix in ((True, "dyn"), (False, "fixed")):
        geoms, keep = D.crop_geometry(page_bgr.shape, quads, [32, 800], dyn)
        got = device_extract(page_bgr[None], geoms)
        for i in range(len(quads)):
            key = "%s%d" % (prefix, i)
            if key in z.files:
                assert got[i].shape == z[key].shape and np.array_equal(got[i], z[key]), (key, quads[i])
                n += 1
    assert n == 48 + 6


def test_device_crops_match_opencv_and_host_build_on_random_quads():
    from oracle import build_crop_host
    lib = ctypes.CDLL(build_crop_host.build())
    cv2.setNumThreads(1)
    rng = np.random.default_rng(4242)
    H, W = 1200, 1600
    pages = rng.integers(0, 256, (3, H, W, 3), dtype=np.uint8)
    pages[1] = cv2.GaussianBlur(pages[1], (0, 0), 2.0)
    for dyn in (True, False):
        all_geoms, expect, same_math = [], [], []
        for pi in range(3):
            quads = [random_quad(rng, H, W, k % 6) for k in range(60)]
            quads.insert(5, [[-3, 5], [50, 5], [50, 30], [-3, 30]])       # dropped
            ds = D.ParseqDataset(CFG, pages[pi], quads, num_workers=1, dynamic_width=dyn)
            geoms, keep = D.crop_geometry(pages[pi].shape, quads, CFG.data.img_size, dyn, page=pi)
            assert len(geoms) == len(ds) == 60
            g0 = geoms.copy()
            g0["page"] = 0
            same_math += host_extract(lib, pages[pi], g0)
            all_geoms.append(geoms)
            expect += ds.data
        geoms = np.concatenate(all_geoms)
        got = device_extract(pages, geoms)          # one call for the crops of all three pages
        assert len(got) == len(expect) == 180
        for i, (a, b, c) in enumerate(zip(got, expect, same_math)):
            assert a.shape == b.shape and np.array_equal(a, c), ("device vs host build of crop_math.h", i)
            assert np.array_equal(a, b), ("device vs OpenCV", i, dict(w=int(geoms[i]["w"]), h=int(geoms[i]["h"]),
                                                                       rot=int(geoms[i]["rot"])))


def test_extract_crops_rejects_inconsistent_records():
    from yomitoku_b200 import _lib
    page = torch.zeros((1, 100, 200, 3), dtype=torch.uint8, device="cuda")
    geoms, _ = D.crop_geometry((100, 200), [[[10, 10], [60, 10], [60, 30], [10, 30]]], [32, 800], True)
    bad = geoms.copy()
    bad["rw"] = 500                                     # bounding box leaves the page
    with pytest.raises(_lib.YtkError):
        extract_crops_device(page, bad)
    with pytest.raises(ValueError):
        extract_crops_device(page.cpu(), geoms)


def _ocr():
    from oracle import parseq as ops
    from oracle import weights
    from yomitoku_b200 import OCR
    o = OCR(configs={"text_detector": {"from_pretrained": False},
                     "text_recognizer": {"from_pretrained": False, "model_name": "parseq-tiny-dynw-v4",
                                         "dynamic_width": True, "batch_bucketing": True}}, device="cuda")
    spec = ops.SPECS["parseq-tiny-dynw-v4"]
    o.recognizer.model.load_state_dict(weights.make_parseq_state_dict(spec, seed=11, peaked=True))
    return o


def test_batched_ocr_device_crops_equals_host_crops():
    """Whole path, both ways: canvases cut by OpenCV in the worker pool vs cut on the GPU from the resident pages; the
    recognizer sees identical bytes, so strings are identical and scores equal; stream() equals per-batch calls."""
    from yomitoku_b200.pipeline import BatchedOCR
    from yomitoku_b200.synth import synthetic_page, synthetic_prob_map
    o = _ocr()
    batches, overrides = [], []
    for k in range(4):
        pages, probs = [], []
        for i in range(2):
            p, q = synthetic_page(140 + 2 * k + i)
            pages.append(p)
            probs.append(synthetic_prob_map(q, (1184, 1600), (1200, 1600)))
        batches.append(pages)
        overrides.append(probs)
    host = BatchedOCR(o.detector, o.recognizer, workers=3, det_batch=2, device_crops=False)
    dev = BatchedOCR(o.detector, o.recognizer, workers=3, det_batch=2, device_crops=True)
    try:
        ref = [host(pg, prob_override=po) for pg, po in zip(batches, overrides)]
        got = [dev(pg, prob_override=po) for pg, po in zip(batches, overrides)]
        streamed = list(dev.stream(batches, lookahead=2, prob_override=overrides))
        single = BatchedOCR(o.detector, o.recognizer, workers=1, det_batch=2, device_crops=True)   # no worker pool
        inproc = single(batches[0], prob_override=overrides[0])
        single.close()
    finally:
        host.close()
        dev.close()
    for r, g, s in zip(ref, got, streamed):
        for pr, pg, ps in zip(r, g, s):
            assert len(pr.words) > 100
            assert [w.points for w in pr.words] == [w.points for w in pg.words] == [w.points for w in ps.words]
            assert [w.content for w in pr.words] == [w.content for w in pg.words] == [w.content for w in ps.words]
            assert np.allclose([w.rec_score for w in pr.words], [w.rec_score for w in pg.words], atol=1e-6)
    assert [[w.content for w in p.words] for p in inproc] == [[w.content for w in p.words] for p in ref[0]]


def test_recognizer_call_device_crops_equals_host_crops():
    from yomitoku_b200.synth import synthetic_page
    o = _ocr()
    page, quads = synthetic_page(3)
    rec = o.recognizer
    rec.device_crops = False
    a, _ = rec(page, quads[:90])
    rec.device_crops = True
    b, _ = rec(page, quads[:90])
    c, _ = rec(page, None)
    rec.device_crops = False
    d, _ = rec(page, None)
    assert a.contents == b.contents and a.directions == b.directions and np.allclose(a.scores, b.scores, atol=1e-6)
    assert c.contents == d.contents


def test_host_canvases_copy():
    """The page-locked host copy of device-cut canvases used for the cross-rank exchange (pipeline._HostCanvases)."""
    from yomitoku_b200.pipeline import _HostCanvases
    t = torch.arange(0, 100000, dtype=torch.int32, device="cuda").to(torch.uint8)
    s = torch.cuda.Stream()
    for st in (None, s):
        h = _HostCanvases(t, st)
        assert h.np.dtype == np.uint8 and np.array_equal(h.np, t.cpu().numpy())
