"""GPU: DBNet engine against the CPU oracle / reference-generated fixture.

Stated tolerances (bf16 activations through ~60 layers vs the fp32 reference, seeded random weights - the sigmoid
head of an untrained net amplifies noise, trained weights are smoother):
  backbone features  relative Frobenius error < 1.5 %
  probability map    mean |d| < 0.012, 99.5 % of the pixels within 0.08
  polygons           (a) the DEVICE'S OWN map of a detector with a trained head (tests/golden/dbnet_head_trained.npz: the
                     map holds the page's ~200 text lines) through the post-processor vs the fp32 oracle's own map
                     through the same post-processor: >= 95 % of the oracle's boxes with a score clear of box_thresh
                     are found with IoU >= 0.9 and corners within 2 px, >= 99 % with
                     IoU >= 0.5 (nothing lost / merged / split), box counts within 3 %;
                     (b) random head: the device's actual error field superimposed on a realistic probability map,
                     every box is found again with IoU >= 0.9 and corner coordinates within 2 px."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dbnet as odb
from oracle import pipeline as opipe
from oracle import weights
from yomitoku_b200 import TextDetector, _lib
from yomitoku_b200.postprocessor import DBnetPostProcessor
from yomitoku_b200.synth import synthetic_page, synthetic_prob_map

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def det():
    d = TextDetector(from_pretrained=False, device="cuda")
    d.model.load_state_dict(weights.make_dbnet_state_dict(seed=1))
    return d


def _debug(model, n, H, W, name):
    L = _lib.lib()
    shape = (ctypes.c_int * 4)()
    cap = n * H * W * 64 + 16
    buf = torch.empty(cap, dtype=torch.float32)
    _lib.check(L.ytk_dbnet_debug_tensor(model._ensure(), n, H, W, name.encode(), buf.data_ptr(), cap, shape))
    n_, h_, w_, c_ = list(shape)
    return buf[: n_ * h_ * w_ * c_].reshape(n_, h_, w_, c_)


def _prob_close(got, ref):
    d = np.abs(got - ref)
    print("[dbnet] prob map mean|d| %.5f, within 0.08: %.5f, max %.4f" % (d.mean(), (d < 0.08).mean(), d.max()))
    assert d.mean() < 0.012, d.mean()
    assert (d < 0.08).mean() > 0.995, (d < 0.08).mean()


def test_reference_fixture_through_model_seam():
    z = np.load(os.path.join(G, "dbnet_ref.npz"))
    d = TextDetector(from_pretrained=False, device="cuda")
    d.model.load_state_dict(weights.make_dbnet_state_dict(seed=int(z["weight_seed"])))
    out = d.model(torch.from_numpy(z["x"]))["binary"].numpy()
    assert out.shape == z["prob"].shape
    _prob_close(out, z["prob"])


def test_backbone_and_prob_vs_oracle(det):
    sd = det.model.state_dict()
    H, W = 256, 384
    x = torch.randn(2, 3, H, W, generator=torch.Generator().manual_seed(0))
    prob = det.model(x)["binary"]
    with torch.inference_mode():
        feats = odb.backbone_features(sd, x)
        ref = odb.decoder_forward(sd, feats)
    for k in ("layer1", "layer2", "layer3", "layer4"):
        got = _debug(det.model, 2, H, W, k)
        r = feats[k].permute(0, 2, 3, 1)
        print("[dbnet] %s rel Frobenius %.5f" % (k, ((got - r).norm() / r.norm()).item()))
        assert ((got - r).norm() / r.norm()).item() < 0.015, k
    _prob_close(prob.numpy(), ref.numpy())


def test_fused_u8_path_full_page_and_polygons(det):
    page, quads = synthetic_page(2)
    prob = det.model.detect_pages_u8(page)[0].numpy()
    assert prob.shape == (1184, 1600)
    x = opipe.detector_preprocess(page)
    ref = odb.dbnet_forward(det.model.state_dict(), x)[0, 0].numpy()
    _prob_close(prob, ref)
    # polygons: superimpose the device's error field on a realistic map of this page's boxes
    base = synthetic_prob_map(quads, (1184, 1600), (1200, 1600))
    pp = DBnetPostProcessor(**det._cfg.post_process)
    q_ref, s_ref = pp({"binary": base[None, None]}, (1200, 1600))
    q_dev, s_dev = pp({"binary": np.clip(base + (prob - ref), 0, 1)[None, None]}, (1200, 1600))
    assert len(q_ref) == len(quads) and len(q_dev) == len(q_ref)

    def rect(q):
        a = np.array(q)
        return a[:, 0].min(), a[:, 1].min(), a[:, 0].max(), a[:, 1].max()

    dev_r = np.array([rect(q) for q in q_dev], dtype=np.float64)
    for q in q_ref:
        r = np.array(rect(q), dtype=np.float64)
        ix = np.clip(np.minimum(dev_r[:, 2], r[2]) - np.maximum(dev_r[:, 0], r[0]), 0, None)
        iy = np.clip(np.minimum(dev_r[:, 3], r[3]) - np.maximum(dev_r[:, 1], r[1]), 0, None)
        inter = ix * iy
        union = (dev_r[:, 2] - dev_r[:, 0]) * (dev_r[:, 3] - dev_r[:, 1]) + (r[2] - r[0]) * (r[3] - r[1]) - inter
        j = int(np.argmax(inter / union))
        assert (inter / union)[j] >= 0.9
        assert np.abs(dev_r[j] - r).max() <= 2


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


@pytest.mark.parametrize("page_id", [2, 60])
def test_polygons_from_the_devices_own_map(page_id):
    """north_star: "detected polygons within a stated IoU/coordinate tolerance".  The detector carries the trained
    binarize head (seeded backbone / FPN), so its own probability map contains the page's text lines; the device's map
    and the fp32 oracle's map of the same weights go through the same post-processor and the polygons are compared."""
    from trained_head import load_trained_head
    d = TextDetector(from_pretrained=False, device="cuda")
    load_trained_head(d.model)
    page, quads = synthetic_page(page_id)
    prob = d.model.detect_pages_u8(page)[0].numpy()
    ref = odb.dbnet_forward(d.model.state_dict(), opipe.detector_preprocess(page))[0, 0].numpy()
    dd = np.abs(prob - ref)
    print("[dbnet trained head] prob map mean|d| %.5f max %.4f" % (dd.mean(), dd.max()))
    assert dd.mean() < 0.004, dd.mean()
    pp = DBnetPostProcessor(**d._cfg.post_process)
    q_ref, s_ref = pp({"binary": ref[None, None]}, page.shape[:2])
    q_dev, s_dev = pp({"binary": prob[None, None]}, page.shape[:2])
    assert len(q_ref) >= 150, len(q_ref)                       # the map is a real one: the page has 200 lines
    gt = _match(quads, q_ref)
    assert (gt[:, 0] > 0.5).sum() >= 170                       # ... and its boxes are the page's text lines
    assert abs(len(q_dev) - len(q_ref)) <= 0.03 * len(q_ref), (len(q_dev), len(q_ref))
    clear = np.asarray(s_ref) >= pp.box_thresh + 0.05
    m = _match(q_ref, q_dev)
    ok = (m[:, 0] >= 0.9) & (m[:, 1] <= 2)
    worst = sorted(((round(float(a), 3), float(b)) for a, b in m[clear & ~ok]), key=lambda t: t[0])
    print("[dbnet trained head] page %d: oracle %d boxes, device %d; %d of %d clear-score boxes found (IoU >= 0.9, 2 px); "
          "all boxes: %d of %d; (IoU, max corner distance) of the others: %s"
          % (page_id, len(q_ref), len(q_dev), int((ok & clear).sum()), int(clear.sum()), int(ok.sum()), len(ok), worst))
    # where the threshold cuts a blob edge with a shallow slope, a map
    # difference of 0.01-0.05 moves the edge by a pixel, which the unclip step scales up to a few pixels of the box
    assert (ok & clear).sum() >= 0.95 * clear.sum()
    assert ((m[:, 0] >= 0.5) & clear).sum() >= 0.99 * clear.sum()      # no box lost, merged or split away
    # the product call (device-side post-processing front half) returns exactly the polygons of the device's map
    res, _ = d(page)
    assert np.array_equal(np.asarray(res.points).reshape(-1, 4, 2), np.asarray(q_dev).reshape(-1, 4, 2))
    assert np.allclose(res.scores, s_dev)


def test_detector_call_contract(det):
    page, _ = synthetic_page(0)
    res, vis = det(page)
    assert vis is None and len(res.points) == len(res.scores)
    for q in res.points[:5]:
        assert len(q) == 4 and all(0 <= x <= 1600 and 0 <= y <= 1200 for x, y in q)
    # batched entry == single-page entry (same device code, batch dimension only)
    two = det.detect_pages([page, page])
    assert two[0].points == two[1].points
    # a page that needs up-scaling goes through the host resize + model seam like the reference
    small = np.ascontiguousarray(page[:300, :420])
    res2, _ = det(small)
    assert isinstance(res2.points, list)


def test_forward_is_deterministic(det):
    """Two forwards of the same pages return the same bits (the ASF channel means are summed in a fixed order), alone
    and as part of a larger batch."""
    pages = np.stack([synthetic_page(80 + i)[0] for i in range(3)])
    t = torch.from_numpy(pages).cuda()
    a = det.model.detect_pages_u8(t).cpu()
    b = det.model.detect_pages_u8(t).cpu()
    assert torch.equal(a, b)
    c = det.model.detect_pages_u8(t[1:2]).cpu()
    assert torch.equal(a[1:2], c)
