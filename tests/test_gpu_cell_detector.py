"""GPU: the table cell detector - the top-k query selection kernel (ytk_op_topk_f32) against a stable sort, the RT-DETRv2
engine at the cell configuration (960 x 960, 1500 queries, 6 classes) against the fp32 oracle (oracle/rtdetr.py, pinned
to the reference's files by tests/test_cell_detector_host.py) and the reference-generated fixture
tests/golden/cell_ref.npz stage by stage, and CellDetector end to end.

Tolerances are those of tests/test_gpu_rtdetr.py (fp16 operands with fp32 accumulation against fp32), with the query
set scaled to 1500:
  backbone / encoder maps     relative Frobenius error < 0.5 %
  encoder scores              max |d| < 0.05; every anchor that only one side selected lies within 2 x 0.05 of the
                              oracle's cut, so at least 1500 - (oracle anchors within 2 x 0.05 of the cut) queries pair up
  paired queries              |d logit| < 0.1, mean < 0.02; |d box| < 0.003, mean < 0.0005
  detections                  every oracle detection with score > 0.6 is found with the same label and IoU > 0.9."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import rtdetr as R
from yomitoku_b200 import _lib
from yomitoku_b200.config import LayoutParserRTDETRv2V2Config, TableCellParserRTDETRv2Config, to_config
from yomitoku_b200.models import RTDETRv2

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_cell import CELL_SEED, CELL_SPEC, CELL_XSEED, cell_input, pooled4  # noqa: E402
from make_golden_rtdetr import rtdetr_input  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(HERE, "golden", "cell_ref.npz"))
SCORE_TOL = 0.05
K = 1500


# ------------------------------------------------------------------------------------------------ top-k kernel
def _keys(scores):
    """The kernel's monotone float -> unsigned map (so -0 < +0), as int64."""
    u = scores.view(np.uint32).astype(np.int64)
    return np.where(u & 0x80000000, 0xFFFFFFFF - u, u | 0x80000000)


def _stable_topk(scores, k):
    idx = np.arange(scores.shape[-1])
    return np.stack([np.lexsort((idx, -_keys(row)))[:k] for row in scores]).astype(np.int32)


def _device_topk(scores, k):
    s = torch.from_numpy(np.ascontiguousarray(scores, np.float32)).cuda()
    out = torch.full((s.shape[0], k), -1, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().ytk_op_topk_f32(s.data_ptr(), s.shape[0], s.shape[1], k, out.data_ptr(), None))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _scores(kind, n, L, rng):
    if kind == "random":
        return rng.standard_normal((n, L)).astype(np.float32)
    if kind == "quantised":                                   # 16 levels: long runs of equal scores
        return (rng.integers(0, 16, (n, L)) * 0.25 - 2.0).astype(np.float32)
    if kind == "equal":
        return np.full((n, L), -4.59512, np.float32)
    if kind == "zeros":                                       # -0 and +0 (distinct keys) and a few others
        s = np.where(rng.random((n, L)) < 0.5, np.float32(-0.0), np.float32(0.0)).astype(np.float32)
        s[:, rng.integers(0, L, 50)] = rng.standard_normal(50).astype(np.float32)
        return s
    if kind == "negative":                                    # large negative values, -inf, the lowest float
        s = -np.abs(rng.standard_normal((n, L))).astype(np.float32) * 1e30
        s[:, ::7] = -np.inf
        s[:, ::11] = np.finfo(np.float32).min
        s[:, ::13] = -3e38
        return s
    raise ValueError(kind)


@pytest.mark.parametrize("L,k", [(8400, 300), (18900, 1500)])
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("kind", ["random", "quantised", "equal", "zeros", "negative"])
def test_topk_equals_stable_sort(L, k, n, kind):
    scores = _scores(kind, n, L, np.random.default_rng(L + 7 * n + len(kind)))
    assert np.array_equal(_device_topk(scores, k), _stable_topk(scores, k))


@pytest.mark.parametrize("L,k", [(8400, 8400), (1000, 1000), (1000, 1), (5001, 777), (1023, 300), (1025, 1024)])
def test_topk_full_and_ragged_sizes(L, k):
    rng = np.random.default_rng(L + k)
    for kind in ("random", "quantised"):
        scores = _scores(kind, 2, L, rng)
        assert np.array_equal(_device_topk(scores, k), _stable_topk(scores, k))


def test_topk_refuses_what_does_not_fit():
    s = torch.zeros((1, 60000), dtype=torch.float32, device="cuda")
    out = torch.zeros((1, 300), dtype=torch.int32, device="cuda")
    for L, k in ((60000, 300), (1000, 1001), (1000, 0)):
        with pytest.raises(_lib.YtkError, match="topk"):
            _lib.check(_lib.lib().ytk_op_topk_f32(s.data_ptr(), 1, L, k, out.data_ptr(), None))
    torch.cuda.synchronize()                                   # nothing was launched: the context is intact
    scores = _scores("random", 1, 8400, np.random.default_rng(0))
    assert np.array_equal(_device_topk(scores, 300), _stable_topk(scores, 300))


# ------------------------------------------------------------------------------------------------ engine
def _model(cfg, sd):
    m = RTDETRv2(cfg=to_config(cfg()))
    m.load_state_dict(sd)
    return m.to("cuda")


def _rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def _iou(a, b):
    """a (4,), b (n, 4) cxcywh -> IoU (n,)."""
    a0, a1 = a[:2] - a[2:] / 2, a[:2] + a[2:] / 2
    b0, b1 = b[:, :2] - b[:, 2:] / 2, b[:, :2] + b[:, 2:] / 2
    wh = (np.minimum(a1, b1) - np.maximum(a0, b0)).clip(min=0)
    inter = wh[:, 0] * wh[:, 1]
    return inter / (a[2] * a[3] + b[:, 2] * b[:, 3] - inter)


def _check_topk_is_stable_order_of_scores(m, n):
    sc = m.debug_tensor(n, "enc.scores").reshape(n, -1)
    tk = m.debug_tensor(n, "topk").view(np.int32).reshape(n, -1)
    assert np.array_equal(tk, _stable_topk(sc, tk.shape[1]))
    return sc, tk


def _check_against_oracle(m, sd, x):
    n = x.shape[0]
    aux = {}
    ref = R.forward(sd, CELL_SPEC, x, aux)
    out = {k: v.cpu() for k, v in m(x.cuda()).items()}
    assert out["pred_logits"].shape == (n, K, 6) and out["pred_boxes"].shape == (n, K, 4)
    for i, name in enumerate(("c3", "c4", "c5")):
        assert _rel(m.debug_tensor(n, name).transpose(0, 3, 1, 2), aux["backbone"][i].numpy()) < 0.005, name
    for i, name in enumerate(("enc_out3", "enc_out4", "enc_out5")):
        assert _rel(m.debug_tensor(n, name).transpose(0, 3, 1, 2), aux["encoder"][i].numpy()) < 0.005, name
    sc_dev, tk = _check_topk_is_stable_order_of_scores(m, n)
    sc_ref = aux["enc_logits"].max(-1).values.numpy()
    assert sc_dev.shape == (n, 18900)
    assert np.abs(sc_dev - sc_ref).max() < SCORE_TOL
    for b in range(n):
        dev_set, ref_list = set(tk[b].tolist()), aux["topk"][b].tolist()
        assert len(dev_set) == K
        cut = np.sort(sc_ref[b])[-K]
        assert all(abs(sc_ref[b][a] - cut) < 2 * SCORE_TOL for a in dev_set ^ set(ref_list))
        pos = {a: i for i, a in enumerate(ref_list)}
        pairs = [(i, pos[a]) for i, a in enumerate(tk[b].tolist()) if a in pos]
        assert len(pairs) >= K - int((np.abs(sc_ref[b] - cut) < 2 * SCORE_TOL).sum())
        di, ri = [p[0] for p in pairs], [p[1] for p in pairs]
        dl = (out["pred_logits"][b][di] - ref["pred_logits"][b][ri]).abs()
        db = (out["pred_boxes"][b][di] - ref["pred_boxes"][b][ri]).abs()
        assert dl.max() < 0.1 and dl.mean() < 0.02, (float(dl.max()), float(dl.mean()))
        assert db.max() < 0.003 and db.mean() < 0.0005, (float(db.max()), float(db.mean()))
        s_ref, s_dev = torch.sigmoid(ref["pred_logits"][b]).numpy(), torch.sigmoid(out["pred_logits"][b]).numpy()
        boxes_dev = out["pred_boxes"][b].numpy()
        found = 0
        for q, c in zip(*np.nonzero(s_ref > 0.6)):
            if ref_list[q] not in dev_set:           # an anchor at the cut that the device did not select (checked above)
                continue
            ok = (s_dev[:, c] > 0.5) & (_iou(ref["pred_boxes"][b][q].numpy(), boxes_dev) > 0.9)
            assert ok.any(), (q, c)
            found += 1
        assert found > 0 or not (s_ref > 0.6).any()
    return out


@pytest.fixture(scope="module")
def cell_model():
    sd = R.make_state_dict(CELL_SPEC, seed=CELL_SEED)
    return sd, _model(TableCellParserRTDETRv2Config, sd)


def test_engine_at_960_matches_oracle_and_reference_fixture(cell_model):
    sd, m = cell_model
    assert (m.img_size, m.num_queries, m.num_classes) == (960, 1500, 6)
    _check_against_oracle(m, sd, cell_input(CELL_XSEED))
    for i in range(3):
        dev = pooled4(torch.from_numpy(m.debug_tensor(1, "c%d" % (i + 3)).transpose(0, 3, 1, 2).copy()))
        assert _rel(dev, GOLD["c%d" % (i + 3)]) < 0.005
        dev = pooled4(torch.from_numpy(m.debug_tensor(1, "enc_out%d" % (i + 3)).transpose(0, 3, 1, 2).copy()))
        assert _rel(dev, GOLD["e%d" % (i + 3)]) < 0.005
    sc = m.debug_tensor(1, "enc.scores").reshape(-1)
    assert np.abs(sc - GOLD["enc_scores"]).max() < SCORE_TOL
    cut = np.sort(GOLD["enc_scores"])[-K]
    tk = set(m.debug_tensor(1, "topk").view(np.int32).reshape(-1).tolist())
    assert all(abs(GOLD["enc_scores"][a] - cut) < 2 * SCORE_TOL for a in tk ^ set(GOLD["topk"].tolist()))


def test_batch_of_two_and_determinism(cell_model):
    """A batch of 2 gives, image by image, what single-image calls give; two runs return the same bits."""
    sd, m = cell_model
    x = cell_input(31, n=2)
    out = _check_against_oracle(m, sd, x)
    again = {k: v.cpu() for k, v in m(x.cuda()).items()}
    assert torch.equal(out["pred_logits"], again["pred_logits"]) and torch.equal(out["pred_boxes"], again["pred_boxes"])
    for i in range(2):
        one = {k: v.cpu() for k, v in m(x[i:i + 1]).items()}          # host input this time
        assert torch.allclose(one["pred_boxes"][0], out["pred_boxes"][i], atol=2e-3)
        assert torch.allclose(one["pred_logits"][0], out["pred_logits"][i], atol=5e-2)


def test_layout_model_topk_is_stable_order_of_its_scores():
    m = _model(LayoutParserRTDETRv2V2Config, R.make_state_dict(R.SPECS["layout"], seed=11))
    m(rtdetr_input(21, n=2).cuda())
    _, tk = _check_topk_is_stable_order_of_scores(m, 2)
    assert tk.shape == (2, 300)


# ------------------------------------------------------------------------------------------------ module API
class _Table:
    def __init__(self, box, role=None):
        self.box, self.role = box, role


def _table_page():
    """A white 1400 x 1100 page with three table crops of the seeded table input pasted in (BGR u8)."""
    import cv2
    page = np.full((1400, 1100, 3), 245, np.uint8)
    tables = [_Table([60, 80, 700, 560]), _Table([120, 640, 1040, 1000]), _Table([740, 60, 1060, 580])]
    for i, t in enumerate(tables):
        x1, y1, x2, y2 = t.box
        rgb = (cell_input(40 + i)[0].permute(1, 2, 0) * 255).to(torch.uint8).numpy()
        page[y1:y2, x1:x2] = cv2.resize(rgb, (x2 - x1, y2 - y1), interpolation=cv2.INTER_AREA)[:, :, ::-1]
    return page, tables


def test_cell_detector_end_to_end():
    """CellDetector on the device model: its detections equal the same post-processing of the oracle's outputs for
    detections away from the threshold (+-3 px), one page with three tables gives what three one-table calls give
    (+-1 px)."""
    from yomitoku_b200 import CellDetector
    from yomitoku_b200.schemas import TableDetectorSchema
    sd = R.make_state_dict(CELL_SPEC, seed=CELL_SEED)
    det = CellDetector(from_pretrained=False, device="cuda")
    det.model.load_state_dict(sd)
    page, tables = _table_page()
    data = det.preprocess(page, tables[:2])
    x = torch.cat([d["tensor"] for d in data])
    dev = det.model(x)
    ref = R.forward(sd, CELL_SPEC, x)
    for i, d in enumerate(data):
        h, w = d["size"]
        size = np.array([[w, h]], np.float32)
        got = det.postprocessor({k: v[i:i + 1] for k, v in dev.items()}, size, det.thresh_score)[0]
        want = det.postprocessor({k: v[i:i + 1] for k, v in ref.items()}, size, det.thresh_score - 0.05)[0]
        assert len(got["boxes"]) > 3
        # the device's detections are the oracle's (+-3 px), except for the few queries at the cut of the top-1500
        # selection that only one side selected
        near = [np.abs(want["boxes"] - b).max(axis=1).min() < 3.5 for b in got["boxes"]]
        assert sum(near) >= 0.9 * len(near), (sum(near), len(near))
    res = det(page, tables)
    assert len(res) == 3 and all(isinstance(r, TableDetectorSchema) for r in res)
    for r, t in zip(res, tables):
        assert r.box == t.box and len(r.cells) > 0
        assert all(t.box[0] - 3 <= c.box[0] and c.box[2] <= t.box[2] + 3 for c in r.cells)
    # three one-table calls: the same detections (+-1 px) for scores away from the threshold; where the device outputs
    # are the same bits, the same cells
    batch = det.model(torch.cat([d["tensor"] for d in det.preprocess(page, tables)]))
    for i, t in enumerate(tables):
        one = det.model(det.preprocess(page, [t])[0]["tensor"])
        h, w = t.box[3] - t.box[1], t.box[2] - t.box[0]
        size = np.array([[w, h]], np.float32)
        b_i = {k: v[i:i + 1] for k, v in batch.items()}
        for a, b in ((b_i, one), (one, b_i)):
            sure = det.postprocessor(a, size, det.thresh_score + 0.02)[0]
            loose = det.postprocessor(b, size, det.thresh_score - 0.02)[0]
            for box, lab in zip(sure["boxes"], sure["labels"]):
                d = np.abs(loose["boxes"] - box).max(axis=1)
                assert ((d <= 1) & (loose["labels"] == lab)).any()
        single = det(page, [t])
        if all(torch.equal(b_i[k], one[k]) for k in one):
            assert len(single) == 1 and [c.model_dump() for c in single[0].cells] == [c.model_dump() for c in res[i].cells]
