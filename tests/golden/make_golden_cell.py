"""Generates tests/golden/cell_ref.npz and tests/golden/cell_wrappers_ref.json from the reference's OWN files, executed
from /root/reference by path (build container only):

  cell_ref.npz              models/rtdetr.py (+ its layers) at the cell detector's configuration (6 classes, 1500
                            queries, 960 x 960; configs/cfg_table_cell_parser_rtdtrv2.py) with the seeded weights of
                            oracle.rtdetr.make_state_dict(CELL_SPEC) on a seeded table-like input: pred_logits /
                            pred_boxes, the backbone and encoder maps (4 x 4 block means), the 18,900 encoder scores and
                            the top-1500 anchors
  cell_wrappers_ref.json    table_cell_detector.py (CellDetector.preprocess / postprocess and the helpers it calls)
                            around the reference's postprocessor/rtdetr_postprocessor.py and utils/misc.py, fed with
                            seeded fake model outputs; modules it imports but this logic never executes (onnx*, base,
                            configs, models, logger, the semantic parser's schemas) are stand-ins.
Usage: python tests/golden/make_golden_cell.py
"""
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from oracle import refcheck as rc  # noqa: E402
from oracle import rtdetr as R  # noqa: E402

# the cell detector's model: RTDETRv2 with 6 classes, 1500 queries at 960 x 960 (reference
# configs/cfg_table_cell_parser_rtdtrv2.py); everything else as the layout models
CELL_SPEC = R.RTDETRSpec(num_classes=6, num_queries=1500, img_size=[960, 960])
CELL_SEED, CELL_XSEED = 13, 23
CATEGORIES = ["table", "cell", "header", "empty", "kv_item", "grid"]


def cell_input(seed, n=1, size=960):
    """Seeded table-crop-like input in [0, 1]: light background, dark ruling lines of an irregular grid, dark text-like
    blocks inside some cells (shared with the tests)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, 12, 12, generator=g)
    x = torch.nn.functional.interpolate(x, size=(size, size), mode="bilinear", align_corners=False) * 0.1 + 0.85
    for b in range(n):
        ys = sorted(set([0, size - 3] + torch.randint(40, size - 40, (7,), generator=g).tolist()))
        xs = sorted(set([0, size - 3] + torch.randint(40, size - 40, (5,), generator=g).tolist()))
        for y in ys:
            x[b, :, y:y + 3, :] = 0.1
        for c in xs:
            x[b, :, :, c:c + 3] = 0.1
        for _ in range(25):
            r, c = int(torch.randint(0, len(ys) - 1, (1,), generator=g)), int(torch.randint(0, len(xs) - 1, (1,), generator=g))
            y0, y1, x0, x1 = ys[r] + 8, ys[r + 1] - 8, xs[c] + 8, xs[c + 1] - 8
            if y1 - y0 > 8 and x1 - x0 > 16:
                h = int(min(y1 - y0, 24))
                w = int(torch.randint(8, x1 - x0, (1,), generator=g))
                x[b, :, y0:y0 + h, x0:x0 + w] = torch.rand(3, 1, 1, generator=g) * 0.3
    return x.contiguous()


def pooled4(t):
    """(1, C, H, W) -> (C, 4, 4) block means: a compact fingerprint of a feature map."""
    return torch.nn.functional.adaptive_avg_pool2d(t, 4)[0].numpy()


def build_reference_cell_model(sd):
    """The reference's RTDETRv2 with the cell detector's decoder settings (1500 queries, eval_spatial_size 960)."""
    RTDETRv2, _ = rc.load_reference_rtdetr()
    cfg = rc.reference_rtdetr_cfg(6)
    cfg["RTDETRTransformerv2"] = dict(cfg["RTDETRTransformerv2"], num_queries=1500, eval_spatial_size=[960, 960])
    m = RTDETRv2(cfg)
    m.load_state_dict(sd, strict=True)
    return m.eval()


def model_case():
    sd = R.make_state_dict(CELL_SPEC, seed=CELL_SEED)
    net = build_reference_cell_model(sd)
    x = cell_input(CELL_XSEED)
    with torch.no_grad():
        feats = net.backbone(x)
        enc = net.encoder(feats)
        res = net.decoder(enc)
        memory, _ = net.decoder._get_encoder_input(enc)
        om = net.decoder.enc_output(net.decoder.valid_mask.to(memory.dtype) * memory)
        scores = net.decoder.enc_score_head(om).max(-1).values[0]
    out = {"logits": res["pred_logits"][0].numpy(), "boxes": res["pred_boxes"][0].numpy(),
           "enc_scores": scores.numpy(), "topk": torch.topk(scores, 1500).indices.numpy().astype(np.int32)}
    for i in range(3):
        out["c%d" % (i + 3)] = pooled4(feats[i])
        out["e%d" % (i + 3)] = pooled4(enc[i])
    return out


# ------------------------------------------------------------------------------------------------ host wrappers
class _Table:
    def __init__(self, box, role=None):
        self.box, self.role = box, role


def _det(logits, boxes, q, cls, box, size, rng):
    """Query q detects `box` (crop pixels) as class cls with a score in (0.55, 0.98)."""
    w, h = size
    x1, y1, x2, y2 = box
    boxes[0, q] = ((x1 + x2) / 2 / w, (y1 + y2) / 2 / h, (x2 - x1) / w, (y2 - y1) / h)
    logits[0, q, cls] = rng.uniform(0.2, 4.0)


def cell_preds(seed, size, kind):
    """Fake (1, 1500, 6) model outputs for a crop of size (w, h).
      "grid":     a 7 x 5 grid of cells in the crop's top-left part (the right and bottom margins stay uncovered, so
                  the flood from (0, 0) - a covered pixel - keeps them as one hole without enough neighbours), a missing
                  cell with two header and two cell neighbours (a hole kept as "cell" by the tie rule), a cell and a
                  header covering the whole crop (dropped) beside a grid and a kv_item covering it (kept), an outer cell
                  around a smaller one, a header and an empty box inside cells, a noise-sized cell, a table box and a
                  partial kv_item
      "random":   a jittered grid with random roles, random missing cells (holes), a few nested boxes
      "fallback": only table / kv_item / grid detections: the whole table becomes one cell"""
    rng = np.random.default_rng(seed)
    logits = np.full((1, 1500, 6), -6.0, np.float32)
    boxes = rng.uniform(0.05, 0.95, (1, 1500, 4)).astype(np.float32)
    w, h = size
    q = 0

    def add(cls, box):
        nonlocal q
        _det(logits, boxes, q, cls, box, size, rng)
        q += 1

    if kind == "grid":
        cw, ch = (w - 80) // 7, (h - 80) // 5
        role = {(0, c): 2 for c in range(7)}                      # header row
        role.update({(2, 2): 2, (1, 3): 2, (2, 4): 1, (3, 3): 1, (4, 6): 3})
        for r in range(5):
            for c in range(7):
                if (r, c) == (2, 3) or (r, c) == (4, 0):
                    continue
                add(role.get((r, c), 1), (c * cw, r * ch, (c + 1) * cw, (r + 1) * ch))
        add(1, (0, 4 * ch, cw, 5 * ch))                           # outer cell around a smaller one: the outer goes
        add(1, (4, 4 * ch + 4, cw - 4, 5 * ch - 4))
        add(2, (1 * cw + 6, 3 * ch + 6, 2 * cw - 6, 4 * ch - 6))  # a header inside cell (3, 1): dropped
        add(3, (5 * cw + 6, 3 * ch + 6, 6 * cw - 6, 4 * ch - 6))  # an empty inside cell (3, 5): dropped
        add(1, (0, 0, w, h))                                      # covers the crop: dropped
        add(2, (1, 1, w - 1, h - 1))                              # covers the crop: dropped
        add(5, (0, 0, w, h))                                      # grid covering the crop: kept
        add(4, (0, 0, w, h))                                      # kv_item covering the crop: kept
        add(4, (cw, ch, 3 * cw, 2 * ch))
        add(0, (2, 2, w - 2, h - 2))
        add(1, (w - 60, h - 60, w - 52, h - 20))                  # 8 px wide: noise
    elif kind == "random":
        nr, nc = int(rng.integers(3, 7)), int(rng.integers(3, 6))
        xs = np.linspace(0, w, nc + 1).astype(int)
        ys = np.linspace(0, h, nr + 1).astype(int)
        for r in range(nr):
            for c in range(nc):
                if rng.random() < 0.15 and 0 < r < nr - 1 and 0 < c < nc - 1:
                    continue                                      # a hole
                j = rng.integers(-2, 3, 4)
                box = (max(0, xs[c] + j[0]), max(0, ys[r] + j[1]), min(w, xs[c + 1] + j[2]), min(h, ys[r + 1] + j[3]))
                add(int(rng.choice([1, 1, 1, 2, 3])), box)
                if rng.random() < 0.1:
                    add(int(rng.choice([1, 2, 3])), (box[0] + 5, box[1] + 5, box[2] - 5, box[3] - 5))
        if rng.random() < 0.5:
            add(5, (0, 0, w, h))
        add(4, (xs[0], ys[1], xs[min(2, nc)], ys[min(3, nr)]))
    else:
        add(0, (0, 0, w, h))
        add(4, (10, 10, w // 2, h // 2))
        add(5, (w // 3, h // 3, w - 5, h - 5))
    perm = rng.permutation(1500)                                  # detections anywhere in the query order
    return {"pred_logits": torch.from_numpy(logits[:, perm]), "pred_boxes": torch.from_numpy(boxes[:, perm])}


WRAPPER_CASES = [  # (seed, kind, table box on the 900 x 1200 page)
    (300, "grid", [100, 80, 740, 560]),
    (301, "grid", [0, 0, 600, 440]),
    (302, "random", [50, 300, 850, 900]),
    (303, "random", [200, 100, 700, 1150]),
    (304, "random", [0, 0, 900, 1200]),
    (305, "fallback", [120, 640, 520, 940]),
    (306, "random", [330, 20, 890, 420]),
]


def load_reference_cell_detector():
    import importlib.machinery
    from make_golden_rtdetr import load_reference_wrappers
    load_reference_wrappers()                 # utils.misc, the postprocessor and the common stand-ins

    def stub(name, **attrs):
        m = types.ModuleType(name)
        m.__spec__ = importlib.machinery.ModuleSpec(name, None)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
        return m

    class Schema(dict):
        def __init__(self, **kw):
            super().__init__(**kw)
            self.__dict__.update(kw)

    added = [n for n in ("onnx", "onnxruntime") if n not in sys.modules]
    for n in added:
        stub(n)
    sys.modules["ytk_ref.configs"].TableCellParserRTDETRv2Config = None
    schemas = rc._pkg("ytk_ref.schemas")
    stub("ytk_ref.schemas.table_semantic_parser", CellSchema=Schema, RegionSchema=Schema, TableDetectorSchema=Schema)
    schemas.table_semantic_parser = sys.modules["ytk_ref.schemas.table_semantic_parser"]
    try:
        return rc._load("ytk_ref.table_cell_detector", "table_cell_detector.py", "ytk_ref")
    finally:
        for n in added:
            sys.modules.pop(n, None)


def reference_cell_detector(mod):
    import torchvision.transforms as T
    d = object.__new__(mod.CellDetector)
    d.device, d.visualize, d.infer_onnx = "cpu", False, False
    d.postprocessor = mod.RTDETRPostProcessor(num_classes=6, num_top_queries=1500)
    d.transforms = T.Compose([T.Resize([960, 960]), T.ToTensor()])
    d.thresh_score = 0.5
    d.label_mapper = dict(enumerate(CATEGORIES))
    return d


def plain(obj):
    if isinstance(obj, dict):
        return {k: plain(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return [plain(v) for v in obj]
    if isinstance(obj, np.generic):
        return obj.item()
    return obj


def wrapper_cases():
    mod = load_reference_cell_detector()
    det = reference_cell_detector(mod)
    # record what the hole logic decided (the fixture must show kept and dropped holes and a tie resolved to "cell")
    calls = {"choose_role": [], "holes": []}
    choose, adjacent = mod.choose_role, mod.calc_adjacent_holes_to_cells

    def rec_choose(counts):
        r = choose(counts)
        calls["choose_role"].append({"counts": dict(counts), "role": r})
        return r

    def rec_adjacent(holes, cells):
        n = len(holes)
        kept = adjacent(holes, cells)
        calls["holes"].append([n, len(kept)])
        return kept

    mod.choose_role, mod.calc_adjacent_holes_to_cells = rec_choose, rec_adjacent
    page = np.random.default_rng(7).integers(0, 255, (1200, 900, 3), dtype=np.uint8)
    out = {"cases": [], "preprocess": []}
    for seed, kind, box in WRAPPER_CASES:
        data = det.preprocess(page, [_Table(box)])[0]
        preds = cell_preds(seed, (box[2] - box[0], box[3] - box[1]), kind)
        cells, kv, grid = det.postprocess(preds, data, box)
        out["cases"].append({"seed": seed, "kind": kind, "box": box, "size": list(data["size"]),
                             "offset": list(data["offset"]), "tensor_sum": float(data["tensor"].double().sum()),
                             "cells": plain([dict(c) for c in cells]), "kv_regions": plain([dict(r) for r in kv]),
                             "grid_regions": plain([dict(r) for r in grid])})
    out["preprocess_probe"] = det.preprocess(page, [_Table([37, 51, 611, 433])])[0]["tensor"][0, :, ::101, ::89].numpy().tolist()
    out["choose_role_calls"] = calls["choose_role"]
    out["hole_counts"] = calls["holes"]
    # the geometry helpers on seeded box pairs (utils/misc.py)
    misc = sys.modules["ytk_ref.utils.misc"]
    rng = np.random.default_rng(11)
    pairs = []
    for _ in range(400):
        a = rng.integers(0, 200, 2).tolist()
        a += [a[0] + int(rng.integers(1, 120)), a[1] + int(rng.integers(1, 120))]
        b = [a[2] + int(rng.integers(-20, 20)), a[1] + int(rng.integers(-60, 60))] if rng.random() < 0.5 else \
            [a[0] + int(rng.integers(-60, 60)), a[3] + int(rng.integers(-20, 20))]
        b += [b[0] + int(rng.integers(1, 120)), b[1] + int(rng.integers(1, 120))]
        pairs.append({"a": a, "b": b, "iou": misc.calc_iou(a, b), "right": misc.is_right_adjacent(a, b),
                      "bottom": misc.is_bottom_adjacent(a, b), "contained": misc.is_contained(a, b)})
    out["pairs"] = pairs
    return out


if __name__ == "__main__":
    np.savez_compressed(os.path.join(HERE, "cell_ref.npz"), **model_case())
    with open(os.path.join(HERE, "cell_wrappers_ref.json"), "w") as f:
        json.dump(wrapper_cases(), f)
    print("wrote cell_ref.npz, cell_wrappers_ref.json")
