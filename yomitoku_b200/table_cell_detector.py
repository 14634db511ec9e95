"""CellDetector: RT-DETRv2 cell / header / empty / kv_item / grid detection on table crops at 960 x 960 with 1500 queries.

Mirrors reference src/yomitoku/table_cell_detector.py:34-522 (catalog name `rtdetrv2`, constructor kwargs, local
`weights_path` checkpoints, `preprocess` / `postprocess` / `extract_cell_elements` / `remove_noise_cells` /
`__call__`, TableDetectorSchema).  All table crops of a page go through the device model as ONE batch (the reference
runs them one by one); the geometry around it - containment filters, the holes between the detected cells and the
roles they inherit from their neighbours - is host code like in the reference.
"""
import os

import cv2
import numpy as np
import torch

from .base import BaseModelCatalog, BaseModule, logger
from .config import TableCellParserRTDETRv2Config, load_config
from .device_pages import as_device_pages, single_page
from .document_analyzer import calc_iou, is_bottom_adjacent, is_contained, is_right_adjacent
from .layout_parser import _area, filter_contained_rectangles_across_categories, rtdetr_device_forward, rtdetr_input_tensor
from .models import RTDETRv2
from .postprocessor import RTDETRPostProcessor
from .schemas import CellSchema, RegionSchema, TableDetectorSchema

__all__ = ["CellDetector", "TableParserModelCatalog", "filter_contained_rectangles_with_category",
           "filter_contained_rectangles_across_categories", "find_holes_as_rects", "choose_role",
           "calc_adjacent_holes_to_cells"]

_CELL_ROLES = ("cell", "header", "empty")


class TableParserModelCatalog(BaseModelCatalog):
    def __init__(self):
        super().__init__()
        self.register("rtdetrv2", TableCellParserRTDETRv2Config, RTDETRv2)


def filter_contained_rectangles_with_category(category_elements, ignore_categories=()):
    """Inside every category except `ignore_categories`, a box that CONTAINS another one (> 80 % of the other's area) is
    dropped; of two boxes that contain each other the larger one is dropped, the first on equal areas (reference
    table_cell_detector.py:41-75; every pair is judged on the original list)."""
    for category, elements in category_elements.items():
        if category in ignore_categories:
            continue
        boxes = [e["box"] for e in elements]
        keep = [True] * len(boxes)
        for i in range(len(boxes)):
            for j in range(i + 1, len(boxes)):
                j_in_i, i_in_j = is_contained(boxes[i], boxes[j]), is_contained(boxes[j], boxes[i])
                if j_in_i and i_in_j:
                    keep[j if _area(boxes[i]) > _area(boxes[j]) else i] = False
                elif j_in_i:
                    keep[i] = False
                elif i_in_j:
                    keep[j] = False
        category_elements[category] = [e for e, k in zip(elements, keep) if k]
    return category_elements


def find_holes_as_rects(table_shape, cell_boxes, pad=2, close_ksize=5, min_area=300):
    """Regions of the crop that no cell covers and that do not touch its border (reference :115-141): paint the cells
    black on a white (h, w) mask, open it with a close_ksize square three times, flood the background from (0, 0) and
    return the padded bounding boxes of the remaining white components with an area of at least min_area."""
    mask = np.full((table_shape[0], table_shape[1]), 255, np.uint8)
    for box in cell_boxes:
        x1, y1, x2, y2 = (int(v) for v in box)
        cv2.rectangle(mask, (x1, y1), (x2, y2), 0, thickness=-1)
    if close_ksize > 1:
        kernel = cv2.getStructuringElement(cv2.MORPH_RECT, (close_ksize, close_ksize))
        mask = cv2.morphologyEx(mask, cv2.MORPH_OPEN, kernel, iterations=3)
    holes = mask.copy()
    cv2.floodFill(holes, np.zeros((mask.shape[0] + 2, mask.shape[1] + 2), np.uint8), (0, 0), 0)
    contours, _ = cv2.findContours(holes, cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_SIMPLE)
    rects = []
    for c in contours:
        x, y, w, h = cv2.boundingRect(c)
        if w * h >= min_area:
            rects.append([x - pad, y - pad, x + w + pad, y + h + pad])
    return rects


def choose_role(role_counts):
    """The most frequent role; a tie that includes "cell" is "cell", any other tie the first in dict order (:144-155)."""
    if not role_counts:
        return None
    best = max(role_counts.values())
    tied = [r for r, n in role_counts.items() if n == best]
    if len(tied) > 1 and "cell" in tied:
        return "cell"
    return tied[0]


def calc_adjacent_holes_to_cells(holes, cells):
    """Keeps the holes that have cell neighbours in more than two of the four directions and gives each the role most
    of those neighbours have (reference :158-192)."""
    kept = []
    for hole in holes:
        sides = {"R": 0, "L": 0, "D": 0, "U": 0}
        roles = {r: 0 for r in _CELL_ROLES}
        for cell in cells:
            for side, hit in (("R", is_right_adjacent(hole["box"], cell["box"])),
                              ("L", is_right_adjacent(cell["box"], hole["box"])),
                              ("D", is_bottom_adjacent(hole["box"], cell["box"])),
                              ("U", is_bottom_adjacent(cell["box"], hole["box"]))):
                if hit:
                    sides[side] += 1
                    roles[cell["role"]] += 1
        if sum(n > 0 for n in sides.values()) > 2:
            hole["role"] = choose_role(roles)
            kept.append(hole)
    return kept


class CellDetector(BaseModule):
    model_catalog = TableParserModelCatalog()

    def __init__(self, model_name="rtdetrv2", path_cfg=None, device="cuda", visualize=False, from_pretrained=True,
                 infer_onnx=False):
        super().__init__()
        # a local training checkpoint (cfg weights_path) takes the place of the hub weights (reference :209-227)
        default_cfg, _ = self.model_catalog.get(model_name)
        weights_path = getattr(load_config(default_cfg, path_cfg), "weights_path", None)
        use_local = bool(weights_path) and os.path.exists(weights_path)
        self.load_model(model_name, path_cfg, from_pretrained=from_pretrained and not use_local)
        if use_local:
            self._load_local_weights(weights_path, getattr(self._cfg, "weights_key", "ema"))
        if infer_onnx:
            logger.warning("CellDetector(infer_onnx=True): there is no ONNX path in yomitoku_b200, the CUDA engine is used")
        self.infer_onnx = False
        self.device = device
        self.visualize = visualize
        self.model.eval().to(self.device)
        dec = self._cfg.RTDETRTransformerv2
        self.postprocessor = RTDETRPostProcessor(num_classes=dec.num_classes, num_top_queries=dec.num_queries)
        self.thresh_score = self._cfg.thresh_score
        self.label_mapper = dict(enumerate(self._cfg.category))

    def _load_local_weights(self, weights_path, weights_key="ema"):
        """An rtdetrv2_pytorch training checkpoint: ckpt["ema"]["module"], else ckpt["model"], else the dict itself;
        loaded non-strictly with warnings for missing and unexpected keys (reference :293-309)."""
        ckpt = torch.load(weights_path, map_location="cpu")
        if weights_key == "ema" and "ema" in ckpt:
            state = ckpt["ema"]["module"]
        elif "model" in ckpt:
            state = ckpt["model"]
        else:
            state = ckpt
        own = self.model.state_dict()
        missing = [k for k in own if k not in state]
        unexpected = [k for k in state if k not in own]
        self.model.load_state_dict(state, strict=False)
        if missing:
            logger.warning("Missing keys when loading local weights: %s", missing)
        if unexpected:
            logger.warning("Unexpected keys when loading local weights: %s", unexpected)
        logger.info("Loaded local cell-detector weights from %s", weights_path)

    def preprocess(self, img, tables):
        """BGR page + table elements -> per table {"tensor" (1, 3, 960, 960), "size" (h, w), "offset" (x1, y1)}
        (reference :311-328)."""
        rgb = cv2.cvtColor(img, cv2.COLOR_BGR2RGB)
        out = []
        for table in tables:
            x1, y1, x2, y2 = (int(v) for v in table.box)
            crop = rgb[y1:y2, x1:x2, :]
            out.append({"tensor": rtdetr_input_tensor(np.ascontiguousarray(crop), self._cfg.data.img_size),
                        "size": crop.shape[:2], "offset": (x1, y1)})
        return out

    def is_close_cell(self, box1, box2, threshold=10):
        """Both vertical or both horizontal edges of the two boxes are closer than threshold (reference :330-338)."""
        if abs(box1[0] - box2[0]) < threshold and abs(box1[2] - box2[2]) < threshold:
            return True
        return abs(box1[1] - box2[1]) < threshold and abs(box1[3] - box2[3]) < threshold

    def is_fully_contained(self, box1, box2, threshold=0.9):
        return calc_iou(box1, box2) >= threshold

    def postprocess(self, preds, data, table_box):
        """Detections of one crop -> (cells, kv_regions, grid_regions) in page coordinates (reference :344-450)."""
        h, w = data["size"]
        det = self.postprocessor(preds, np.array([[w, h]], np.float32), self.thresh_score)[0]
        elements = {c: [] for c in self.label_mapper.values()}
        elements["hole"] = []
        for box, score, label in zip(det["boxes"], det["scores"], det["labels"]):
            category = self.label_mapper[int(label)]
            box = box.astype(int).tolist()
            # a detection that covers the whole crop is dropped, except grid / kv_item (they may span the whole table)
            if category not in ("grid", "kv_item") and self.is_fully_contained(box, [0, 0, w, h]):
                continue
            elements[category].append({"box": box, "score": float(score), "role": category})
        elements = filter_contained_rectangles_with_category(elements, ignore_categories=("kv_item", "grid"))
        elements = filter_contained_rectangles_across_categories(elements, "cell", "header")
        elements = filter_contained_rectangles_across_categories(elements, "cell", "empty")
        cell_boxes = [e["box"] for c in _CELL_ROLES for e in elements[c]]
        for box in find_holes_as_rects(data["size"], cell_boxes):
            elements["hole"].append({"box": box, "score": 1.0, "role": "hole"})
        ox, oy = data["offset"]
        for group in elements.values():
            for e in group:
                e["box"] = [e["box"][0] + ox, e["box"][1] + oy, e["box"][2] + ox, e["box"][3] + oy]
        if not any(elements[c] for c in _CELL_ROLES):     # no cell at all: the whole table is one cell
            elements["cell"] = [{"box": table_box, "role": "cell"}]
        cells = self.remove_noise_cells(self.extract_cell_elements(elements), min_width=10, min_height=10)
        kv_regions = [RegionSchema(id=None, box=e["box"], role="kv_item", score=e["score"]) for e in elements["kv_item"]]
        grid_regions = [RegionSchema(id=None, box=e["box"], role="grid", score=e["score"]) for e in elements["grid"]]
        return cells, kv_regions, grid_regions

    def remove_noise_cells(self, cells, min_width=30, min_height=30):
        return [c for c in cells if c.box[2] - c.box[0] > min_width and c.box[3] - c.box[1] > min_height]

    def extract_cell_elements(self, elements):
        """Holes next to cells become cells with their neighbours' role; cells, headers, empties and kept holes (in that
        order) -> CellSchema with ids c0, c1, ... (reference :463-487)."""
        elements["hole"] = calc_adjacent_holes_to_cells(elements["hole"], [e for c in _CELL_ROLES for e in elements[c]])
        cells = []
        for category, values in elements.items():
            if category in ("cell", "header", "empty", "group", "hole"):
                for v in values:
                    cells.append(CellSchema(id="c%d" % len(cells), box=v["box"], role=v["role"], contents=None, row=None,
                                            col=None, row_span=None, col_span=None))
        return cells

    def __call__(self, img, tables):
        """BGR page (numpy, or on the GPU: a CUDA (H, W, 3) uint8 tensor or a one-page DevicePages) + the layout
        parser's tables -> List[TableDetectorSchema], tables without cells left out."""
        outputs = []
        if not tables:
            return outputs
        dp = as_device_pages(img)
        # every table of the page in one batch, resized on the device when rtdetr_device_forward applies
        boxes = [[int(v) for v in table.box] for table in tables]
        pages = [img] if dp is None else single_page(dp, "CellDetector")
        dev = rtdetr_device_forward(self.model, pages, [(0, b) for b in boxes])
        if dev is not None:
            preds, data = dev[0], [{"size": s, "offset": (b[0], b[1])} for s, b in zip(dev[1], boxes)]
        else:
            data = self.preprocess(img if dp is None else dp.numpy(0), tables)
            preds = self.model(torch.cat([d["tensor"] for d in data]))
        for i, (d, table) in enumerate(zip(data, tables)):
            cells, kv_regions, grid_regions = self.postprocess({k: v[i:i + 1] for k, v in preds.items()}, d, table.box)
            if not cells:
                continue
            outputs.append(TableDetectorSchema(id=None, box=table.box, role=table.role, cells=cells,
                                               kv_regions=kv_regions, grid_regions=grid_regions))
        return outputs

    def detect_pages(self, pages, tables_per_page):
        """Batched entry (new surface): `__call__` for many pages with ONE model forward over the table crops of all of
        them.  pages: a DevicePages or a list of BGR numpy pages; tables_per_page: the layout parser's tables of each
        page.  Returns a list (per page) of List[TableDetectorSchema], equal to `__call__(page, tables)` per page."""
        recs = [(i, [int(v) for v in t.box]) for i, tables in enumerate(tables_per_page) for t in tables]
        out = [[] for _ in tables_per_page]
        if not recs:
            return out
        dp = as_device_pages(pages)
        dev = rtdetr_device_forward(self.model, dp if dp is not None else pages, recs)
        if dev is not None:
            preds, data = dev[0], [{"size": s, "offset": (b[0], b[1])} for s, (_, b) in zip(dev[1], recs)]
        else:
            data = [d for i, tables in enumerate(tables_per_page) if tables
                    for d in self.preprocess(dp.numpy(i) if dp is not None else pages[i], tables)]
            preds = self.model(torch.cat([d["tensor"] for d in data]))
        tables = [t for ts in tables_per_page for t in ts]
        for k, ((i, _), d, table) in enumerate(zip(recs, data, tables)):
            cells, kv_regions, grid_regions = self.postprocess({n: v[k:k + 1] for n, v in preds.items()}, d, table.box)
            if cells:
                out[i].append(TableDetectorSchema(id=None, box=table.box, role=table.role, cells=cells,
                                                  kv_regions=kv_regions, grid_regions=grid_regions))
        return out
