"""TableStructureRecognizer: RT-DETRv2 row / column / span detection on table crops, cells from their intersections.

Mirrors reference src/yomitoku/table_structure_recognizer.py:21-290 (catalog name `rtdetrv2`, constructor kwargs,
`preprocess` / `postprocess` / `extract_cell_elements` / `__call__`, TableStructureRecognizerSchema).  All table crops
of a page go through the device model as ONE batch (the reference runs them one by one); the geometry behind it is host
code like in the reference.
"""
import cv2
import numpy as np
import torch

from .base import BaseModelCatalog, BaseModule, logger
from .config import TableStructureRecognizerRTDETRv2Config
from .device_pages import DevicePages, as_device_pages, host_page, single_page
from .document_analyzer import _intersection, is_contained
from .layout_parser import filter_contained_rectangles_within_category, rtdetr_device_forward, rtdetr_input_tensor
from .models import RTDETRv2
from .postprocessor import RTDETRPostProcessor
from .schemas import TableStructureRecognizerSchema


class TableStructureRecognizerModelCatalog(BaseModelCatalog):
    def __init__(self):
        super().__init__()
        self.register("rtdetrv2", TableStructureRecognizerRTDETRv2Config, RTDETRv2)


def extract_cells(row_boxes, col_boxes):
    """One cell per intersecting (row, column) pair, numbered from 1 (reference table_structure_recognizer.py:28-47)."""
    cells = []
    for r, row in enumerate(row_boxes, 1):
        for c, col in enumerate(col_boxes, 1):
            box = _intersection(row, col)
            if box is not None:
                cells.append({"col": c, "row": r, "col_span": 1, "row_span": 1, "box": box, "contents": None})
    return cells


def filter_contained_cells_within_spancell(cells, span_boxes):
    """Cells inside a span box are replaced by one cell that covers their rows / columns (reference :50-88)."""
    children = [[cell for cell in cells if is_contained(span, cell["box"])] for span in span_boxes]
    swallowed = {id(cell) for group in children for cell in group}
    out = [cell for cell in cells if id(cell) not in swallowed]
    for span, group in zip(span_boxes, children):
        if not group:
            continue
        rows, cols = [c["row"] for c in group], [c["col"] for c in group]
        out.append({"col": min(cols), "row": min(rows), "col_span": max(cols) - min(cols) + 1,
                    "row_span": max(rows) - min(rows) + 1, "box": [int(v) for v in span], "contents": None})
    return sorted(out, key=lambda c: (c["row"], c["col"]))


class TableStructureRecognizer(BaseModule):
    model_catalog = TableStructureRecognizerModelCatalog()

    def __init__(self, model_name="rtdetrv2", path_cfg=None, device="cuda", visualize=False, from_pretrained=True,
                 infer_onnx=False):
        super().__init__()
        self.load_model(model_name, path_cfg, from_pretrained=from_pretrained)
        if infer_onnx:
            logger.warning("TableStructureRecognizer(infer_onnx=True): there is no ONNX path in yomitoku_b200, the CUDA "
                           "engine is used")
        self.infer_onnx = False
        self.device = device
        self.visualize = visualize
        self.model.eval().to(self.device)
        dec = self._cfg.RTDETRTransformerv2
        self.postprocessor = RTDETRPostProcessor(num_classes=dec.num_classes, num_top_queries=dec.num_queries)
        self.thresh_score = self._cfg.thresh_score
        self.label_mapper = dict(enumerate(self._cfg.category))

    def preprocess(self, img, boxes):
        """BGR page + table boxes -> per table {"tensor" (1,3,640,640), "size" (h, w), "offset" (x1, y1)}; :169-188."""
        rgb = cv2.cvtColor(img, cv2.COLOR_BGR2RGB)
        out = []
        for box in boxes:
            x1, y1, x2, y2 = (int(v) for v in box)
            crop = rgb[y1:y2, x1:x2, :]
            out.append({"tensor": rtdetr_input_tensor(np.ascontiguousarray(crop), self._cfg.data.img_size),
                        "size": crop.shape[:2], "offset": (x1, y1)})
        return out

    def postprocess(self, preds, data):
        h, w = data["size"]
        det = self.postprocessor(preds, np.array([[w, h]], np.float32), self.thresh_score)[0]
        ox, oy = data["offset"]
        elements = {c: [] for c in self.label_mapper.values()}
        for box, score, label in zip(det["boxes"], det["scores"], det["labels"]):
            x1, y1, x2, y2 = box.astype(int).tolist()
            elements[self.label_mapper[int(label)]].append({"box": [x1 + ox, y1 + oy, x2 + ox, y2 + oy],
                                                            "score": float(score)})
        elements = filter_contained_rectangles_within_category(elements)
        cells, rows, cols, spans = self.extract_cell_elements(elements)
        return TableStructureRecognizerSchema(box=[ox, oy, ox + w, oy + h], n_row=len(rows), n_col=len(cols), rows=rows,
                                              cols=cols, spans=spans, cells=cells, order=0)

    def extract_cell_elements(self, elements):
        rows = sorted(elements["row"], key=lambda e: e["box"][1])
        cols = sorted(elements["col"], key=lambda e: e["box"][0])
        spans = sorted(elements["span"], key=lambda e: e["box"][1])
        cells = extract_cells([e["box"] for e in rows], [e["box"] for e in cols])
        cells = filter_contained_cells_within_spancell(cells, [e["box"] for e in elements["span"]])
        return cells, rows, cols, spans

    def _infer(self, img, table_boxes, pages_dev=None):
        """(outputs on the host, per table {"size", "offset"}) for every table of the page in one batch: resized on the
        device when rtdetr_device_forward applies, else `preprocess` on the host."""
        boxes = [[int(v) for v in box] for box in table_boxes]
        pages = img if isinstance(img, DevicePages) else [img]
        dev = rtdetr_device_forward(self.model, pages, [(0, b) for b in boxes], pages_dev)
        if dev is not None:
            return dev[0], [{"size": s, "offset": (b[0], b[1])} for s, b in zip(dev[1], boxes)]
        data = self.preprocess(host_page(img), table_boxes)
        return self.model(torch.cat([d["tensor"] for d in data])), data

    def __call__(self, img, table_boxes, vis=None, pages_dev=None):
        """img: BGR page (numpy, or on the GPU: a CUDA (H, W, 3) uint8 tensor or a one-page DevicePages).  pages_dev
        (optional, numpy pages): `img` already on the device as upload_pages([img], ...) made it."""
        dp = as_device_pages(img)
        if dp is not None:
            img = single_page(dp, "TableStructureRecognizer")
        outputs = []
        if len(table_boxes):
            preds, data = self._infer(img, table_boxes, pages_dev)
            for i, d in enumerate(data):
                table = self.postprocess({k: v[i:i + 1] for k, v in preds.items()}, d)
                if table.n_row > 0 and table.n_col > 0:
                    outputs.append(table)
        if self.visualize:
            vis = host_page(img).copy() if vis is None else vis
            for table in outputs:
                vis = table_visualizer(vis, table)
        return outputs, vis


def table_visualizer(img, table):
    out = img.copy()
    for cell in table.cells:
        x1, y1, x2, y2 = cell.box
        cv2.rectangle(out, (x1, y1), (x2, y2), (255, 0, 255), 1)
    return out
