"""LayoutParser: RT-DETRv2 page-layout detection behind the reference's module API.

Mirrors reference src/yomitoku/layout_parser.py:23-274 - same catalog names (`rtdetrv2`, `rtdetrv2v2`), constructor
kwargs, `preprocess` / `postprocess` / `filtering_elements` / `__call__` contract and result schema.  The model forward
runs as sm_90a kernels (csrc/rtdetr_engine.cu).  On a CUDA device the page goes up as u8 and the PIL resize in front of
the model runs there too, bit for bit (csrc/resample_ops.cu behind ytk_rtdetr_forward_u8, shared with the table
structure recognizer and the cell detector through `rtdetr_device_forward`); `preprocess` stays the host form of it.
The containment filters behind the model are host code like in the reference.  `infer_onnx` is accepted and ignored.
"""
import cv2
import numpy as np
import torch
from PIL import Image

from . import _lib
from .base import BaseModelCatalog, BaseModule, logger
from .config import LayoutParserRTDETRv2Config, LayoutParserRTDETRv2V2Config
from .document_analyzer import is_contained
from .models import RTDETRv2
from .postprocessor import RTDETRPostProcessor
from .schemas import LayoutParserSchema


class LayoutParserModelCatalog(BaseModelCatalog):
    def __init__(self):
        super().__init__()
        self.register("rtdetrv2", LayoutParserRTDETRv2Config, RTDETRv2)
        self.register("rtdetrv2v2", LayoutParserRTDETRv2V2Config, RTDETRv2)


def _area(box):
    return (box[2] - box[0]) * (box[3] - box[1])


def filter_contained_rectangles_within_category(category_elements):
    """Inside every category: a box that lies (> 80 % of its area) inside another one is dropped; of two boxes that
    contain each other the one that is NOT larger is dropped (reference layout_parser.py:31-61; every pair is judged
    on the original list, a box already dropped still eliminates others)."""
    for category, elements in category_elements.items():
        boxes = [e["box"] for e in elements]
        keep = [True] * len(boxes)
        for i in range(len(boxes)):
            for j in range(i + 1, len(boxes)):
                j_in_i, i_in_j = is_contained(boxes[i], boxes[j]), is_contained(boxes[j], boxes[i])
                if j_in_i and i_in_j:
                    keep[j if _area(boxes[i]) > _area(boxes[j]) else i] = False
                elif j_in_i:
                    keep[j] = False
                elif i_in_j:
                    keep[i] = False
        category_elements[category] = [e for e, k in zip(elements, keep) if k]
    return category_elements


def filter_contained_rectangles_across_categories(category_elements, source, target):
    """`target` boxes that lie inside any `source` box are dropped (reference layout_parser.py:64-78)."""
    sources = [e["box"] for e in category_elements[source]]
    category_elements[target] = [e for e in category_elements[target]
                                 if not any(is_contained(s, e["box"]) for s in sources)]
    return category_elements


def rtdetr_input_tensor(rgb, img_size):
    """What the reference's `T.Compose([T.Resize(img_size), T.ToTensor()])` makes of an RGB uint8 array: PIL bilinear
    (antialiased) resize to (h, w) = img_size, then CHW float32 / 255, with a batch axis."""
    h, w = int(img_size[0]), int(img_size[1])
    small = np.asarray(Image.fromarray(rgb).resize((w, h), Image.BILINEAR), dtype=np.uint8)
    return torch.from_numpy(np.ascontiguousarray(small.transpose(2, 0, 1))).to(torch.float32).div(255)[None]


RTDETR_SRC_DTYPE = np.dtype(_lib.YtkRtdetrSrc)


def rtdetr_sources(page_shapes, boxes):
    """Model inputs of RTDETRv2.forward_u8: page_shapes are the (h, w, ...) shapes of the pages packed back to back,
    boxes are (page index, (x1, y1, x2, y2)) pairs.  Each box is read as the modules read it, `int(v)` per coordinate,
    with numpy slicing semantics: `rgb[y1:y2, x1:x2]`, x2 / y2 clamped to the page.  Returns (records, sizes), sizes[i]
    = (h, w) of that crop (its `crop.shape[:2]`), or None when numpy would not make a plain crop of some box (a
    negative coordinate wraps around, or the crop is empty): the caller then takes the host path for the whole call."""
    offs, off = [], 0
    for shape in page_shapes:
        offs.append(off)
        off += int(shape[0]) * int(shape[1]) * 3
    recs = np.zeros(len(boxes), RTDETR_SRC_DTYPE)
    sizes = []
    for i, (p, box) in enumerate(boxes):
        H, W = int(page_shapes[p][0]), int(page_shapes[p][1])
        x1, y1, x2, y2 = (int(v) for v in box)
        if min(x1, y1, x2, y2) < 0:
            return None
        x2, y2 = min(x2, W), min(y2, H)
        if x1 >= x2 or y1 >= y2:
            return None
        recs[i] = (offs[p], H, W, x1, y1, x2, y2)
        sizes.append((y2 - y1, x2 - x1))
    return recs, sizes


def upload_pages(pages, model):
    """BGR u8 pages -> one flat uint8 tensor on `model`'s CUDA device, pages back to back (what forward_u8 reads), so
    that several RT-DETRv2 models read one upload.  None when the device path does not apply: the model is not on a
    CUDA device, or a page is not a non-empty (h, w, 3) uint8 array."""
    if model._device.type != "cuda" or not torch.cuda.is_available() or not pages:
        return None
    for p in pages:
        if not (isinstance(p, np.ndarray) and p.dtype == np.uint8 and p.ndim == 3 and p.shape[2] == 3 and p.size):
            return None
    flat = np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in pages])
    return torch.from_numpy(flat).to(model.cuda_device())


def rtdetr_device_forward(model, pages, boxes, pages_dev=None):
    """The device path of the three RT-DETRv2 modules: `model`'s outputs (on the host) for the crops `boxes` (page
    index, box) of the BGR u8 `pages`, resized on the device, and the crop sizes.  pages_dev: those pages as
    upload_pages made them (shared with another model), else they are uploaded here.  None when the device path does
    not apply (upload_pages, rtdetr_sources): the caller then runs `model(torch.cat(preprocess(...)))`, which gives the
    same bits."""
    if model._device.type != "cuda" or not torch.cuda.is_available():
        return None
    src = rtdetr_sources([p.shape for p in pages], boxes)
    if src is None:
        return None
    if pages_dev is None or pages_dev.device != model.cuda_device():
        pages_dev = upload_pages(pages, model)
        if pages_dev is None:
            return None
    recs, sizes = src
    preds = model.forward_u8(pages_dev, recs)
    return {k: v.cpu() for k, v in preds.items()}, sizes


class LayoutParser(BaseModule):
    model_catalog = LayoutParserModelCatalog()

    def __init__(self, model_name="rtdetrv2v2", path_cfg=None, device="cuda", visualize=False, from_pretrained=True,
                 infer_onnx=False):
        super().__init__()
        self.load_model(model_name, path_cfg, from_pretrained=from_pretrained)
        weights_path = getattr(self._cfg, "weights_path", None)
        if weights_path:
            raise NotImplementedError("LayoutParser: local training checkpoints (weights_path) are not supported, load a "
                                      "state_dict into .model instead")
        if infer_onnx:
            logger.warning("LayoutParser(infer_onnx=True): there is no ONNX path in yomitoku_b200, the CUDA engine is used")
        self.infer_onnx = False
        self.device = device
        self.visualize = visualize
        self.model.eval().to(self.device)
        dec = self._cfg.RTDETRTransformerv2
        self.postprocessor = RTDETRPostProcessor(num_classes=dec.num_classes, num_top_queries=dec.num_queries)
        self.thresh_score = self._cfg.thresh_score
        self.label_mapper = dict(enumerate(self._cfg.category))
        self.role = self._cfg.role

    def preprocess(self, img):
        """BGR u8 page -> (1, 3, 640, 640) fp32 in [0, 1]; reference layout_parser.py:195-199."""
        return rtdetr_input_tensor(cv2.cvtColor(img, cv2.COLOR_BGR2RGB), self._cfg.data.img_size)

    def postprocess(self, preds, image_size):
        h, w = image_size
        outputs = self.postprocessor(preds, np.array([[w, h]], np.float32), self.thresh_score)
        return LayoutParserSchema(**self.filtering_elements(outputs[0]))

    def filtering_elements(self, preds):
        """Detections -> per-category element dicts (role classes become paragraphs with a role), containment filters
        (reference layout_parser.py:209-246)."""
        by_category = {c: [] for c in self.label_mapper.values() if c not in self.role}
        for box, score, label in zip(preds["boxes"], preds["scores"], preds["labels"]):
            category = self.label_mapper[int(label)]
            role = category if category in self.role else None
            by_category["paragraphs" if role else category].append(
                {"id": None, "box": box.astype(int).tolist(), "score": float(score), "role": role, "contents": None})
        by_category = filter_contained_rectangles_within_category(by_category)
        return filter_contained_rectangles_across_categories(by_category, "tables", "paragraphs")

    def __call__(self, img, pages_dev=None):
        """pages_dev (optional): `img` already on the device as upload_pages([img], ...) made it."""
        results = self.parse_pages([img], pages_dev)[0]
        vis = layout_visualizer(results, img) if self.visualize else None
        return results, vis

    def parse_pages(self, pages, pages_dev=None):
        """Batched entry (new surface): list of BGR pages (any sizes) -> list of LayoutParserSchema; one device call.
        On a CUDA device the pages go up once as u8 (or are read from pages_dev, upload_pages(pages, ...)) and are
        resized there; otherwise they are preprocessed on the host."""
        whole = [(i, (0, 0, p.shape[1], p.shape[0])) for i, p in enumerate(pages)]
        dev = rtdetr_device_forward(self.model, pages, whole, pages_dev)
        preds = dev[0] if dev is not None else self.model(torch.cat([self.preprocess(p) for p in pages]))
        return [self.postprocess({k: v[i:i + 1] for k, v in preds.items()}, p.shape[:2]) for i, p in enumerate(pages)]


_PALETTE = {"paragraphs": (0, 200, 0), "tables": (200, 0, 0), "figures": (0, 0, 200)}


def layout_visualizer(results, img):
    out = img.copy()
    for kind, color in _PALETTE.items():
        for e in getattr(results, kind):
            x1, y1, x2, y2 = e.box
            cv2.rectangle(out, (x1, y1), (x2, y2), color, 2)
    return out
