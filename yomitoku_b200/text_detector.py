"""TextDetector: DBNet++ behind the reference's module API.

Mirrors reference src/yomitoku/text_detector.py:26-146 - same catalog names (`dbnet`, `dbnetv2`, `dbnetv2_1`),
constructor kwargs, `preprocess` / `postprocess` / `__call__` contract and result schema.  The resize + normalisation
(cv2.resize INTER_AREA, whether the page shrinks or grows) and the model forward run as sm_90a kernels; contour
extraction / unclip stay on the host like the reference (SURVEY.md R3).  `infer_onnx` is accepted and ignored:
ONNX / multi-backend dispatch is out of scope for this path.
"""
import os

import numpy as np
import torch

from .base import BaseModelCatalog, BaseModule, logger
from .config import TextDetectorDBNetConfig, TextDetectorDBNetV2_1Config, TextDetectorDBNetV2Config
from .data import array_to_tensor, resize_shortest_edge, standardization_image
from .models import DBNet
from .postprocessor import DBnetPostProcessor
from .schemas import TextDetectorSchema


# catalog names of the reference (text_detector.py:26-31): one architecture, three threshold / weight sets
_DETECTORS = (("dbnet", TextDetectorDBNetConfig), ("dbnetv2", TextDetectorDBNetV2Config),
              ("dbnetv2_1", TextDetectorDBNetV2_1Config))


class TextDetectorModelCatalog(BaseModelCatalog):
    def __init__(self):
        super().__init__()
        for name, cfg in _DETECTORS:
            self.register(name, cfg, DBNet)


class TextDetector(BaseModule):
    model_catalog = TextDetectorModelCatalog()

    def __init__(self, model_name="dbnetv2_1", path_cfg=None, device="cuda", visualize=False, from_pretrained=True,
                 infer_onnx=False):
        super().__init__()
        self.visualize = visualize
        if infer_onnx:
            logger.warning("TextDetector(infer_onnx=True): there is no ONNX path in yomitoku_b200, the CUDA engine is used")
        self.infer_onnx = False   # accepted for API compatibility; there is no ONNX path here
        self.device = device
        self.load_model(model_name, path_cfg, from_pretrained=from_pretrained)
        self.model.eval().to(self.device)
        self.post_processor = DBnetPostProcessor(**self._cfg.post_process)
        # the pre-processing is a CUDA kernel: a detector placed on the CPU (a stand-in model with only the reference's
        # `model(tensor)` contract) runs the reference's host flow, preprocess + model + postprocess
        self.on_cuda = torch.device(device).type == "cuda"
        # front half of the post-processing (threshold, connected components, per-component sums) on the device: only
        # the components' row runs come back instead of the probability map.  Pages that need OpenCV's view of the
        # bitmap (a component with a hole) fall back to the host path per page - the result is the same either way.
        self.device_post = (self.on_cuda and os.environ.get("YTK_DEVICE_POST", "1") != "0"
                            and torch.cuda.is_available())

    def preprocess(self, img):
        """BGR u8 page -> normalised (1,3,H',W') fp32 tensor; reference text_detector.py:99-107 (host path: the
        reference's API and the model-level seam `model(preprocess(img))`; on a CUDA device `__call__` pre-processes the
        u8 page on the device instead)."""
        img = img.copy()
        img = img[:, :, ::-1].astype(np.float32)
        resized = resize_shortest_edge(img, self._cfg.data.shortest_size, self._cfg.data.limit_size)
        return array_to_tensor(standardization_image(resized))

    def postprocess(self, preds, image_size):
        return self.post_processor(preds, image_size)

    def postprocess_device(self, prob_dev, image_size, stream=None):
        """prob_dev: (n, Hn, Wn) fp32 cuda probability maps -> per page (quads, scores), equal to `postprocess` of the
        downloaded maps.  image_size: the (h, w) of every page, or a list with one (h, w) per page."""
        from .models import dbnet_post_front
        pp = self.post_processor
        runs, _ = dbnet_post_front(prob_dev, pp.thresh, stream)
        hn, wn = prob_dev.shape[1:]
        sizes = image_size if isinstance(image_size, list) else [image_size] * len(runs)
        out = []
        for i, (r, size) in enumerate(zip(runs, sizes)):
            if r is None:
                out.append(self.postprocess({"binary": prob_dev[i:i + 1, None].cpu().numpy()}, size))
            else:
                out.append(pp.boxes_from_runs(r, wn, hn, size[1], size[0]))
        return out

    def _detect_device(self, pages_u8):
        """(n, H0, W0, 3) u8 pages -> per page (quads, scores) through the device front half."""
        t = torch.from_numpy(pages_u8).to(self.model.cuda_device(), non_blocking=False)
        prob = self.model.detect_pages_u8(t)
        return self.postprocess_device(prob, pages_u8.shape[1:3])

    def _probability_map(self, img):
        if not self.on_cuda:
            with torch.inference_mode():
                return self.model(self.preprocess(img))["binary"].cpu().numpy()
        # fused GPU pre-processing straight from the u8 page, whether it shrinks or grows
        prob = self.model.detect_pages_u8(np.ascontiguousarray(img))
        return prob.cpu().numpy()[:, None] if prob.is_cuda else prob.numpy()[:, None]

    def __call__(self, img):
        """Apply the detection model to a BGR page (np.ndarray HxWx3 u8); returns (TextDetectorSchema, vis)."""
        ori_h, ori_w = img.shape[:2]
        if self.device_post:
            quads, scores = self._detect_device(np.ascontiguousarray(img)[None])[0]
        else:
            preds = {"binary": self._probability_map(img)}
            quads, scores = self.postprocess(preds, (ori_h, ori_w))
        results = TextDetectorSchema(points=quads, scores=scores)
        vis = None
        if self.visualize:
            vis = det_visualizer(img, quads, line_color=tuple(self._cfg.visualize.color[::-1]))
        return results, vis

    def detect_pages(self, pages):
        """Batched entry (new surface, SURVEY.md section 0): list of BGR pages, of one size or of many -> list of
        TextDetectorSchema.  The pages go to the device back to back with a page table (data.page_table); one device
        launch sequence per group of pages that share a detector input size (a same-size batch is one group), host
        post-processing per page."""
        from .pipeline import BatchPlan
        plan = BatchPlan([p.shape[:2] for p in pages], self.model.input_size, max(1, len(pages)))
        flat = torch.from_numpy(np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in pages]))
        if self.device_post:
            flat = flat.to(self.model.cuda_device(), non_blocking=False)
        out = [None] * len(pages)
        for ch in plan.chunks:
            idx = ch[2]
            prob = self.model.detect_pages_table(flat, plan.table[idx])
            if self.device_post:
                res = self.postprocess_device(prob, [plan.shapes[i] for i in idx])
            else:
                prob = prob.cpu().numpy() if prob.is_cuda else prob.numpy()
                res = [self.postprocess({"binary": prob[j:j + 1, None]}, plan.shapes[i]) for j, i in enumerate(idx)]
            for i, (quads, scores) in zip(idx, res):
                out[i] = TextDetectorSchema(points=quads, scores=scores)
        return out


def det_visualizer(img, quads, line_color=(0, 255, 0), **_):
    import cv2
    out = img.copy()
    for q in quads:
        cv2.polylines(out, [np.array(q, dtype=np.int32)], True, line_color, 2)
    return out
