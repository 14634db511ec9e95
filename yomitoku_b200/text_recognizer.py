"""TextRecognizer: PARSeq behind the reference's module API.

Mirrors reference src/yomitoku/text_recognizer.py:33-399 - same catalog names, constructor kwargs, width-bucketing
order (`np.argsort(content_widths)`, :135-140), mini-batch formation (`_make_mini_batch`, :158-203: width-budget greedy
fill for configs that have `data.width_budget`, fixed `data.batch_size` chunks otherwise), per-batch padded width
(`_collate`, :146-156), decode + NFKC + direction (`postprocess`, :232-245), optional 180-degree orientation fallback
(:319-350) and result order restoration (:364-373).

What changes: the mini-batches are *descriptors* - every crop keeps the padded width and the group id its reference
mini-batch would give it (outputs depend on both, SURVEY.md Appendix A9/A11) - and all crops of the call go to the GPU
as ONE packed ragged launch sequence (`PARSeq.recognize_crops`); only (token id, probability) per position come back.
`infer_onnx` / `num_parallel_batches` are accepted and ignored (no ONNX path; the reference's parallel path is
unreachable, Appendix A17).
"""
import os
import unicodedata

import cv2
import numpy as np

from .base import BaseModelCatalog, BaseModule, logger
from .config import (TextRecognizerPARSeqConfig, TextRecognizerPARSeqLargeV41Config, TextRecognizerPARSeqSmallConfig,
                     TextRecognizerPARSeqTinyConfig, TextRecognizerPARSeqTinyDynwV4Config,
                     TextRecognizerPARSeqV2Config)
from .data import ParseqDataset, crop_records, resize_with_padding
from .device_pages import as_device_pages, require_device, single_page
from .models import PARSeq
from .postprocessor import ParseqTokenizer as Tokenizer
from .schemas import TextRecognizerSchema


def load_charset(charset_path):
    with open(charset_path, "r", encoding="utf-8") as f:
        return f.read()


class TextRecognizerModelCatalog(BaseModelCatalog):
    def __init__(self):
        super().__init__()
        self.register("parseq", TextRecognizerPARSeqConfig, PARSeq)
        self.register("parseqv2", TextRecognizerPARSeqV2Config, PARSeq)
        self.register("parseq-small", TextRecognizerPARSeqSmallConfig, PARSeq)
        self.register("parseq-tiny", TextRecognizerPARSeqTinyConfig, PARSeq)
        self.register("parseq-large-v4_1", TextRecognizerPARSeqLargeV41Config, PARSeq)
        self.register("parseq-tiny-dynw-v4", TextRecognizerPARSeqTinyDynwV4Config, PARSeq)


def plan_mini_batches(widths, order, dynamic_width, batch_size, width_budget=None, max_batch_size=None):
    """Reference TextRecognizer._make_mini_batch (text_recognizer.py:158-203) on widths only.

    widths[i]: canvas width of crop i (dataset[i].shape[-1]); order: iteration order (bucketing) or None.
    Returns a list of index lists (the reference's mini-batches, in order)."""
    indices = list(order) if order is not None else list(range(len(widths)))
    batches = []
    if dynamic_width and width_budget:
        cur, cur_max = [], 0
        for idx in indices:
            w = widths[idx]
            new_max = w if w > cur_max else cur_max
            over_budget = (len(cur) + 1) * new_max > width_budget
            over_count = max_batch_size is not None and len(cur) >= max_batch_size
            if cur and (over_budget or over_count):
                batches.append(cur)
                cur = []
                new_max = w
            cur.append(idx)
            cur_max = new_max
        if cur:
            batches.append(cur)
        return batches
    cur = []
    for idx in indices:
        cur.append(idx)
        if len(cur) == batch_size:
            batches.append(cur)
            cur = []
    if cur:
        batches.append(cur)
    return batches


class TextRecognizer(BaseModule):
    model_catalog = TextRecognizerModelCatalog()

    def __init__(self, model_name="parseq-large-v4_1", path_cfg=None, device="cuda", visualize=False,
                 from_pretrained=True, infer_onnx=False, rec_orientation_fallback=False,
                 rec_orientation_fallback_thresh=0.75, batch_bucketing=False, dynamic_width=False,
                 num_parallel_batches=1, source_downscale=False):
        super().__init__()
        self.load_model(model_name, path_cfg, from_pretrained=from_pretrained)
        self.charset = load_charset(self._cfg.charset)
        self.tokenizer = Tokenizer(self.charset)
        self.device = device
        self.model.tokenizer = self.tokenizer
        self.model.eval()
        self.visualize = visualize
        if infer_onnx:
            logger.warning("TextRecognizer(infer_onnx=True): there is no ONNX path in yomitoku_b200, the CUDA engine is used")
        if visualize:
            logger.warning("TextRecognizer(visualize=True): the recognized text is not drawn (the reference's "
                           "rec_visualizer needs its bundled font); `vis` is the detector's image or a copy of the page")
        self.infer_onnx = False
        self.rec_orientation_fallback = rec_orientation_fallback
        self.rec_orientation_fallback_thresh = rec_orientation_fallback_thresh
        self.batch_bucketing = batch_bucketing
        self.dynamic_width = dynamic_width
        self.num_parallel_batches = num_parallel_batches
        self.source_downscale = source_downscale
        # device-side crop extraction (csrc/crop_ops.cu, bit-exact with the OpenCV path): the page goes to HBM once and
        # the canvases are cut there - including the orientation fallback's 180-degree second look and the
        # source_downscale pyramid.
        self.device_crops = os.environ.get("YTK_DEVICE_CROPS", "1") != "0" and self.device.type == "cuda"
        self.model.to(self.device)

    # ------------------------------------------------------------------------------------------ batching
    def preprocess(self, img, polygons):
        """Crops + bucketing order + mini-batch plan; reference text_recognizer.py:115-144."""
        if polygons is None:
            h, w = img.shape[:2]
            polygons = [[[0, 0], [w, 0], [w, h], [0, h]]]
        dataset = ParseqDataset(self._cfg, img, polygons, dynamic_width=self.dynamic_width,
                                source_downscale=self.source_downscale)
        order = None
        if self.batch_bucketing and len(dataset) == len(polygons) and len(dataset) > 1:
            order = np.argsort(dataset.content_widths).tolist()
        plan = self._make_mini_batch(dataset, order)
        return plan, polygons, dataset, order

    def _make_mini_batch(self, dataset, order=None):
        widths = [d.shape[1] for d in dataset.data]
        return plan_mini_batches(widths, order, self.dynamic_width, self._cfg.data.batch_size,
                                 getattr(self._cfg.data, "width_budget", None),
                                 getattr(self._cfg.data, "max_batch_size", None))

    def _collate_widths(self, canvases, plan):
        """Per crop: (padded width, group id) = what reference _collate (:146-156) does to each mini-batch."""
        widths = [c if isinstance(c, (int, np.integer)) else c.shape[1] for c in canvases]   # canvases or widths
        padded = [0] * len(widths)
        group = [0] * len(widths)
        for g, batch in enumerate(plan):
            wmax = max(widths[i] for i in batch) if self.dynamic_width else None
            for i in batch:
                padded[i] = wmax if wmax is not None else widths[i]
                group[i] = g
        return padded, group

    # ------------------------------------------------------------------------------------------ inference
    def _run_plan(self, canvases, plan):
        """All mini-batches of `plan` in one packed device call; returns (ids, probs) in `canvases` order."""
        flat = [i for b in plan for i in b]
        padded, group = self._collate_widths(canvases, plan)
        group = np.asarray([group[i] for i in flat], np.int64)
        ids, probs, glen = self.model.recognize_crops([canvases[i] for i in flat], [padded[i] for i in flat],
                                                      group.tolist(), len(plan))
        self._eos_tail(ids, probs, glen[group])
        return flat, ids, probs

    def _eos_tail(self, ids, probs, lens):
        """With refine_iters == 0 the reference's output has only the positions its mini-batch's AR loop ran: row r
        keeps lens[r] positions, the rest reads as EOS with probability 1.  In place."""
        if self.model.refine_iters == 0:
            cut = np.arange(ids.shape[1])[None, :] >= np.asarray(lens, np.int64)[:, None]
            ids[cut] = self.tokenizer.eos_id
            probs[cut] = 1.0

    def _decode_in_order(self, ids, probs, points, order):
        """Rows of (ids, probs) in plan order -> (texts, scores, directions) in detection order.  order: the bucketing
        order the plan followed (None: detection order).  The reference pairs the rows with the points in plan order
        (:271-283, 364-373); with dropped quads `points` is longer than the rows, exactly as there."""
        if not len(ids):
            return [], [], []
        pts = [points[i] for i in order] if order is not None else points
        p, s, d = self.postprocess_ids(ids, probs, pts[:len(ids)])
        if order is not None:
            inverse = np.argsort(order)
            p, s, d = [p[i] for i in inverse], [s[i] for i in inverse], [d[i] for i in inverse]
        return p, s, d

    def postprocess_ids(self, ids, probs, points):
        pred, score = self.tokenizer.decode_ids(ids, probs)
        pred = [unicodedata.normalize("NFKC", x) for x in pred]
        if len(points) == 0:
            return pred, score, []
        pts = np.asarray(points, dtype=np.float64)          # (n, 4, 2); same float64 norms as np.linalg.norm per quad
        w = np.sqrt(((pts[:, 0] - pts[:, 1]) ** 2).sum(axis=1))
        h = np.sqrt(((pts[:, 1] - pts[:, 2]) ** 2).sum(axis=1))
        directions = ["vertical" if v else "horizontal" for v in (h > w * 2).tolist()]
        return pred, score, directions

    def postprocess(self, p, points):
        """Reference entry (:232-245) on a softmax tensor (B,S,C)."""
        mx, ids = p.max(-1)
        return self.postprocess_ids(ids.cpu().numpy(), mx.float().cpu().numpy(), points)

    def _run_batch_inference(self, canvases, plan, points_in_plan_order):
        flat, ids, probs = self._run_plan(canvases, plan)
        return self.postprocess_ids(ids, probs, points_in_plan_order)

    def _apply_orientation_fallback(self, dataset, points, preds, scores, directions):
        """Re-run low-score crops rotated by 180 degrees; reference text_recognizer.py:319-350."""
        retry = [i for i, s in enumerate(scores) if s < self.rec_orientation_fallback_thresh]
        if not retry:
            return
        img_size = self._cfg.data.img_size
        canv = [resize_with_padding(cv2.rotate(dataset.roi_images[i], cv2.ROTATE_180), img_size) for i in retry]
        bs = self._cfg.data.batch_size
        plan = [list(range(s, min(s + bs, len(canv)))) for s in range(0, len(canv), bs)]
        keep_dw = self.dynamic_width
        self.dynamic_width = False           # the fallback batch is a fixed-width tensor in the reference (:205-210)
        try:
            r_preds, r_scores, r_dirs = self._run_batch_inference(canv, plan, [points[i] for i in retry])
        finally:
            self.dynamic_width = keep_dw
        for j, idx in enumerate(retry):
            if r_scores[j] > scores[idx] and r_scores[j] >= self.rec_orientation_fallback_thresh:
                preds[idx], scores[idx], directions[idx] = r_preds[j], r_scores[j], r_dirs[j]

    def _upload_page(self, img):
        import torch
        return torch.from_numpy(np.ascontiguousarray(img))[None].to(self.model.cuda_device())

    def _run_records(self, pages, sel, levels, padded, group, n_groups):
        """Cuts the crops of the records `sel` (already in packing order) on the GPU and runs them as one packed call.
        pages[k] = the page at pyramid level k (models.extract_crops_pyramid), levels[r] = level of record r; padded[r] / group[r] =
        padded width and mini-batch index of record r.  Returns (ids, probs) with the positions a `refine_iters == 0`
        model never produced filled like the host path does."""
        from . import models
        canv, total, pix_off = models.extract_crops_pyramid(pages, sel, levels)
        descs = models.crop_descriptors(self._cfg, pix_off, sel["canvas_w"], padded, group)
        ids, probs, glen = self.model.run_packed_ptr(canv.data_ptr(), 1, total, descs, len(sel), n_groups)
        self._eos_tail(ids, probs, glen[np.asarray(group, np.int64)])
        return ids, probs

    def _device_records(self, img, points, dp=None):
        """Page on the device + one crop record per valid quad, in quad order (data.crop_records); the pyramid levels
        of source_downscale are built on the device when a record needs them.  dp: the page already in HBM (a one-page
        DevicePages, `img` is then unused), else `img` is uploaded."""
        shape = img.shape if dp is None else dp.shapes[0] + (3,)
        geoms, levels, _ = crop_records(shape, points, self._cfg.data.img_size, self.dynamic_width,
                                        self.source_downscale)
        return {0: self._upload_page(img) if dp is None else dp.pair()}, geoms, levels

    def _call_device_crops(self, img, points, dp=None):
        """`__call__` with the crops cut on the GPU: same order / plan / pairing decisions as the host path, taken
        from the crop records (canvas and content widths follow from the quads alone).  dp: the page already in HBM
        (a one-page DevicePages), else `img` is uploaded."""
        shape = dp.shapes[0] + (3,) if dp is not None else img.shape
        if points is None:
            h, w = shape[:2]
            points = [[[0, 0], [w, 0], [w, h], [0, h]]]
        pages, geoms, levels = self._device_records(img, points, dp)
        n = len(geoms)
        if n == 0:
            return TextRecognizerSchema(contents=[], scores=[], points=points, directions=[])
        order = None
        if self.batch_bucketing and n == len(points) and n > 1:
            # a Python list -> int64, like the reference's np.argsort(dataset.content_widths): numpy's unstable sort may
            # order ties differently for another dtype (SURVEY.md Appendix A9)
            order = np.argsort(geoms["cw"].tolist()).tolist()
        widths = geoms["canvas_w"].tolist()
        plan = plan_mini_batches(widths, order, self.dynamic_width, self._cfg.data.batch_size,
                                 getattr(self._cfg.data, "width_budget", None),
                                 getattr(self._cfg.data, "max_batch_size", None))
        flat = np.asarray([i for b in plan for i in b], np.int64)
        padded, group = self._collate_widths(widths, plan)
        ids, probs = self._run_records(pages, geoms[flat].copy(), levels[flat], [padded[i] for i in flat],
                                       [group[i] for i in flat], len(plan))
        p, s, d = self._decode_in_order(ids, probs, points, order)
        if self.rec_orientation_fallback:
            self._device_orientation_fallback(pages, geoms, levels, points, p, s, d)
        return TextRecognizerSchema(contents=p, scores=s, points=points, directions=d)

    def _device_orientation_fallback(self, pages, geoms, levels, points, preds, scores, directions):
        """`_apply_orientation_fallback` (reference text_recognizer.py:319-350) with the second look cut on the GPU: the
        same rectified crop rotated by 180 degrees (record bit `rot & 2`) on the fixed-width canvas, in chunks of
        `batch_size` (a fixed-width tensor in the reference: :205-210)."""
        retry = [i for i, sc in enumerate(scores) if sc < self.rec_orientation_fallback_thresh]
        if not retry:
            return
        sel = geoms[np.asarray(retry, np.int64)].copy()
        sel["rot"] |= 2
        sel["canvas_w"] = self._cfg.data.img_size[1]
        bs = self._cfg.data.batch_size
        group = [k // bs for k in range(len(retry))]
        ids, probs = self._run_records(pages, sel, levels[np.asarray(retry, np.int64)], sel["canvas_w"].tolist(), group,
                                       group[-1] + 1)
        r_preds, r_scores, r_dirs = self.postprocess_ids(ids, probs, [points[i] for i in retry])
        for j, idx in enumerate(retry):
            if r_scores[j] > scores[idx] and r_scores[j] >= self.rec_orientation_fallback_thresh:
                preds[idx], scores[idx], directions[idx] = r_preds[j], r_scores[j], r_dirs[j]

    def __call__(self, img, points=None, vis=None):
        """img: BGR page (numpy, or on the GPU: a CUDA (H, W, 3) uint8 tensor or a one-page DevicePages); points: list of
        quads (4 clockwise points).  Returns (TextRecognizerSchema, vis)."""
        dp = as_device_pages(img)
        if dp is not None:
            if not self.device_crops:
                raise ValueError("TextRecognizer: pages on the GPU need the device crop extraction, which is off "
                                 "(YTK_DEVICE_CROPS=0 or a recognizer not on a CUDA device)")
            single_page(dp, "TextRecognizer")
            require_device(dp, self.model.cuda_device(), "TextRecognizer")
            results = self._call_device_crops(None, points, dp.ready())
            if self.visualize and vis is None:
                vis = dp.numpy(0)
            return results, vis
        if self.device_crops:
            results = self._call_device_crops(img, points)
            if self.visualize and vis is None:
                vis = img.copy()
            return results, vis
        plan, points, dataset, order = self.preprocess(img, points)
        n = len(dataset)
        if n == 0:
            preds, scores, directions = [], [], []
        else:
            _, ids, probs = self._run_plan(dataset.data, plan)
            preds, scores, directions = self._decode_in_order(ids, probs, points, order)
        if self.rec_orientation_fallback and n:
            self._apply_orientation_fallback(dataset, points, preds, scores, directions)
        results = TextRecognizerSchema(contents=preds, scores=scores, points=points, directions=directions)
        if self.visualize:
            if vis is None:
                vis = img.copy()
        return results, vis
