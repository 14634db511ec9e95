"""Host-side image functions of the hot path (numpy / OpenCV), same names and semantics as the reference's
src/yomitoku/data/functions.py:196-439 and data/dataset.py:19-129.

These are the host versions of rows R1 / R4 of SURVEY.md section 8a, exactly as the reference runs them; both rows also
exist on the GPU: the detector's resize + normalisation fused in csrc/dbnet_ops.cu (preprocess_kernel, for pages that
shrink or grow; the functions here serve the model-level seam), and the crop extraction in csrc/crop_ops.cu, for which
`crop_geometry` / `crop_records` below compute the per-quad records (everything that follows from the quads alone).
"""
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import cv2
import numpy as np
import torch
from PIL import Image

from .base import set_logger

logger = set_logger(__name__, "WARNING")

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)

SUPPORT_INPUT_FORMAT = ["jpg", "jpeg", "png", "bmp", "tiff", "tif"]
MIN_IMAGE_SIZE = 32
WARNING_IMAGE_SIZE = 720


# ------------------------------------------------------------------------------------------------ page files
def validate_image(img):
    """A page with a side under 32 px is refused; a shorter side under 720 px is read with a warning (reference
    data/functions.py:19-30)."""
    h, w = img.shape[:2]
    if h < MIN_IMAGE_SIZE or w < MIN_IMAGE_SIZE:
        raise ValueError("Image size is too small.")
    if min(h, w) < WARNING_IMAGE_SIZE:
        logger.warning("The image size is small (%dx%d), which may result in reduced OCR accuracy. The process will "
                       "continue; pages with a shorter side of at least 720 pixels are recommended." % (w, h))


def load_image(image_path):
    """The pages of an image file as a list of BGR uint8 arrays (reference data/functions.py:33-78): jpg, jpeg, png,
    bmp, tif and tiff, opened with Pillow and converted to RGB; every frame of a TIFF is a page, each checked by
    `validate_image`.  PDF files are refused: rendering PDF pages is not part of this package."""
    image_path = Path(image_path)
    if not image_path.exists():
        raise FileNotFoundError(f"File not found: {image_path}")
    ext = image_path.suffix[1:].lower()
    if ext == "pdf":
        raise ValueError(f"{image_path}: PDF input is not supported, rendering PDF pages is not part of this package "
                         f"(it has no PDF renderer); convert the pages to images first")
    if ext not in SUPPORT_INPUT_FORMAT:
        raise ValueError(f"Unsupported image format. Supported formats are {SUPPORT_INPUT_FORMAT}")
    try:
        img = Image.open(image_path)
    except Exception:
        raise ValueError("Invalid image data.") from None
    frames = getattr(img, "n_frames", 1) if ext in ("tif", "tiff") else 1
    pages = []
    for i in range(frames):
        img.seek(i)
        rgb = np.asarray(img.convert("RGB"))
        validate_image(rgb)
        pages.append(np.ascontiguousarray(rgb[:, :, ::-1]))
    return pages


def shortest_edge_size(h, w, shortest_edge_length, max_length):
    """Target (new_h, new_w) of resize_shortest_edge: reference data/functions.py:212-224 (two int() truncations, then
    floor to a multiple of 32, minimum 32)."""
    scale = shortest_edge_length / min(h, w)
    if h < w:
        new_h, new_w = shortest_edge_length, int(w * scale)
    else:
        new_h, new_w = int(h * scale), shortest_edge_length
    if max(new_h, new_w) > max_length:
        scale = float(max_length) / max(new_h, new_w)
        new_h, new_w = int(new_h * scale), int(new_w * scale)
    return max(int(new_h / 32) * 32, 32), max(int(new_w / 32) * 32, 32)


def resize_shortest_edge(img, shortest_edge_length, max_length):
    newh, neww = shortest_edge_size(img.shape[0], img.shape[1], shortest_edge_length, max_length)
    return cv2.resize(img, (neww, newh), interpolation=cv2.INTER_AREA)


def standardization_image(img, rgb=IMAGENET_MEAN, std=IMAGENET_STD):
    """reference data/functions.py:230-247: flip the channel axis, /255, (x - mean) / std in float64, cast to f32."""
    img = img[:, :, ::-1] / 255.0
    return ((img - np.array(rgb)) / np.array(std)).astype(np.float32)


def array_to_tensor(img):
    """(H, W, C) -> (1, C, H, W) float tensor (reference data/functions.py:250-264)."""
    return torch.as_tensor(np.transpose(img, (2, 0, 1)), dtype=torch.float)[None]


def validate_quads(img, quad):
    """True if the quad has 4 (x, y) vertices whose int bounding box lies inside the image (x2 == w allowed), else
    None - reference data/functions.py:267-298."""
    if len(quad) != 4 or any(len(p) != 2 for p in quad):
        return None
    q = np.array(quad, dtype=int)
    h, w = img.shape[:2]
    if q[:, 0].min() < 0 or q[:, 0].max() > w or q[:, 1].min() < 0 or q[:, 1].max() > h:
        return None
    return True


def extract_roi_with_perspective(img, quad):
    """Perspective-rectified crop of one quad (reference data/functions.py:301-333): vertices truncated to int64, the
    warp is computed inside the quad's bounding-box slice, output size = (int |p0p1|, int |p1p2|)."""
    q = np.array(quad, dtype=np.int64)
    x0, y0 = int(q[:, 0].min()), int(q[:, 1].min())
    roi = img[y0:int(q[:, 1].max()), x0:int(q[:, 0].max()), :]
    q = q - np.array([x0, y0], dtype=np.int64)
    width = int(np.linalg.norm(q[0] - q[1]))
    height = int(np.linalg.norm(q[1] - q[2]))
    src = np.float32(q)
    dst = np.float32([[0, 0], [width, 0], [width, height], [0, height]])
    return cv2.warpPerspective(roi, cv2.getPerspectiveTransform(src, dst), (width, height))


def rotate_text_image(img, thresh_aspect=2):
    """Tall crops (h > thresh * w) are vertical text: rotate 90 degrees counter-clockwise (functions.py:336-350)."""
    h, w = img.shape[:2]
    return cv2.rotate(img, cv2.ROTATE_90_COUNTERCLOCKWISE) if h > thresh_aspect * w else img


def calc_resize_without_padding(img, target_size):
    """Down-scale-only fit into target (H, W); returns (new_h, new_w) (functions.py:353-376)."""
    h, w = img.shape[:2]
    s = min(target_size[1] / w if w > target_size[1] else 1.0, target_size[0] / h if h > target_size[0] else 1.0)
    return max(1, int(h * s)), max(1, int(w * s))


def _paste(img, target_h, canvas_w, new_h, new_w, background_color):
    resized = cv2.resize(img, (new_w, new_h), interpolation=cv2.INTER_AREA)
    canvas = np.zeros((target_h, canvas_w, 3), dtype=np.uint8)
    if any(background_color):          # black (the only colour the path uses) is what np.zeros already holds
        canvas[:, :] = background_color
    canvas[: resized.shape[0], : resized.shape[1], :] = resized
    return canvas


def resize_with_padding(img, target_size, background_color=(0, 0, 0)):
    """Fixed canvas: content top-left on a target_size background (functions.py:379-401)."""
    new_h, new_w = calc_resize_without_padding(img, target_size)
    return _paste(img, target_size[0], target_size[1], new_h, new_w, background_color)


def resize_with_dynamic_padding(img, target_size, align=8, margin=64, background_color=(0, 0, 0)):
    """Dynamic canvas: width = min(target_w, ceil((content + margin) / align) * align) (functions.py:404-439)."""
    new_h, new_w = calc_resize_without_padding(img, target_size)
    canvas_w = min(target_size[1], ((new_w + margin + align - 1) // align) * align)
    return _paste(img, target_size[0], canvas_w, new_h, new_w, background_color)


def _calc_source_levels(quads, target_height, max_level=3):
    """Pyramid level per quad: floor(log2(short_side / target_height)) clipped to [0, max_level]
    (reference data/dataset.py:19-41)."""
    if len(quads) == 0:
        return np.zeros(0, dtype=int)
    q = np.asarray(quads, dtype=np.float32).reshape(-1, 4, 2)
    short = np.maximum(1.0, np.minimum(np.linalg.norm(q[:, 0] - q[:, 1], axis=1),
                                       np.linalg.norm(q[:, 1] - q[:, 2], axis=1)))
    return np.clip(np.floor(np.log2(short / float(target_height))).astype(int), 0, max_level)


def crop_to_tensor(crop_u8):
    """torchvision ToTensor + Normalize(0.5, 0.5): HWC u8 -> CHW f32 in [-1, 1] (reference data/dataset.py:57-62)."""
    t = torch.from_numpy(np.ascontiguousarray(crop_u8)).permute(2, 0, 1).to(torch.float32).div_(255.0)
    return t.sub_(0.5).div_(0.5)


# ------------------------------------------------------------------------------------------ device-side crop extraction
# Layout of ytk_page / ytk_rtdetr_src (include/yomitoku_b200.h): one page of a flat buffer and a rectangle of it.
PAGE_DTYPE = np.dtype([("page_off", "<i8"), ("H", "<i4"), ("W", "<i4"), ("x0", "<i4"), ("y0", "<i4"), ("x1", "<i4"),
                       ("y1", "<i4")])


def page_table(shapes):
    """Pages of the given (h, w) shapes back to back in one flat BGR uint8 buffer: (PAGE_DTYPE records covering each
    whole page, total bytes).  Same-size pages give the byte layout of their (n, h, w, 3) stack."""
    hw = np.asarray([(int(s[0]), int(s[1])) for s in shapes], np.int64).reshape(-1, 2)
    size = hw[:, 0] * hw[:, 1] * 3
    t = np.zeros(len(hw), PAGE_DTYPE)
    t["page_off"] = np.cumsum(size) - size
    t["H"] = t["y1"] = hw[:, 0]
    t["W"] = t["x1"] = hw[:, 1]
    return t, int(size.sum())


# Layout of ytk_crop_geom (include/yomitoku_b200.h) / ytk::CropGeom (csrc/crop_math.h).
CROP_GEOM_DTYPE = np.dtype([
    ("minv", "<f8", (9,)), ("roi_off", "<i8"), ("pix_off", "<i8"), ("page", "<i4"), ("x0", "<i4"), ("y0", "<i4"),
    ("rw", "<i4"), ("rh", "<i4"), ("w", "<i4"), ("h", "<i4"), ("rot", "<i4"), ("cw", "<i4"), ("ch", "<i4"),
    ("canvas_w", "<i4"), ("canvas_h", "<i4")], align=True)


def crop_geometry(img_shape, quads, target_size, dynamic_width, page=0, align=8, margin=64):
    """Everything about the crops of one page that follows from the quads alone - the host half of the device-side
    crop extraction (csrc/crop_ops.cu does the pixel work).  Per valid quad, exactly the scalar decisions of
    `ParseqDataset._preprocess_on` (reference data/dataset.py:106-123): bounding-box slice and output size of
    extract_roi_with_perspective (functions.py:301-333; the 3x3 matrix comes from the same cv2.getPerspectiveTransform
    call, inverted like cv2.warpPerspective does internally), the rotation test of rotate_text_image (:336-350), the
    down-scale-only size of calc_resize_without_padding (:353-376) and the canvas width of resize_with_padding /
    resize_with_dynamic_padding (:379-439).

    Returns (geoms, keep): a CROP_GEOM_DTYPE array for the valid quads (roi_off / pix_off are filled by the caller) and
    the indices of those quads; invalid quads are dropped like validate_quads does (functions.py:267-298)."""
    H, W = int(img_shape[0]), int(img_shape[1])
    th, tw = int(target_size[0]), int(target_size[1])
    out = np.zeros(len(quads), dtype=CROP_GEOM_DTYPE)
    keep = []
    k = 0
    for qi, quad in enumerate(quads):
        if len(quad) != 4 or any(len(p) != 2 for p in quad):
            continue
        q = np.array(quad, dtype=np.int64)
        x0, y0, x1, y1 = int(q[:, 0].min()), int(q[:, 1].min()), int(q[:, 0].max()), int(q[:, 1].max())
        if x0 < 0 or x1 > W or y0 < 0 or y1 > H:
            continue
        ql = q - np.array([x0, y0], dtype=np.int64)
        w = int(np.linalg.norm(ql[0] - ql[1]))
        h = int(np.linalg.norm(ql[1] - ql[2]))
        if w <= 0 or h <= 0 or x1 <= x0 or y1 <= y0:
            # the reference fails inside cv2.warpPerspective here (empty source or destination)
            raise cv2.error("crop_geometry: degenerate quad %s (roi %dx%d, output %dx%d)" % (quad, x1 - x0, y1 - y0, w, h))
        m = cv2.getPerspectiveTransform(np.float32(ql), np.float32([[0, 0], [w, 0], [w, h], [0, h]]))
        g = out[k]
        g["minv"] = cv2.invert(m)[1].reshape(-1)
        g["page"], g["x0"], g["y0"], g["rw"], g["rh"], g["w"], g["h"] = page, x0, y0, x1 - x0, y1 - y0, w, h
        rot = h > 2 * w
        sh, sw = (w, h) if rot else (h, w)
        s = min(tw / sw if sw > tw else 1.0, th / sh if sh > th else 1.0)
        ch, cw = max(1, int(sh * s)), max(1, int(sw * s))
        g["rot"], g["cw"], g["ch"] = int(rot), cw, ch
        g["canvas_w"] = min(tw, ((cw + margin + align - 1) // align) * align) if dynamic_width else tw
        g["canvas_h"] = th
        keep.append(qi)
        k += 1
    return out[:k], keep


def pyramid_shapes(img_shape, max_level):
    """(H, W) of the source_downscale pyramid levels 0..max_level: each level is cv2.resize(prev, None, fx=0.5, fy=0.5),
    i.e. (cvRound(H / 2), cvRound(W / 2)) with round-half-to-even (reference data/dataset.py:76-86)."""
    shapes = [(int(img_shape[0]), int(img_shape[1]))]
    for _ in range(max_level):
        h, w = shapes[-1]
        shapes.append((int(np.rint(h * 0.5)), int(np.rint(w * 0.5))))
    return shapes


def crop_records(img_shape, quads, target_size, dynamic_width, source_downscale=False, page=0):
    """Crop records of one page in quad order, what `ParseqDataset.__init__` decides per quad (reference
    data/dataset.py:45-95) without touching a pixel: with `source_downscale` a quad whose short side is >= 2^k * 32 px is
    cut from pyramid level k with its coordinates divided by 2^k as float32 (:26-41, 64-86).
    Returns (geoms, levels, keep): CROP_GEOM_DTYPE records of the valid quads, their pyramid level, their quad index."""
    quad_levels = np.zeros(len(quads), dtype=int)
    if source_downscale and len(quads) > 0:
        quad_levels = _calc_source_levels(quads, target_size[0])
    shapes = pyramid_shapes(img_shape, int(quad_levels.max()) if len(quads) else 0)
    rows, levels, keep = [], [], []
    for k in sorted(set(quad_levels.tolist())):
        idx = np.nonzero(quad_levels == k)[0]
        qs = [quads[i] if k == 0 else (np.asarray(quads[i], dtype=np.float32) / (2.0 ** k)).tolist() for i in idx]
        g, kept = crop_geometry(shapes[k], qs, target_size, dynamic_width, page=page)
        rows += list(g)
        levels += [k] * len(g)
        keep += [int(idx[j]) for j in kept]
    order = np.argsort(np.asarray(keep, np.int64), kind="stable")
    geoms = np.zeros(len(rows), dtype=CROP_GEOM_DTYPE)
    for r, o in enumerate(order):
        geoms[r] = rows[o]
    return geoms, np.asarray(levels, np.int64)[order], [keep[o] for o in order]


def layout_crop_buffers(geoms):
    """Fills roi_off / pix_off (crops packed back to back) and returns (scratch_bytes, canvas_bytes)."""
    roi = geoms["w"].astype(np.int64) * geoms["h"] * 3
    pix = geoms["canvas_w"].astype(np.int64) * geoms["canvas_h"] * 3
    geoms["roi_off"] = np.cumsum(roi) - roi
    geoms["pix_off"] = np.cumsum(pix) - pix
    return int(roi.sum()), int(pix.sum())


class ParseqDataset:
    """Crops of one page for the recognizer; reference data/dataset.py:44-129.

    `data[i]` is the padded 32-px-high RGB u8 canvas, `roi_images[i]` the rectified crop before resizing,
    `content_widths[i]` the resized content width; invalid quads are dropped (valid_quads keeps the survivors)."""

    def __init__(self, cfg, img, quads, num_workers=8, dynamic_width=False, source_downscale=False):
        self.quads = quads
        self.cfg = cfg
        self.dynamic_width = dynamic_width
        self.transform = crop_to_tensor
        levels = {0: img[:, :, ::-1]}          # BGR -> RGB view
        quad_levels = np.zeros(len(quads), dtype=int)
        if source_downscale and len(quads) > 0:
            quad_levels = _calc_source_levels(quads, cfg.data.img_size[0])
            level_img = img
            for k in range(1, int(quad_levels.max()) + 1):
                level_img = cv2.resize(level_img, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_AREA)
                if (quad_levels >= k).any():
                    levels[k] = level_img[:, :, ::-1]
        self.img = levels[0]
        jobs = [(q, int(lv), levels.get(int(lv), self.img)) for q, lv in zip(quads, quad_levels)]
        if len(jobs) > 1 and num_workers > 1:
            with ThreadPoolExecutor(max_workers=num_workers) as ex:
                done = list(ex.map(self._job, jobs))
        else:
            done = [self._job(j) for j in jobs]
        self.data = [d[0] for d in done if d is not None]
        self.roi_images = [d[1] for d in done if d is not None]
        self.content_widths = [d[2] for d in done if d is not None]
        self.valid_quads = [q for q, d in zip(quads, done) if d is not None]

    def _job(self, job):
        quad, level, level_img = job
        if level > 0:
            quad = (np.asarray(quad, dtype=np.float32) / (2.0 ** level)).tolist()
        return self._preprocess_on(level_img, quad)

    def preprocess(self, quad):
        return self._preprocess_on(self.img, quad)

    def _preprocess_on(self, img, quad):
        if validate_quads(img, quad) is None:
            return None
        roi = extract_roi_with_perspective(img, quad)
        if roi is None:
            return None
        roi = rotate_text_image(roi, thresh_aspect=2)
        size = self.cfg.data.img_size
        canvas = resize_with_dynamic_padding(roi, size) if self.dynamic_width else resize_with_padding(roi, size)
        return canvas, roi, calc_resize_without_padding(roi, size)[1]

    def __len__(self):
        return len(self.data)

    def __getitem__(self, index):
        return self.transform(self.data[index])
