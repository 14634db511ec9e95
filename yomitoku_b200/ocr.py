"""OCR: text detection followed by text recognition on one page, behind the reference's `OCR` surface
(reference src/yomitoku/ocr.py:6-63): `OCR(configs={}, device="cuda", visualize=False)` where `configs` may carry a
`"text_detector"` and a `"text_recognizer"` dict of constructor overrides (anything but a dict raises ValueError), and
`ocr(img) -> (OCRSchema, vis)`.  `ocr_aggregate` pairs detections with recognitions positionally - with a quad dropped
by the recognizer the lists mis-align exactly as in the reference (SURVEY.md section 8b, error conventions)."""
from .device_pages import as_device_pages
from .schemas import OCRSchema
from .text_detector import TextDetector
from .text_recognizer import TextRecognizer

_WORD_FIELDS = ("points", "det_score", "content", "rec_score", "direction")


def ocr_aggregate(det_outputs, rec_outputs):
    """One dict per word; stops at the shorter of the five lists (zip), like the reference."""
    columns = (det_outputs.points, det_outputs.scores, rec_outputs.contents, rec_outputs.scores, rec_outputs.directions)
    return [dict(zip(_WORD_FIELDS, row)) for row in zip(*columns)]


class OCR:
    def __init__(self, configs={}, device="cuda", visualize=False):
        if not isinstance(configs, dict):
            raise ValueError("configs must be a dict. See the https://kotaro-kinoshita.github.io/yomitoku-dev/usage/")
        common = {"device": device, "visualize": visualize}
        self.detector = TextDetector(**{**common, **configs.get("text_detector", {})})
        self.recognizer = TextRecognizer(**{**common, **configs.get("text_recognizer", {})})

    def __call__(self, img):
        """img: BGR page (numpy, or on the GPU: a CUDA (H, W, 3) uint8 tensor or a one-page DevicePages, packed once and
        read by both modules).  Returns (OCRSchema, visualisation or None)."""
        dp = as_device_pages(img)
        if dp is not None:
            img = dp
        detected, vis = self.detector(img)
        recognized, vis = self.recognizer(img, detected.points, vis=vis)
        return OCRSchema(words=ocr_aggregate(detected, recognized)), vis
