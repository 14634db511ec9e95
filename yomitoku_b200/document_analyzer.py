"""DocumentAnalyzer: OCR (DBNet -> PARSeq on the GPU, this repo's hot path) merged with a layout analysis into
paragraphs / tables / figures in reading order, behind the reference's constructor / configs-dict / call surface
(reference src/yomitoku/document_analyzer.py:426-678).

What is here
  * the host logic that CALLS the hot path and shapes its input / output (SURVEY.md section 8f rows 3-4):
    `aggregate` (:482-601), the words-in-element assignment with the optional ruby filter (:69-237),
    `split_text_across_cells` (:251-423: detected lines that run across table cells are cut at the cell borders
    BEFORE recognition, so the recognizer sees one crop per cell), reading order (reading_order.py);
  * `analyze_pages`: the batched multi-page form - every page's detection + recognition goes through `BatchedOCR`
    (one packed recognizer call per batch) while the layout analyzer works on the pages in a thread pool.
What is not here: the layout MODELS (RT-DETRv2 layout parser + table structure recognizer, SURVEY.md section 8f row
2).  A layout analyzer with the reference's protocol - `layout(img) -> (LayoutAnalyzerSchema, vis)` - is plugged in
through `layout_analyzer=`; without one the layout is empty (every word becomes its own paragraph, which is exactly
what the reference's `aggregate` produces for an empty layout), and options that need a layout raise instead of
being silently ignored.
"""
import math
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from .ocr import ocr_aggregate
from .reading_order import prediction_reading_order
from .schemas import (DocumentAnalyzerSchema, FigureSchema, LayoutAnalyzerSchema, OCRSchema, ParagraphSchema,
                      TextDetectorSchema)
from .text_detector import TextDetector
from .text_recognizer import TextRecognizer

_HIRAGANA = re.compile(r"^[\u3040-\u309F]+$")
_KATAKANA = re.compile(r"^[\u30A0-\u30FF]+$")


# ------------------------------------------------------------------------------------------------ geometry
def quad_to_xyxy(quad):
    xs = [p[0] for p in quad]
    ys = [p[1] for p in quad]
    return min(xs), min(ys), max(xs), max(ys)


def _intersection(a, b):
    """Integer intersection rectangle of two xyxy boxes or None (utils/misc.py:75-91)."""
    x1, y1 = max(int(a[0]), int(b[0])), max(int(a[1]), int(b[1]))
    x2, y2 = min(int(a[2]), int(b[2])), min(int(a[3]), int(b[3]))
    if max(0, x2 - x1) == 0 or max(0, y2 - y1) == 0:
        return None
    return [x1, y1, x2, y2]


def overlap_ratio(a, b):
    """(share of b's area that lies inside a, intersection) (utils/misc.py:35-50); b's area uses the raw values."""
    inter = _intersection(a, b)
    if inter is None:
        return 0, None
    return ((inter[2] - inter[0]) * (inter[3] - inter[1])) / ((b[2] - b[0]) * (b[3] - b[1])), inter


def is_contained(a, b, threshold=0.8):
    return overlap_ratio(a, b)[0] > threshold


def calc_iou(a, b):
    """Intersection over union (utils/misc.py:182-201): the intersection of the int-truncated boxes, the areas of the
    raw values."""
    inter = _intersection(a, b)
    if inter is None:
        return 0
    i_area = (inter[2] - inter[0]) * (inter[3] - inter[1])
    return i_area / ((a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - i_area)


def _point_segment_dist(px, py, ax, ay, bx, by):
    """Distance of (px, py) to the segment (ax, ay)-(bx, by) (utils/misc.py:208-221)."""
    dx, dy = bx - ax, by - ay
    den = dx * dx + dy * dy
    if den == 0:
        return math.hypot(px - ax, py - ay)
    t = min(1.0, max(0.0, ((px - ax) * dx + (py - ay) * dy) / den))
    return math.hypot(px - (ax + t * dx), py - (ay + t * dy))


def _edge_dists(a1, a2, b1, b2, edge_a, edge_b, vertical):
    """The four corner-to-edge distance pairs between the edge of A at coordinate edge_a spanning [a1, a2] and the edge
    of B at edge_b spanning [b1, b2] (utils/misc.py:224-267).  vertical: the edges are vertical (x = edge)."""
    def d(e_p, p, e0, e1, e):        # corner (e_p, p) of one box to the edge e spanning [e0, e1] of the other
        return (_point_segment_dist(e_p, p, e, e0, e, e1) if vertical else _point_segment_dist(p, e_p, e0, e, e1, e))
    d1 = d(edge_a, a1, b1, b2, edge_b)
    d2 = d(edge_a, a2, b1, b2, edge_b)
    d3 = d(edge_b, b1, a1, a2, edge_a)
    d4 = d(edge_b, b2, a1, a2, edge_a)
    return max(d1, d4), max(d2, d3), max(d3, d4), max(d1, d2)


def _adjacent(a, b, axis, dist_threshold, overlap_ratio_th, ignore_dist_threshold):
    """B lies next to A along `axis` (0: to the right, 1: below); utils/misc.py:299-427 with rule "soft"."""
    c, o = axis, 1 - axis                            # the coordinate that advances / the one that must overlap
    if b[c] < a[c]:
        return False
    if max(0.0, min(a[o + 2], b[o + 2]) - max(a[o], b[o])) < overlap_ratio_th * min(a[o + 2] - a[o], b[o + 2] - b[o]):
        return False
    # corners that touch diagonally are no neighbours: A's far corner vs B's near corner, and the crossed pair
    if math.hypot(a[2] - b[0], a[3] - b[1]) < ignore_dist_threshold:
        return False
    if axis == 0 and math.hypot(a[2] - b[0], a[1] - b[3]) < ignore_dist_threshold:
        return False
    if axis == 1 and math.hypot(a[0] - b[2], a[3] - b[1]) < ignore_dist_threshold:
        return False
    dists = _edge_dists(a[o], a[o + 2], b[o], b[o + 2], a[c + 2], b[c], vertical=(axis == 0))
    return any(v < dist_threshold for v in dists)


def is_right_adjacent(box_a, box_b, dist_threshold=15, overlap_ratio_th=0.1, ignore_dist_threshold=10):
    return _adjacent(box_a, box_b, 0, dist_threshold, overlap_ratio_th, ignore_dist_threshold)


def is_bottom_adjacent(box_a, box_b, dist_threshold=15, overlap_ratio_th=0.1, ignore_dist_threshold=10):
    return _adjacent(box_a, box_b, 1, dist_threshold, overlap_ratio_th, ignore_dist_threshold)


def _side_lengths(quad):
    q = np.array(quad)
    return np.linalg.norm(q[0] - q[1]), np.linalg.norm(q[1] - q[2])


def is_vertical(quad, thresh_aspect=2):
    w, h = _side_lengths(quad)
    return h > w * thresh_aspect


def is_noise(quad, thresh=15):
    w, h = _side_lengths(quad)
    return w < thresh or h < thresh


def judge_page_direction(paragraphs):
    """'vertical' when vertical paragraphs cover more area than horizontal ones (:23-41)."""
    area = {"h": 0, "v": 0}
    for p in paragraphs:
        x1, y1, x2, y2 = p.box
        area["h" if p.direction == "horizontal" else "v"] += (x2 - x1) * (y2 - y1)
    return "vertical" if area["v"] > area["h"] else "horizontal"


# ------------------------------------------------------------------------------------------------ ruby filter
def _mad_threshold(sizes):
    """median - 2 * MAD, or None when it degenerates (:73-94)."""
    med = sorted(sizes)[len(sizes) // 2]
    if med == 0:
        return None
    mad = sorted(abs(s - med) for s in sizes)[len(sizes) // 2]
    if mad == 0:
        return None
    t = med - 2 * mad
    return t if t > 0 else None


def _ruby_size_threshold(sizes, k):
    """Split point of a bimodal size distribution: histogram of log sizes, the valley between the two highest peaks
    when they are separated strongly enough (ratio >= k), else the MAD rule (:97-150)."""
    n = len(sizes)
    if n < 3:
        return None
    logs = [math.log(s) for s in sizes]
    lo_v, hi_v = min(logs), max(logs)
    if hi_v - lo_v < 1e-9:
        return None
    bins = max(8, int(math.sqrt(n)))
    width = (hi_v - lo_v) / bins
    hist = [0] * bins
    for v in logs:
        hist[min(int((v - lo_v) / width), bins - 1)] += 1
    p1 = max(range(bins), key=lambda i: hist[i])
    p2, best = None, -1
    for i in range(bins):
        if abs(i - p1) >= 2 and hist[i] > best:
            p2, best = i, hist[i]
    if p2 is None:
        return _mad_threshold(sizes)
    a, b = min(p1, p2), max(p1, p2)
    if b - a <= 1:
        return _mad_threshold(sizes)
    between = range(a + 1, b)
    low = min(hist[i] for i in between)
    lows = [i for i in between if hist[i] == low]
    valley = lows[len(lows) // 2]
    if (hist[p1] + hist[p2]) / (2 * low + 1e-6) >= k:
        return math.exp(lo_v + (valley + 0.5) * width)
    return _mad_threshold(sizes)


def filter_ruby(words, ruby_threshold):
    """Drops small all-hiragana / all-katakana lines (furigana) from the words of one element (:153-191)."""
    if len(words) <= 1:
        return words
    sizes = [math.sqrt((w.box[2] - w.box[0]) * (w.box[3] - w.box[1])) for w in words]
    valid = [s for s in sizes if s > 0]
    if len(valid) < 2:
        return words
    t = _ruby_size_threshold(valid, ruby_threshold)
    if t is None:
        return words
    kept = []
    for w, s in zip(words, sizes):
        if 0 < s < t:
            text = w.contents.replace(" ", "")
            if _HIRAGANA.match(text) or _KATAKANA.match(text):
                continue
        kept.append(w)
    return kept


# ------------------------------------------------------------------------------------------------ aggregation
def extract_words_within_element(pred_words, element, ignore_ruby=False, ruby_threshold=2.0):
    """Words whose box lies (> 50 %) inside `element.box`, joined in reading order.  Returns (text, direction, flags) with
    flags[i] = word i was used; (None, None, flags) when the element holds no word (:194-237)."""
    flags = [False] * len(pred_words)
    inside = []
    for i, w in enumerate(pred_words):
        box = quad_to_xyxy(w.points)
        if is_contained(element.box, box, threshold=0.5):
            flags[i] = True
            inside.append(ParagraphSchema(box=box, contents=w.content, direction=w.direction, order=0, role=None))
    if not inside:
        return None, None, flags
    n_h = sum(1 for w in inside if w.direction == "horizontal")
    n_v = sum(1 for w in inside if w.direction == "vertical")
    direction = "horizontal" if n_h > n_v else "vertical"
    if ignore_ruby:
        inside = filter_ruby(inside, ruby_threshold)
        if not inside:
            return None, None, flags
    prediction_reading_order(inside, "left2right" if direction == "horizontal" else "right2left")
    inside = sorted(inside, key=lambda w: w.order)
    return "\n".join(w.contents for w in inside), direction, flags


def extract_paragraph_within_figure(paragraphs, figures):
    """Figures with the paragraphs they contain (> 70 %) in reading order, and which paragraphs were taken (:44-66)."""
    out, taken = [], [False] * len(paragraphs)
    for fig in figures:
        inside = []
        for i, p in enumerate(paragraphs):
            if is_contained(fig.box, p.box, threshold=0.7):
                inside.append(p)
                taken[i] = True
        direction = judge_page_direction(inside)
        ordered = prediction_reading_order(inside, "left2right" if direction == "horizontal" else "right2left")
        out.append(FigureSchema(box=fig.box, order=0, direction=direction,
                                paragraphs=sorted(ordered, key=lambda p: p.order)))
    return out, taken


# ------------------------------------------------------------------------------------------------ split across cells
def _words_in_table(det, table, used):
    horizontal, vertical = [], []
    for i, (points, score) in enumerate(zip(det.points, det.scores)):
        if is_contained(table.box, quad_to_xyxy(points), threshold=0.5):
            (vertical if is_vertical(points) else horizontal).append({"points": points, "score": score})
            used[i] = True
    return horizontal, vertical


def _best_line(lines, word):
    """Index of the table row / column the word overlaps most (first one on ties, like list.index(max(...)))."""
    box = quad_to_xyxy(word["points"])
    ratios = [overlap_ratio(line.box, box)[0] for line in lines]
    return ratios.index(max(ratios))


def _cut_words(table, words, lines, along_rows):
    """Cuts every word at the borders of the cells of its row (horizontal words) / column (vertical words) (:303-377)."""
    pts_out, scores_out = [], []
    for word in words:
        k = _best_line(lines, word) + 1
        if along_rows:
            cells = [c for c in table.cells if c.row <= k < c.row + c.row_span]
        else:
            cells = [c for c in table.cells if c.col <= k < c.col + c.col_span]
        p = word["points"]
        for cell in cells:
            _, inter = overlap_ratio(cell.box, quad_to_xyxy(p))
            if inter is None:
                continue
            x1, y1, x2, y2 = inter
            if along_rows:
                q = [[max(p[0][0], x1), p[0][1]], [min(p[1][0], x2), p[1][1]],
                     [min(p[2][0], x2), p[2][1]], [max(p[3][0], x1), p[3][1]]]
            else:
                q = [[p[0][0], max(p[0][1], y1)], [p[1][0], max(p[1][1], y1)],
                     [p[2][0], min(p[2][1], y2)], [p[3][0], min(p[3][1], y2)]]
            if not is_noise(q):
                pts_out.append(q)
                scores_out.append(word["score"])
    return pts_out, scores_out


def split_text_across_cells(det, layout):
    """Detected lines inside a table are replaced by their pieces per cell; the rest keeps its place after them
    (:380-423).  Returns a new TextDetectorSchema (the input is not modified)."""
    used = [False] * len(det.points)
    points, scores = [], []
    for table in layout.tables:
        horizontal, vertical = _words_in_table(det, table, used)
        if not table.rows and horizontal or not table.cols and vertical:
            raise ValueError("max() arg is an empty sequence")      # what the reference's rows.index(max(rows)) raises
        for words, lines, along_rows in ((horizontal, table.rows, True), (vertical, table.cols, False)):
            p, s = _cut_words(table, words, lines, along_rows)
            points += p
            scores += s
    for i, flag in enumerate(used):
        if not flag:
            points.append(det.points[i])
            scores.append(det.scores[i])
    return TextDetectorSchema(points=points, scores=scores)


# ------------------------------------------------------------------------------------------------ the module
def _recursive_update(original, new_data):
    for key, value in new_data.items():
        if isinstance(original.get(key), dict) and isinstance(value, dict):
            _recursive_update(original[key], value)
        else:
            original[key] = value
    return original


def _empty_layout():
    return LayoutAnalyzerSchema(paragraphs=[], tables=[], figures=[])


class DocumentAnalyzer:
    def __init__(self, configs={}, device="cuda", visualize=False, ignore_meta=False, reading_order="auto",
                 split_text_across_cells=False, ignore_ruby=False, ruby_threshold=2.0, layout_analyzer=None):
        default_configs = {
            "ocr": {
                "text_detector": {"device": device, "visualize": visualize},
                "text_recognizer": {"device": device, "visualize": visualize},
            },
            "layout_analyzer": {
                "layout_parser": {"device": device, "visualize": visualize},
                "table_structure_recognizer": {"device": device, "visualize": visualize},
            },
        }
        if isinstance(configs, dict):
            _recursive_update(default_configs, configs)
        else:
            raise ValueError("configs must be a dict. See the https://kotaro-kinoshita.github.io/yomitoku/module/#config")
        self.text_detector = TextDetector(**default_configs["ocr"]["text_detector"])
        self.text_recognizer = TextRecognizer(**default_configs["ocr"]["text_recognizer"])
        # layout half: by default the reference's LayoutAnalyzer (RT-DETRv2 layout parser + table structure recognizer,
        # layout_analyzer.py:7-36) on the device engine; any object with its `layout(img) -> (LayoutAnalyzerSchema, vis)`
        # protocol can be passed instead; False = no layout (every word becomes its own paragraph)
        if layout_analyzer is None:
            from .layout_analyzer import LayoutAnalyzer
            layout_analyzer = LayoutAnalyzer(configs=default_configs["layout_analyzer"], device=device, visualize=visualize)
        self.layout = layout_analyzer or None
        if self.layout is None and split_text_across_cells:
            raise NotImplementedError("split_text_across_cells needs table cells: it cannot be combined with "
                                      "layout_analyzer=False")
        self.visualize = visualize
        self.ignore_meta = ignore_meta
        self.reading_order = reading_order
        self.split_text_across_cells = split_text_across_cells
        self.ignore_ruby = ignore_ruby
        self.ruby_threshold = ruby_threshold
        self._batched = None

    # -------------------------------------------------------------------------------------- aggregation
    def aggregate(self, ocr_res, layout_res, img=None):
        """words + layout -> paragraphs / tables / figures with contents and reading order (:482-601)."""
        words = ocr_res.words
        used = [False] * len(words)
        kw = dict(ignore_ruby=self.ignore_ruby, ruby_threshold=self.ruby_threshold)
        for table in layout_res.tables:
            for cell in table.cells:
                text, _, flags = extract_words_within_element(words, cell, **kw)
                cell.contents = "" if text is None else text
                used = [a or b for a, b in zip(used, flags)]
        paragraphs = []
        for region in layout_res.paragraphs:
            text, direction, flags = extract_words_within_element(words, region, **kw)
            if text is None:
                continue
            used = [a or b for a, b in zip(used, flags)]
            paragraphs.append(ParagraphSchema(contents=text, box=region.box, direction=direction, order=0,
                                              role=region.role))
        for word, flag in zip(words, used):       # words no layout region claimed stand alone
            if not flag:
                paragraphs.append(ParagraphSchema(contents=word.content, box=quad_to_xyxy(word.points),
                                                  direction=word.direction, order=0, role=None))
        figures, in_figure = extract_paragraph_within_figure(paragraphs, layout_res.figures)
        paragraphs = [p for p, f in zip(paragraphs, in_figure) if not f]
        page_direction = judge_page_direction(paragraphs)
        headers = [p for p in paragraphs if p.role == "page_header" and not self.ignore_meta]
        footers = [p for p in paragraphs if p.role == "page_footer" and not self.ignore_meta]
        body = [p for p in paragraphs if p.role is None or p.role == "section_headings"]
        elements = body + list(layout_res.tables) + figures
        prediction_reading_order(headers, "left2right")
        prediction_reading_order(footers, "left2right")
        if self.reading_order == "auto":
            order = "right2left" if page_direction == "vertical" else "top2bottom"
        else:
            order = self.reading_order
        prediction_reading_order(elements, order, img)
        for e in elements:
            e.order += len(headers)
        for f in footers:
            f.order += len(elements) + len(headers)
        return {"paragraphs": sorted(headers + body + footers, key=lambda p: p.order),
                "tables": sorted(layout_res.tables, key=lambda t: t.order),
                "figures": sorted(figures, key=lambda f: f.order),
                "words": words}

    # -------------------------------------------------------------------------------------- one page
    def _detect_and_recognize(self, img):
        det, vis = self.text_detector(img)
        rec, vis = self.text_recognizer(img, det.points, vis=vis)
        return det, rec, vis

    def _layout(self, img):
        if self.layout is None:
            return _empty_layout(), None
        return self.layout(img)

    def __call__(self, img):
        """(DocumentAnalyzerSchema, ocr_vis, layout_vis) like the reference (:603-678): detection -> recognition in one
        worker thread, the layout analyzer in another; with split_text_across_cells the recognizer waits for the layout
        because its crops are the detected lines cut at the cell borders."""
        with ThreadPoolExecutor(max_workers=2) as ex:
            if self.split_text_across_cells:
                f_det = ex.submit(self.text_detector, img)
                f_lay = ex.submit(self._layout, img)
                (det, vis), (layout, layout_vis) = f_det.result(), f_lay.result()
                det = split_text_across_cells(det, layout)
                rec, ocr_vis = self.text_recognizer(img, det.points, vis=vis)
            else:
                f_ocr = ex.submit(self._detect_and_recognize, img)
                f_lay = ex.submit(self._layout, img)
                (det, rec, ocr_vis), (layout, layout_vis) = f_ocr.result(), f_lay.result()
        ocr = OCRSchema(words=ocr_aggregate(det, rec))
        return DocumentAnalyzerSchema(**self.aggregate(ocr, layout, img)), ocr_vis, layout_vis

    # -------------------------------------------------------------------------------------- many pages
    def analyze_pages(self, pages, layouts=None):
        """Batched multi-page form (SURVEY.md section 8f row 3): `pages` = list of BGR pages, of one size or of many.  Detection and
        recognition of ALL pages run through `pipeline.BatchedOCR` (detector batches, one packed recognizer call,
        host post-processing in the process pool) while the layout analyzer works through the pages in a thread pool;
        then `aggregate` per page.  `layouts` (optional list of LayoutAnalyzerSchema) replaces the layout analyzer.
        With split_text_across_cells the detected lines are cut at the cell borders between the two device stages.
        Returns a list of DocumentAnalyzerSchema."""
        from .pipeline import BatchedOCR
        if self._batched is None:
            self._batched = BatchedOCR(self.text_detector, self.text_recognizer)
        ocr = self._batched
        with ThreadPoolExecutor(max_workers=max(1, min(4, len(pages)))) as ex:
            if layouts is None and hasattr(self.layout, "analyze_pages"):
                # the built-in LayoutAnalyzer: all pages' layouts in one device batch (its own thread: the OCR stages
                # below run meanwhile)
                f_all = ex.submit(self.layout.analyze_pages, pages)

                class _One:
                    def __init__(self, i):
                        self.i = i

                    def result(self):
                        return f_all.result()[self.i], None
                f_lay = [_One(i) for i in range(len(pages))]
            elif layouts is None:
                f_lay = [ex.submit(self._layout, p) for p in pages]
            if self.split_text_across_cells:
                dets = self.text_detector.detect_pages(pages)
                lay = layouts if layouts is not None else [f.result()[0] for f in f_lay]
                quads = [split_text_across_cells(d, l) for d, l in zip(dets, lay)]
                results = ocr(pages, quads_override=[q.points for q in quads])
                for r, q in zip(results, quads):            # det scores of the cut lines (the override carries 1.0)
                    for w, s in zip(r.words, q.scores):
                        w.det_score = float(s)
            else:
                results = ocr(pages)
                lay = layouts if layouts is not None else [f.result()[0] for f in f_lay]
        return [DocumentAnalyzerSchema(**self.aggregate(r, l, p)) for r, l, p in zip(results, lay, pages)]
