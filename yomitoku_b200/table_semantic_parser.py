"""TableSemanticParser: tables of forms and documents as grids and key-value items, behind the reference's surface
(reference src/yomitoku/table_semantic_parser.py:623-991): `TableSemanticParser(configs={}, device="cuda",
visualize=False)` with the config keys "table_detector", "table_cell_parser", "text_detector" and "text_recognizer",
and `parser(img, template=None, id=None, grid_only=False, kv_only=False) -> (TableSemanticParserSchema, vis_layout,
vis_ocr)`.

The four models run on the device: DBNet and PARSeq (text), the RT-DETRv2 layout parser (tables and paragraphs) and
the cell detector (cells, kv_item and grid regions of every table crop).  The word-to-cell assignment, a loop over
every word and every cell in the reference, is one CUDA launch for all tables and paragraphs
(`models.assign_best_overlap`, csrc/table_ops.cu); the reading order inside each cell, the grid and key-value
structure (grid_parser.py, kv_parser.py) and the ids are host code like in the reference.  `parse_pages` is the
batched form: the pages go to the device once, text and layout run side by side, one cell-detector forward covers
the tables of all pages and one launch assigns all their words.
"""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from .base import logger
from .device_pages import as_device_pages, device_pages, host_page, single_page
from .document_analyzer import is_contained, quad_to_xyxy
from .grid_parser import parse_grid_from_bottom_up
from .kv_parser import parse_kv_items
from .layout_parser import LayoutParser
from .models import assign_best_overlap
from .ocr import ocr_aggregate
from .reading_order import prediction_reading_order
from .schemas import (Element, OCRSchema, ParagraphSchema, TableSemanticContentsSchema, TableSemanticParserSchema)
from .table_cell_detector import CellDetector
from .text_detector import TextDetector
from .text_recognizer import TextRecognizer

__all__ = ["TableSemanticParser", "aggregate_pages", "sort_cells", "replace_table_to_paragraphs"]

_VALUE_ROLES = ("cell", "header", "empty")


# ------------------------------------------------------------------------------------------------ words into elements
def aggregate_pages(pages, overlap_th=0.2, device="cuda"):
    """pages: list of (words, [element lists]) - the WordPredictions of a page and the lists whose elements take its
    words (one table's cells, the page's paragraphs).  Every word goes to the element of its list that covers the
    largest share of it (one launch for every list of every page); each element's `contents` becomes its words in
    reading order (reference aggregate :683-732)."""
    word_boxes, elem_boxes, skip, groups, spans = [], [], [], [], []
    for words, lists in pages:
        w0 = len(word_boxes)
        word_boxes.extend(quad_to_xyxy(w.points) for w in words)
        for elements in lists:
            e0 = len(elem_boxes)
            elem_boxes.extend(e.box for e in elements)
            skip.extend(e.role == "group" for e in elements)
            groups.append((w0, len(word_boxes), e0, len(elem_boxes)))
            spans.append((words, elements, e0))
    best, _ = assign_best_overlap(np.asarray(word_boxes, np.float64).reshape(-1, 4),
                                  np.asarray(elem_boxes, np.float64).reshape(-1, 4), np.asarray(skip, np.uint8),
                                  np.asarray(groups, np.int32).reshape(-1, 4), overlap_th, device)
    o = 0
    for words, elements, e0 in spans:
        taken = [[] for _ in elements]
        for w, b in zip(words, best[o:o + len(words)]):
            if b >= 0:
                box = quad_to_xyxy(w.points)
                taken[b - e0].append(ParagraphSchema(box=box, contents=w.content, direction=w.direction, order=0,
                                                     role=None))
        o += len(words)
        for element, contained in zip(elements, taken):
            _join_contents(element, contained)


def _join_contents(element, contained):
    """The element's text: its words in the reading order of their majority direction, newlines removed."""
    if not contained:
        element.contents = ""
        return
    dirs = [w.direction for w in contained]
    direction = "horizontal" if dirs.count("horizontal") >= dirs.count("vertical") else "vertical"
    prediction_reading_order(contained, "left2right" if direction == "horizontal" else "right2left")
    contained = sorted(contained, key=lambda x: x.order)
    element.contents = "\n".join(w.contents for w in contained).replace("\n", "").strip()


# ------------------------------------------------------------------------------------------------ structure helpers
def _split_nodes_with_role(cells):
    """role -> cells, with "header", "cell" and "empty" always present (reference :40-55)."""
    nodes = {"header": [], "cell": [], "empty": []}
    for cell in cells:
        nodes.setdefault(cell.role, []).append(cell)
    return nodes


def _region_cell_ids(region, cells, threshold=0.5):
    return {c.id for c in cells if is_contained(region.box, c.box, threshold=threshold)}


def _resolve_overlapping_regions(grid_regions, kv_regions, value_cells, conflict_ratio_th=0.5):
    """Regions the model predicted twice (reference :199-268): of two grids sharing most of the smaller one's cells
    the higher score stays; of a grid and a kv_item region sharing most of the smaller one's cells, the one holding
    more cells stays, the grid on a tie."""
    grid_sets = [_region_cell_ids(g, value_cells) for g in grid_regions]
    kv_sets = [_region_cell_ids(k, value_cells) for k in kv_regions]
    drop_grid, drop_kv, kept = set(), set(), []
    for gi in sorted(range(len(grid_regions)), key=lambda i: getattr(grid_regions[i], "score", 1.0), reverse=True):
        dup = False
        for gj in kept:
            denom = min(len(grid_sets[gi]), len(grid_sets[gj]))
            if denom and len(grid_sets[gi] & grid_sets[gj]) / denom >= conflict_ratio_th:
                dup = True
                break
        if dup:
            drop_grid.add(gi)
        else:
            kept.append(gi)
    for gi in range(len(grid_regions)):
        for ki in range(len(kv_regions)):
            if gi in drop_grid or ki in drop_kv:
                continue
            inter = grid_sets[gi] & kv_sets[ki]
            denom = min(len(grid_sets[gi]), len(kv_sets[ki]))
            if not inter or denom == 0 or len(inter) / denom < conflict_ratio_th:
                continue
            if len(grid_sets[gi]) >= len(kv_sets[ki]):
                drop_kv.add(ki)
            else:
                drop_grid.add(gi)
    return ([g for i, g in enumerate(grid_regions) if i not in drop_grid],
            [k for i, k in enumerate(kv_regions) if i not in drop_kv])


def _gap_valley_tol(coords, min_tol=8.0):
    """Split distance for clustering coordinates into rows: the middle of the largest relative jump between the sorted
    neighbour gaps (min_tol leading), so jitter of a few pixels stays on one side of it (reference :390-411)."""
    coords = sorted(coords)
    gaps = sorted(b - a for a, b in zip(coords, coords[1:]))
    if not gaps or gaps[-1] <= min_tol:
        return min_tol
    gaps = [min_tol] + gaps
    best_i, best_ratio = 0, 0.0
    for i in range(len(gaps) - 1):
        ratio = (gaps[i + 1] + 1) / (gaps[i] + 1)
        if ratio >= best_ratio:
            best_ratio, best_i = ratio, i
    return (gaps[best_i] + gaps[best_i + 1]) / 2


def _cluster_centers(coords, tol):
    """Sorted coordinates split where the gap exceeds tol; the mean of each run (reference :414-426)."""
    coords = sorted(coords)
    centers, run = [], [coords[0]]
    for v in coords[1:]:
        if v - run[-1] > tol:
            centers.append(sum(run) / len(run))
            run = [v]
        else:
            run.append(v)
    centers.append(sum(run) / len(run))
    return centers


def sort_cells(cells):
    """Cells in reading order with position ids: r<row>c<col> for cell / header / empty (row from clustering the top
    edges, col = rank from the left inside the row), grp<i> for groups.  Returns (cells, old id -> new id)
    (reference :433-479)."""
    cells = list(cells)
    if not cells:
        return cells, {}
    min_height = min(c.box[3] - c.box[1] for c in cells)
    values = sorted((c for c in cells if c.role in _VALUE_ROLES), key=lambda c: (c.box[1] // min_height, c.box[0]))
    groups = sorted((c for c in cells if c.role == "group"), key=lambda c: (c.box[1], c.box[0]))
    remap = {}
    if values:
        ys = [c.box[1] for c in values]
        centers = _cluster_centers(ys, _gap_valley_tol(ys))
        rows = {}
        for cell in values:
            rows.setdefault(min(range(len(centers)), key=lambda i: abs(centers[i] - cell.box[1])), []).append(cell)
        for r, row_cells in rows.items():
            row_cells.sort(key=lambda c: c.box[0])
            for col, cell in enumerate(row_cells):
                remap[cell.id] = "r%dc%d" % (r, col)
                cell.id = remap[cell.id]
    for i, cell in enumerate(groups):
        remap[cell.id] = "grp%d" % i
        cell.id = remap[cell.id]
    return values + groups, remap


def _sort_elements(elements, prefix):
    """Reading order by (top // smallest height, left); ids <prefix>0, <prefix>1, ... (reference :482-492)."""
    if not elements:
        return elements
    min_height = min(e.box[3] - e.box[1] for e in elements)
    elements = sorted(elements, key=lambda e: (e.box[1] // min_height, e.box[0]))
    for i, e in enumerate(elements):
        e.id = "%s%d" % (prefix, i)
    return elements


def _assign_ids(info):
    """Grid ids g<i>, kv ids kv<i>, cell position ids, and every reference to a cell renamed (reference :495-534)."""
    for i, grid in enumerate(info["grids"]):
        grid.id = "g%d" % i
    for i, kv in enumerate(info["kv_items"]):
        kv.id = "kv%d" % i
    cells, remap = sort_cells(info["cells"].values())
    info["cells"] = {c.id: c for c in cells}
    for kv in info["kv_items"]:
        kv.key = [remap[k] for k in kv.key]
        kv.value = remap[kv.value]
    for grid in info["grids"]:
        grid.data = [[remap[c] if c is not None else None for c in row] for row in grid.data]
        grid.col_headers = [[remap[c] if c is not None else None for c in col] for col in grid.col_headers]


def replace_table_to_paragraphs(tables, paragraphs):
    """Tables with fewer than two cell / header cells become empty paragraphs (appended to `paragraphs`); the others
    are returned (reference :734-755)."""
    kept = []
    for table in tables:
        if sum(c.role in ("cell", "header") for c in table.cells) < 2:
            paragraphs.append(Element(id=None, box=table.box, contents="", score=1.0, role=None))
        else:
            kept.append(table)
    return kept


def _table_contents(i, table, grid_only, kv_only, structured):
    """One detected table (cells with their texts) -> TableSemanticContentsSchema (reference __call__ :847-969)."""
    cells = {c.id: c for c in table.cells}
    info = {"id": "t%d" % i, "box": table.box, "cells": {}, "style": "border", "kv_items": [], "grids": []}
    if structured:
        values = [c for c in table.cells if c.role in _VALUE_ROLES]
        grid_regions = [] if kv_only else list(table.grid_regions)
        kv_regions = [] if grid_only else list(table.kv_regions)
        grid_regions, kv_regions = _resolve_overlapping_regions(grid_regions, kv_regions, values)
        claimed = set()
        for region in grid_regions:
            inside = [c for c in values if is_contained(region.box, c.box, threshold=0.5)]
            if not inside:
                continue
            result = parse_grid_from_bottom_up(cells, _split_nodes_with_role(inside))
            if result is None:
                continue
            grid, grid_cells, _ = result
            info["grids"].append(grid)
            info["cells"].update(grid_cells)
            claimed.update(c.id for c in inside)
        remaining = [c for c in values if c.id not in claimed]
        if remaining:
            for k, region in enumerate(kv_regions):
                region.id = "kvr%d" % k
            kv_items, _, kv_cells = parse_kv_items(_split_nodes_with_role(remaining), cells, kv_regions)
            info["kv_items"].extend(kv_items)
            info["cells"].update(kv_cells)
    for cell in cells.values():
        if cell.id not in info["cells"]:
            info["cells"][cell.id] = cell
    info["kv_items"] = sorted(info["kv_items"], key=lambda kv: info["cells"][kv.value].box[1])
    info["grids"] = sorted(info["grids"], key=lambda g: g.box[1])
    _assign_ids(info)
    return TableSemanticContentsSchema(**info)


def semantic_page(words, tables, paragraphs, template=None, grid_only=False, kv_only=False):
    """Everything after the models and the word assignment for one page: tables -> TableSemanticContentsSchema in
    reading order, paragraphs in reading order, the template applied (reference __call__ :841-981)."""
    contents = [_table_contents(i, t, grid_only, kv_only, template is None) for i, t in enumerate(tables)]
    result = TableSemanticParserSchema(tables=_sort_elements(contents, "t"), paragraphs=_sort_elements(paragraphs, "p"),
                                       words=words)
    if template is not None:
        result.load_template_json(template)
    return result


# ------------------------------------------------------------------------------------------------ the module
class TableSemanticParser:
    def __init__(self, configs={}, device="cuda", visualize=False):
        if not isinstance(configs, dict):
            raise ValueError("configs must be a dict. See the https://kotaro-kinoshita.github.io/yomitoku/module/#config")
        kwargs = {"table_detector": {"device": device, "visualize": visualize},
                  "table_cell_parser": {"device": device, "visualize": visualize},
                  "text_detector": {"device": device}, "text_recognizer": {"device": device}}
        for key in kwargs:
            kwargs[key].update(configs.get(key, {}))
        self.layout_parser = LayoutParser(**kwargs["table_detector"])
        self.cell_detector = CellDetector(**kwargs["table_cell_parser"])
        self.text_detector = TextDetector(**kwargs["text_detector"])
        self.text_recognizer = TextRecognizer(**kwargs["text_recognizer"])
        self.device = device
        self.visualize = visualize
        self._batched = None
        if visualize:
            logger.warning("TableSemanticParser(visualize=True): layouts and texts are not drawn (the reference's "
                           "visualisers are not part of yomitoku_b200); vis_layout and vis_ocr are copies of the page")

    def aggregate(self, ocr_res, *element_lists, overlap_th=0.2):
        """The texts of the elements of every list (one table's cells, the paragraphs) from the page's words, in one
        device launch (reference :683-732 takes one list per call)."""
        aggregate_pages([(ocr_res.words, element_lists)], overlap_th, self.device)

    def replace_table_to_paragraphs(self, tables, paragraphs):
        return replace_table_to_paragraphs(tables, paragraphs)

    def _vis(self, img):
        if not self.visualize:
            return None, None
        page = host_page(img)
        return page.copy(), page.copy()

    def __call__(self, img, template=None, id=None, grid_only=False, kv_only=False):
        """img: BGR page (numpy, or on the GPU: a CUDA (H, W, 3) uint8 tensor or a one-page DevicePages, packed once
        and read by all four models).  Returns (TableSemanticParserSchema, vis_layout, vis_ocr); the visualisations
        are None unless visualize=True."""
        dp = as_device_pages(img)
        if dp is not None:
            img = single_page(dp, "TableSemanticParser")
        with ThreadPoolExecutor(max_workers=2) as ex:
            f_det = ex.submit(self.text_detector, img)
            f_lay = ex.submit(self.layout_parser, img)
            (det, _), (layout, _) = f_det.result(), f_lay.result()
        tables = self.cell_detector(img, list(layout.tables))
        tables = replace_table_to_paragraphs(tables, layout.paragraphs)
        rec, _ = self.text_recognizer(img, det.points)
        ocr = OCRSchema(words=ocr_aggregate(det, rec))
        aggregate_pages([(ocr.words, [t.cells for t in tables] + [layout.paragraphs])], device=self.device)
        result = semantic_page(ocr.words, tables, layout.paragraphs, template, grid_only, kv_only)
        return (result,) + self._vis(img)

    def parse_pages(self, pages, grid_only=False, kv_only=False):
        """Batched multi-page form: `pages` = list of BGR numpy pages of any sizes, pages already on the GPU (a list of
        CUDA (H, W, 3) uint8 tensors, an (n, H, W, 3) CUDA tensor) or a DevicePages.  The pages are packed on the device
        once; text detection and recognition of all pages (`pipeline.BatchedOCR`) run while the layout parser takes
        them in one batch; then one cell-detector forward covers the tables of all pages and one launch assigns the
        words of all pages.  Returns a list of TableSemanticParserSchema, each equal to `__call__` on its page."""
        from .pipeline import BatchedOCR
        if self._batched is None:
            self._batched = BatchedOCR(self.text_detector, self.text_recognizer)
        dp = as_device_pages(pages)
        if dp is None and torch.device(self.device).type == "cuda":
            dev = self.layout_parser.model.cuda_device()
            dp = device_pages([torch.from_numpy(np.ascontiguousarray(p)).to(dev) for p in pages])
        src = dp if dp is not None else pages
        with ThreadPoolExecutor(max_workers=1) as ex:
            f_lay = ex.submit(self.layout_parser.parse_pages, src)
            ocr = self._batched(src)
            layouts = f_lay.result()
        tables = self.cell_detector.detect_pages(src, [list(lay.tables) for lay in layouts])
        tables = [replace_table_to_paragraphs(t, lay.paragraphs) for t, lay in zip(tables, layouts)]
        aggregate_pages([(r.words, [t.cells for t in ts] + [lay.paragraphs]) for r, ts, lay in zip(ocr, tables, layouts)],
                        device=self.device)
        return [semantic_page(r.words, ts, lay.paragraphs, None, grid_only, kv_only)
                for r, ts, lay in zip(ocr, tables, layouts)]

    def extract_pages(self, pages, schema, normalize=True, simple=False):
        """The fields of an extraction schema (extractor.py; an ExtractionSchema, a dict in its form or a YAML path)
        from every page: `parse_pages` on the batch, then `extractor.extract` on each page's result.  Returns one dict
        per page, each equal to `extract(self(page)[0], schema, normalize, simple)`."""
        from .extractor import as_schema, extract
        schema = as_schema(schema)
        return [extract(r, schema, normalize, simple) for r in self.parse_pages(pages)]
