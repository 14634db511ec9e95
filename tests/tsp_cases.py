"""The cases of tests/golden/tsp_ref.json (made by tests/golden/make_golden_tsp.py from the reference's own table
semantic parser) as the product's model outputs, and a TableSemanticParser whose four models are stand-ins returning
them, for the host and GPU tests of the table semantic parser."""
import json
import os

import numpy as np

from oracle import table_semantic as ots

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tsp_ref.json")


def load_cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def case_id(case):
    return "%d-%s%s" % (case["seed"], case["kind"], "-grid_only" if case["grid_only"] else
                        "-kv_only" if case["kv_only"] else "")


def model_outputs(case):
    """(OCRSchema, LayoutParserSchema, tables as CellDetector returns them) of a case."""
    from yomitoku_b200.schemas import (CellSchema, Element, LayoutParserSchema, OCRSchema, RegionSchema,
                                       TableDetectorSchema)
    inp = case["input"]
    ocr = OCRSchema(words=inp["words"])
    layout = LayoutParserSchema(paragraphs=[Element(id=None, contents=None, **p) for p in inp["paragraphs"]],
                                tables=[Element(id=None, box=t["box"], score=0.9, role=None) for t in inp["tables"]],
                                figures=[])
    tables = [TableDetectorSchema(
        id=None, box=t["box"], role=t["role"],
        cells=[CellSchema(id=c["id"], box=c["box"], role=c["role"], contents=None, row=None, col=None, row_span=None,
                          col_span=None) for c in t["cells"]],
        kv_regions=[RegionSchema(id=None, role="kv_item", **r) for r in t["kv_regions"]],
        grid_regions=[RegionSchema(id=None, role="grid", **r) for r in t["grid_regions"]]) for t in inp["tables"]]
    return ocr, layout, tables


def oracle_assign(word_boxes, elem_boxes, elem_skip, groups, overlap_th=0.2, device=None):
    """models.assign_best_overlap restated by the Python loop of oracle/table_semantic.py."""
    best, ratio = ots.assign_best_overlap(word_boxes, elem_boxes, elem_skip, np.asarray(groups).reshape(-1, 4),
                                          overlap_th)
    return np.asarray(best, np.int32), np.asarray(ratio, np.float64)


def standin_parser(case, device="cuda"):
    """A TableSemanticParser whose text detector, recognizer, layout parser and cell detector return the case's model
    outputs; everything after them is the product's."""
    from yomitoku_b200 import TableSemanticParser
    from yomitoku_b200.schemas import TextDetectorSchema, TextRecognizerSchema
    ocr, layout, tables = model_outputs(case)
    words = ocr.words
    p = object.__new__(TableSemanticParser)
    p.text_detector = lambda img: (TextDetectorSchema(points=[w.points for w in words],
                                                      scores=[w.det_score for w in words]), None)
    p.text_recognizer = lambda img, points: (TextRecognizerSchema(
        contents=[w.content for w in words], directions=[w.direction for w in words],
        scores=[w.rec_score for w in words], points=points), None)
    p.layout_parser = lambda img: (layout.model_copy(deep=True), None)
    p.cell_detector = lambda img, t: [x.model_copy(deep=True) for x in tables]
    p.device, p.visualize, p._batched = device, False, None
    return p
