"""Host half of the table semantic parser (yomitoku_b200/table_semantic_parser.py, grid_parser.py, kv_parser.py and
the schemas) against tests/golden/tsp_ref.json: the reference's own TableSemanticParser run on the same seeded model
outputs.  The word assignment runs as the Python loop of oracle/table_semantic.py here; the GPU tests run the same
cases through the CUDA kernel."""
import ctypes
import os

import numpy as np
import pytest

from oracle import table_semantic as ots
from tsp_cases import case_id, load_cases, model_outputs, oracle_assign, standin_parser

CASES = load_cases()


def _parse_host(case, monkeypatch):
    from yomitoku_b200 import table_semantic_parser as tsp
    monkeypatch.setattr(tsp, "assign_best_overlap", oracle_assign)
    res, vis_layout, vis_ocr = standin_parser(case, device="cpu")(np.zeros((8, 8, 3), np.uint8),
                                                                  grid_only=case["grid_only"], kv_only=case["kv_only"])
    assert vis_layout is None and vis_ocr is None
    return res


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_host_restatement_equals_reference(case, monkeypatch):
    res = _parse_host(case, monkeypatch)
    assert ots.canonical_kv(res.model_dump()) == ots.canonical_kv(case["output"])


def test_goldens_cover_the_cases_the_parser_distinguishes():
    outs = [c["output"] for c in CASES]
    tables = [t for o in outs for t in o["tables"]]
    assert any(t["grids"] for t in tables) and any(t["kv_items"] for t in tables)
    assert any(g["n_row"] > 1 and any(len(h) > 1 for h in g["col_headers"]) for t in tables for g in t["grids"])
    assert any(c["row_span"] and c["row_span"] > 1 for t in tables for c in t["cells"].values())
    assert any(c["col_span"] and c["col_span"] > 1 for t in tables for c in t["cells"].values())
    assert any(len(kv["key"]) > 1 for t in tables for kv in t["kv_items"])
    assert any(kv["key"] == [] for t in tables for kv in t["kv_items"])
    assert any(c["role"] == "group" for t in tables for c in t["cells"].values())
    assert any(c["role"] == "empty" for t in tables for c in t["cells"].values())
    # a table with fewer than two cells became an empty paragraph
    assert any(p["box"] == [890, 890, 1010, 950] and p["score"] == 1.0 for o in outs for p in o["paragraphs"])
    assert {(c["grid_only"], c["kv_only"]) for c in CASES} == {(False, False), (True, False), (False, True)}


def _assignment_inputs(case):
    from yomitoku_b200.document_analyzer import quad_to_xyxy
    ocr, layout, tables = model_outputs(case)
    words = np.array([quad_to_xyxy(w.points) for w in ocr.words], np.float64)
    lists = [t.cells for t in tables] + [layout.paragraphs]
    elems = np.array([e.box for lst in lists for e in lst], np.float64)
    skip = np.array([e.role == "group" for lst in lists for e in lst], np.uint8)
    groups, e0 = [], 0
    for lst in lists:
        groups.append((0, len(words), e0, e0 + len(lst)))
        e0 += len(lst)
    return words, elems, skip, np.array(groups, np.int32)


def test_oracle_assignment_rules():
    """The oracle's loop (the kernel tests' reference; the goldens above pin it through the element texts): one result
    per (group, word), first maximum wins, group roles never take a word, shares below the threshold are dropped."""
    for case in CASES:
        words, elems, skip, groups = _assignment_inputs(case)
        best, ratio = ots.assign_best_overlap(words, elems, skip, groups)
        assert len(best) == len(words) * len(groups)
        assert all(b == -1 or r >= 0.2 for b, r in zip(best, ratio))
    # a word split evenly between two cells goes to the first of them
    best, ratio = ots.assign_best_overlap([[90, 0, 110, 10]], [[0, 0, 100, 10], [100, 0, 200, 10]], [0, 0],
                                          [(0, 1, 0, 2)])
    assert best == [0] and ratio == [0.5]
    # a group-role element never takes a word; a share at the threshold is kept, below it dropped
    best, _ = ots.assign_best_overlap([[0, 0, 10, 10], [0, 0, 10, 10]], [[0, 0, 10, 10], [0, 0, 2, 10]], [1, 0],
                                      [(0, 1, 0, 2), (1, 2, 1, 2)], overlap_th=0.2)
    assert best == [1, 1]
    best, _ = ots.assign_best_overlap([[0, 0, 10, 10]], [[0, 0, 1, 10]], [0], [(0, 1, 0, 1)])
    assert best == [-1]


def test_schema_round_trip(monkeypatch, tmp_path):
    from yomitoku_b200.schemas import TableSemanticParserSchema
    res = _parse_host(CASES[4], monkeypatch)
    path = os.path.join(str(tmp_path), "tsp.json")
    res.to_json(path)
    back = TableSemanticParserSchema.load_json(path)
    assert back.model_dump() == res.model_dump()
    d = res.to_dict()
    assert set(d) == {t.id for t in res.tables}
    assert all(set(v) == {"kv_items", "grids"} for v in d.values())
    res.to_csv(str(tmp_path / "csv"))
    grids = [(t.id, g.id) for t in res.tables for g in t.grids]
    assert grids and all(os.path.exists(str(tmp_path / "csv" / ("table_%s_%s.csv" % ids))) for ids in grids)
    assert res.find_table_by_id(res.tables[0].id) is res.tables[0]


def test_template_round_trip(monkeypatch, tmp_path):
    """save_template_json -> edit a cell -> load_template_json overrides that cell's text and keeps the structure."""
    import json
    res = _parse_host(CASES[4], monkeypatch)
    path = str(tmp_path / "template.json")
    res.save_template_json(path)
    with open(path) as f:
        tmpl = json.load(f)
    table = tmpl["tables"][0]
    cid = next(iter(table["cells"]))
    table["cells"][cid]["contents"] = "EDITED"
    with open(path, "w") as f:
        json.dump(tmpl, f)
    fresh = _parse_host(CASES[4], monkeypatch)
    fresh.load_template_json(path)
    assert fresh.tables[0].cells[cid].contents == "EDITED"
    assert [kv.model_dump() for kv in fresh.tables[0].kv_items] == [kv.model_dump() for kv in res.tables[0].kv_items]
    key_text = res.tables[0].cells[res.tables[0].kv_items[0].key[0]].contents if res.tables[0].kv_items[0].key else ""
    if key_text:
        assert res.search_kv_items_by_key(key_text)


def test_c_symbol_exported():
    from yomitoku_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libytk_b200.so is not built")
    lib = ctypes.CDLL(_lib.LIB_PATH)
    assert hasattr(lib, "ytk_op_assign_best_overlap_f64")
