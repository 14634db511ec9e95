"""The table semantic parser on the GPU: the word-to-element assignment kernel (csrc/table_ops.cu) bit for bit against
the Python loop of oracle/table_semantic.py, the parser end to end through the kernel against the reference's
goldens, and the device page forms (numpy vs CUDA page, parse_pages vs per-page calls) with seeded weights."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import rtdetr as R
from oracle import table_semantic as ots
from trained_head import load_trained_head
from tsp_cases import case_id, load_cases, standin_parser
from yomitoku_b200 import TableSemanticParser, _lib
from yomitoku_b200.models import OVERLAP_GROUP_DTYPE, assign_best_overlap
from yomitoku_b200.schemas import Element
from yomitoku_b200.synth import synthetic_page

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = load_cases()


# ------------------------------------------------------------------------------------------------ kernel
def _random_case(seed, n_groups, max_words, max_elems, tile_big=False):
    """Seeded boxes with negative and fractional coordinates, zero-width words, grid-aligned cells (ties: a word half
    in each of two cells) and shares exactly at 0.2, groups that share words, empty groups."""
    rng = np.random.default_rng(seed)
    words, elems, skip, groups = [], [], [], []
    for g in range(n_groups):
        nw = 0 if g % 7 == 3 else int(rng.integers(1, max_words + 1))
        ne = 0 if g % 11 == 5 else (1500 if tile_big and g == 0 else int(rng.integers(1, max_elems + 1)))
        w0, e0 = len(words), len(elems)
        for _ in range(ne):
            if rng.random() < 0.5:                  # on a 50 px lattice: ties and exact shares
                x, y = rng.integers(-4, 20) * 50, rng.integers(-4, 20) * 50
                elems.append([x, y, x + 50 * rng.integers(1, 3), y + 50])
            else:
                x, y = rng.uniform(-300, 1000, 2)
                elems.append([x, y, x + rng.uniform(0, 200), y + rng.uniform(0, 100)])
            skip.append(int(rng.random() < 0.08))
        for _ in range(nw):
            r = rng.random()
            if r < 0.3:                              # straddling two lattice cells, or 20 % inside one
                x, y = rng.integers(-4, 20) * 50 + 50, rng.integers(-4, 20) * 50
                words.append([x - 10, y + 10, x + 10, y + 20] if rng.random() < 0.5 else [x - 40, y, x + 10, y + 50])
            elif r < 0.4:                            # zero width / zero height
                x, y = rng.integers(-200, 1000, 2)
                words.append([x, y, x, y + 20] if rng.random() < 0.5 else [x, y, x + 30, y])
            else:
                x, y = rng.uniform(-300, 1000, 2)
                words.append([x, y, x + rng.uniform(0.5, 120), y + rng.uniform(0.5, 40)])
        if g % 5 == 1 and g > 0:                     # a group over the words of the group before it
            pw0, pw1 = groups[-1][0], groups[-1][1]
            groups.append((pw0, pw1, e0, len(elems)))
        else:
            groups.append((w0, len(words), e0, len(elems)))
    return (np.array(words, np.float64).reshape(-1, 4), np.array(elems, np.float64).reshape(-1, 4),
            np.array(skip, np.uint8), np.array(groups, np.int32).reshape(-1, 4))


@pytest.mark.parametrize("seed,n_groups,max_words,max_elems,tile_big", [
    (0, 4, 40, 30, False), (1, 37, 300, 300, False), (2, 3, 200, 1500, True), (3, 400, 20, 12, False),
    (4, 1, 1000, 3000, False)])
def test_kernel_equals_oracle_bit_for_bit(seed, n_groups, max_words, max_elems, tile_big):
    words, elems, skip, groups = _random_case(seed, n_groups, max_words, max_elems, tile_big)
    best, ratio = assign_best_overlap(words, elems, skip, groups, 0.2, DEV)
    want_best, want_ratio = ots.assign_best_overlap(words, elems, skip, groups, 0.2)
    assert np.array_equal(best, np.array(want_best, np.int32))
    assert np.array_equal(ratio.view(np.int64), np.array(want_ratio, np.float64).view(np.int64))
    # the case exercises what it claims
    assert (np.array(want_ratio) == 0.2).any() or seed == 4
    assert (groups[:, 1] == groups[:, 0]).any() or n_groups < 4


def test_kernel_ties_and_threshold():
    words = np.array([[90, 0, 110, 10], [0, 0, 10, 10], [0, 0, 10, 10], [3.7, -2.2, 9.9, 7.1]], np.float64)
    elems = np.array([[0, 0, 100, 10], [100, 0, 200, 10], [0, 0, 2, 10], [0, 0, 1, 10], [-1.5, -3.9, 5.2, 4.0]])
    skip = np.array([0, 0, 0, 0, 0], np.uint8)
    groups = [(0, 1, 0, 2), (1, 2, 2, 3), (2, 3, 3, 4), (3, 4, 4, 5)]
    best, ratio = assign_best_overlap(words, elems, skip, groups, 0.2, DEV)
    want = ots.assign_best_overlap(words, elems, skip, groups, 0.2)
    assert best.tolist() == want[0] == [0, 2, -1, 4]
    assert ratio.tolist() == want[1]


def test_kernel_rejects_bad_input():
    lib = _lib.lib()
    boxes = torch.zeros((4, 4), dtype=torch.float64, device=DEV)
    skip = torch.zeros(4, dtype=torch.uint8, device=DEV)
    best = torch.empty(8, dtype=torch.int32, device=DEV)
    ratio = torch.empty(8, dtype=torch.float64, device=DEV)

    def call(groups, n_words=4, n_elems=4, cap=8):
        g = np.array(groups, np.int32).reshape(-1, 4).copy().view(OVERLAP_GROUP_DTYPE).reshape(-1)
        return lib.ytk_op_assign_best_overlap_f64(boxes.data_ptr(), n_words, boxes.data_ptr(), skip.data_ptr(), n_elems,
                                                  g.ctypes.data, len(g), 0.2, best.data_ptr(), ratio.data_ptr(), cap,
                                                  None)

    for bad in ([(0, 5, 0, 4)], [(0, 4, 2, 1)], [(-1, 2, 0, 4)], [(0, 4, 0, 9)]):
        assert call(bad) != 0
        assert b"group 0" in lib.ytk_last_error()
    assert call([(0, 4, 0, 4), (0, 4, 0, 4), (0, 4, 0, 4)]) != 0           # 12 results, capacity 8
    assert b"capacity" in lib.ytk_last_error()
    assert call([(0, 4, 0, 4)]) == 0
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        assign_best_overlap([[0, 0, np.nan, 1]], [[0, 0, 1, 1]], [0], [(0, 1, 0, 1)], 0.2, DEV)
    with pytest.raises(ValueError):
        assign_best_overlap([[0, 0, 1, 1]], [[0, 0, 2.0 ** 31, 1]], [0], [(0, 1, 0, 1)], 0.2, DEV)
    with pytest.raises(_lib.YtkError):
        assign_best_overlap([[0, 0, 1, 1]], [[0, 0, 1, 1]], [0], [(0, 1, 0, 2)], 0.2, DEV)


# ------------------------------------------------------------------------------------------------ the parser
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_parser_through_the_kernel_equals_reference(case):
    res, _, _ = standin_parser(case, DEV)(np.zeros((8, 8, 3), np.uint8), grid_only=case["grid_only"],
                                          kv_only=case["kv_only"])
    assert ots.canonical_kv(res.model_dump()) == ots.canonical_kv(case["output"])


_TABLES = [[40, 60, 700, 420], [100, 480, 760, 760]]


def _parser(tables=_TABLES):
    nop = {"from_pretrained": False}
    p = TableSemanticParser(configs={"table_detector": nop, "table_cell_parser": nop, "text_detector": nop,
                                     "text_recognizer": {"from_pretrained": False, "model_name": "parseq-tiny-dynw-v4",
                                                         "dynamic_width": True, "batch_bucketing": True}},
                            device="cuda")
    p.layout_parser.model.load_state_dict(R.make_state_dict(R.SPECS["layout"], seed=11))
    load_trained_head(p.text_detector.model)
    # random layout weights find tables of any number and size: every page gets the same fixed tables instead (the
    # paragraphs stay the model's)
    lp = p.layout_parser
    parse_pages = lp.parse_pages

    def with_tables(pages, pages_dev=None):
        out = parse_pages(pages, pages_dev)
        for lay in out:
            lay.tables = [Element(id=None, box=b, score=0.9, role=None) for b in tables]
        return out
    lp.parse_pages = with_tables
    forwards = []
    fwd = p.cell_detector.model.forward_u8

    def counted(*a, **k):
        forwards.append(1)
        return fwd(*a, **k)
    p.cell_detector.model.forward_u8 = counted
    return p, forwards


def _pages(first, shapes):
    return [synthetic_page(first + i, height=h, width=w)[0] for i, (h, w) in enumerate(shapes)]


def test_numpy_page_equals_cuda_page():
    p, _ = _parser()
    page = _pages(500, [(1000, 800)])[0]
    a = p(page)[0]
    b = p(torch.from_numpy(page).to(DEV))[0]
    assert len(a.words) > 10 and len(a.tables) + len(a.paragraphs) > 0
    assert b.model_dump() == a.model_dump()


def test_parse_pages_equals_per_page_calls_with_one_cell_forward():
    p, forwards = _parser()
    pages = _pages(510, [(1200, 900), (900, 1000), (800, 800)])
    try:
        per_page = [p(pg)[0].model_dump() for pg in pages]
        del forwards[:]
        batch = p.parse_pages(pages)
        assert len(forwards) == 1
        assert [r.model_dump() for r in batch] == per_page
        assert sum(len(r["words"]) for r in per_page) > 30
        del forwards[:]
        dev = p.parse_pages([torch.from_numpy(pg).to(DEV) for pg in pages])
        assert len(forwards) == 1
        assert [r.model_dump() for r in dev] == per_page
    finally:
        if p._batched is not None:
            p._batched.close()
