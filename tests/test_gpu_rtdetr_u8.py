"""GPU: the u8 entry of the RT-DETRv2 models (ytk_rtdetr_forward_u8, csrc/resample_ops.cu).

  * the device resize (ytk_op_resize_bilinear_u8) equals Pillow's Image.resize(..., BILINEAR) bit for bit, in one call
    over pages of mixed sizes with several rectangles per page;
  * RTDETRv2.forward_u8 is torch.equal to forward on torch.cat(preprocess(...)) for the layout parser (640), the table
    structure recognizer (640) and the cell detector (960), with the pages on the host and already on the device;
  * LayoutParser, parse_pages, TableStructureRecognizer, CellDetector, LayoutAnalyzer and analyze_pages, which take the
    device path on a GPU, return exactly what the host path (postprocess(model(torch.cat(preprocess(...))))) returns;
  * a box the device path refuses falls back to the host path, a bad record is a clean error without a launch, and
    two runs on a non-default stream give the same bits."""
import os
import sys

import cv2
import numpy as np
import pytest
import torch

from oracle import rtdetr as R
from yomitoku_b200 import _lib
from yomitoku_b200.layout_parser import rtdetr_sources

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_cell import CELL_SEED, CELL_SPEC, cell_input  # noqa: E402
from make_golden_rtdetr import rtdetr_input  # noqa: E402
from test_resample_math import CASES, make_page, pil_resize  # noqa: E402

pytestmark = pytest.mark.gpu


class _Table:
    def __init__(self, box, role=None):
        self.box, self.role = box, role


def _flat(pages):
    return np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in pages])


def _device_resize(pages, rects, S):
    recs, _ = rtdetr_sources([p.shape for p in pages], rects)
    lib = _lib.lib()
    need = lib.ytk_op_resize_bilinear_scratch_bytes(recs.ctypes.data, len(recs), S)
    assert need > 0
    buf = torch.from_numpy(_flat(pages)).cuda()
    scratch = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = torch.full((len(recs), S, S, 3), 77, dtype=torch.uint8, device="cuda")
    _lib.check(lib.ytk_op_resize_bilinear_u8(buf.data_ptr(), buf.numel(), recs.ctypes.data, len(recs), S,
                                             scratch.data_ptr(), need, out.data_ptr(), None))
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("S", [640, 960])
def test_resize_op_equals_pillow(S):
    """Every size case of the CPU test plus sub-rectangles, pages of mixed sizes and contents in ONE call."""
    kinds = ("random", "gradient", "constant")
    pages = [make_page(H, W, kinds[i % 3], seed=i) for i, ((H, W), _) in enumerate(CASES)]
    rects = []
    for i, p in enumerate(pages):
        H, W = p.shape[:2]
        rects.append((i, (0, 0, W, H)))
        if H > 4 and W > 4:
            rects.append((i, (W // 5, H // 3, W - W // 7, H - 1)))
            rects.append((i, (W // 2, 0, W // 2 + 3, H)))
    got = _device_resize(pages, rects, S)
    for j, (i, r) in enumerate(rects):
        np.testing.assert_array_equal(got[j], pil_resize(pages[i], r, S), err_msg="page %d rect %s" % (i, r))


# ------------------------------------------------------------------------------------------------ models and modules
def _layout_page(seed, size):
    rgb = (rtdetr_input(seed)[0].permute(1, 2, 0) * 255).to(torch.uint8).numpy()
    return np.ascontiguousarray(cv2.resize(rgb, size, interpolation=cv2.INTER_LINEAR)[:, :, ::-1])


def _table_page():
    """A 1400 x 1100 page with table crops of the seeded cell input pasted in; the third is larger than 960 on one side."""
    page = np.full((1400, 1100, 3), 245, np.uint8)
    tables = [_Table([60, 80, 700, 560]), _Table([120, 640, 1040, 1000]), _Table([30, 20, 1090, 1390])]
    for i, t in enumerate(tables[:2]):
        x1, y1, x2, y2 = t.box
        rgb = (cell_input(40 + i)[0].permute(1, 2, 0) * 255).to(torch.uint8).numpy()
        page[y1:y2, x1:x2] = cv2.resize(rgb, (x2 - x1, y2 - y1), interpolation=cv2.INTER_AREA)[:, :, ::-1]
    return page, tables


@pytest.fixture(scope="module")
def modules():
    from yomitoku_b200 import CellDetector, LayoutAnalyzer
    nop = {"from_pretrained": False}
    an = LayoutAnalyzer(configs={"layout_parser": nop, "table_structure_recognizer": nop}, device="cuda")
    an.layout_parser.model.load_state_dict(R.make_state_dict(R.SPECS["layout"], seed=11))
    an.table_structure_recognizer.model.load_state_dict(R.make_state_dict(R.SPECS["table"], seed=12))
    cell = CellDetector(from_pretrained=False, device="cuda")
    cell.model.load_state_dict(R.make_state_dict(CELL_SPEC, seed=CELL_SEED))
    return an.layout_parser, an.table_structure_recognizer, cell, an


def _equal(a, b):
    return all(torch.equal(a[k].cpu(), b[k].cpu()) for k in ("pred_logits", "pred_boxes"))


def _check_model(model, pages, rects, host_x):
    recs, _ = rtdetr_sources([p.shape for p in pages], rects)
    ref = model(host_x)
    host = model.forward_u8(_flat(pages), recs)
    assert not host["pred_logits"].is_cuda
    assert _equal(host, ref)
    dev = model.forward_u8(torch.from_numpy(_flat(pages)).cuda(), recs)
    assert dev["pred_logits"].is_cuda
    assert _equal(dev, ref)


def test_forward_u8_equals_forward_on_preprocess(modules):
    parser, tsr, cell, _ = modules
    pages = [_layout_page(21, (1600, 1200)), _layout_page(22, (900, 1300))]
    _check_model(parser.model, pages, [(i, (0, 0, p.shape[1], p.shape[0])) for i, p in enumerate(pages)],
                 torch.cat([parser.preprocess(p) for p in pages]))
    page, tables = _table_page()
    boxes = [t.box for t in tables]
    _check_model(tsr.model, [page], [(0, b) for b in boxes], torch.cat([d["tensor"] for d in tsr.preprocess(page, boxes)]))
    # cell: 640 x 480 and 920 x 360 crops are up-scaled to 960, the 1060 x 1370 crop is down-scaled
    _check_model(cell.model, [page], [(0, b) for b in boxes],
                 torch.cat([d["tensor"] for d in cell.preprocess(page, tables)]))


def _host_parse(parser, pages):
    preds = parser.model(torch.cat([parser.preprocess(p) for p in pages]))
    return [parser.postprocess({k: v[i:i + 1] for k, v in preds.items()}, p.shape[:2]) for i, p in enumerate(pages)]


def _host_tables(tsr, page, boxes):
    data = tsr.preprocess(page, boxes)
    if not data:
        return []
    preds = tsr.model(torch.cat([d["tensor"] for d in data]))
    out = [tsr.postprocess({k: v[i:i + 1] for k, v in preds.items()}, d) for i, d in enumerate(data)]
    return [t for t in out if t.n_row > 0 and t.n_col > 0]


def _host_cells(cell, page, tables):
    from yomitoku_b200.schemas import TableDetectorSchema
    data = cell.preprocess(page, tables)
    preds = cell.model(torch.cat([d["tensor"] for d in data]))
    out = []
    for i, (d, t) in enumerate(zip(data, tables)):
        cells, kv, grid = cell.postprocess({k: v[i:i + 1] for k, v in preds.items()}, d, t.box)
        if cells:
            out.append(TableDetectorSchema(id=None, box=t.box, role=t.role, cells=cells, kv_regions=kv, grid_regions=grid))
    return out


def _dump(items):
    return [x.model_dump() for x in items]


def test_modules_match_the_host_path(modules):
    from yomitoku_b200.schemas import LayoutAnalyzerSchema
    parser, tsr, cell, an = modules
    pages = [_layout_page(21, (1600, 1200)), _layout_page(22, (900, 1300))]
    ref = _host_parse(parser, pages)
    res, _ = parser(pages[0])
    assert res.model_dump() == _host_parse(parser, pages[:1])[0].model_dump()
    assert len(res.paragraphs) + len(res.tables) + len(res.figures) > 3
    assert _dump(parser.parse_pages(pages)) == _dump(ref)

    page, tables = _table_page()
    boxes = [t.box for t in tables]
    got, _ = tsr(page, boxes)
    assert len(got) > 0 and _dump(got) == _dump(_host_tables(tsr, page, boxes))
    got = cell(page, tables)
    assert len(got) > 0 and _dump(got) == _dump(_host_cells(cell, page, tables))

    def host_analyze(p, layout):
        return LayoutAnalyzerSchema(paragraphs=layout.paragraphs, tables=_host_tables(tsr, p, [t.box for t in layout.tables]),
                                    figures=layout.figures)
    layout, _ = an(pages[0])
    assert layout.model_dump() == host_analyze(pages[0], _host_parse(parser, pages[:1])[0]).model_dump()
    batch = an.analyze_pages(pages + [page])
    want = [host_analyze(p, lay) for p, lay in zip(pages + [page], _host_parse(parser, pages + [page]))]
    assert _dump(batch) == _dump(want)
    assert sum(len(b.tables) for b in batch) > 0


def test_refused_boxes_fall_back_to_the_host_path(modules):
    _, tsr, cell, _ = modules
    page, tables = _table_page()
    boxes = [[-100, 80, 1100, 560], tables[1].box]      # numpy wraps x1 = -100 to 1000: a 100-wide crop
    assert rtdetr_sources([page.shape], [(0, b) for b in boxes]) is None
    got, _ = tsr(page, boxes)
    assert _dump(got) == _dump(_host_tables(tsr, page, boxes))
    odd = [_Table(boxes[0]), tables[1]]
    assert _dump(cell(page, odd)) == _dump(_host_cells(cell, page, odd))


def test_bad_records_and_repeats(modules):
    parser, _, _, _ = modules
    m = parser.model
    pages = [_layout_page(23, (700, 500))]
    recs, _ = rtdetr_sources([pages[0].shape], [(0, (0, 0, 700, 500))])
    lib = _lib.lib()
    before = lib.ytk_launch_count()
    for field, value in (("x1", 701), ("y1", 501), ("y0", 500), ("x0", -1), ("page_off", 1)):
        bad = recs.copy()
        bad[field][0] = value
        with pytest.raises(_lib.YtkError, match="source 0"):
            m.forward_u8(_flat(pages), bad)
        with pytest.raises(_lib.YtkError, match="source 0"):
            m.forward_u8(torch.from_numpy(_flat(pages)).cuda(), bad)
    assert lib.ytk_launch_count() == before

    buf = torch.from_numpy(_flat(pages)).cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    outs = []
    for _ in range(2):
        o = m.forward_u8(buf, recs, stream=s)
        s.synchronize()
        outs.append({k: v.cpu() for k, v in o.items()})
    assert _equal(outs[0], outs[1])
    assert _equal(outs[0], m(parser.preprocess(pages[0])))
