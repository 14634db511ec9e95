"""CPU: the host half of device pages (yomitoku_b200/device_pages.py) - the ytk_page_src record layout, the library
export, the source records built from strided torch views (checked by gathering through them on CPU tensors) and the
ValueError of every rejected input."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from yomitoku_b200 import DevicePages, _lib, build, device_pages
from yomitoku_b200.device_pages import PAGE_SRC_DTYPE, as_device_pages, page_sources

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_CTYPES = {"const uint8_t*": ctypes.c_void_p, "long long": ctypes.c_longlong, "int": ctypes.c_int}


def _header_struct(name):
    """ctypes Structure built from the field list of `typedef struct {...} name;` in the public header."""
    header = open(os.path.join(ROOT, "include", "yomitoku_b200.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} %s;" % name, header).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        ctype = next(t for t in _CTYPES if decl.startswith(t + " "))
        fields += [(f.strip(), _CTYPES[ctype]) for f in decl[len(ctype):].split(",")]
    return type(name, (ctypes.Structure,), {"_fields_": fields})


def test_page_src_dtype_matches_header():
    S = _header_struct("ytk_page_src")
    assert ctypes.sizeof(S) == PAGE_SRC_DTYPE.itemsize == 48          # the size the header states
    assert [f[0] for f in S._fields_] == list(PAGE_SRC_DTYPE.names)
    for f, _ in S._fields_:
        assert getattr(S, f).offset == PAGE_SRC_DTYPE.fields[f][1], f


def test_library_exports_pack_entry():
    build.build(verbose=False)
    assert hasattr(_lib.lib(), "ytk_pack_pages_u8")


def _gather(rec, t):
    """The H x W x 3 BGR page the kernel reads through record `rec` from the storage of CPU tensor `t`."""
    base = t.untyped_storage().data_ptr()
    storage = np.frombuffer(bytes(t.untyped_storage()), np.uint8)
    off = int(rec["data"]) - base
    y, x, c = np.meshgrid(np.arange(rec["H"]), np.arange(rec["W"]), np.arange(3), indexing="ij")
    src_c = 2 - c if rec["rgb"] else c
    return storage[off + y * int(rec["sh"]) + x * int(rec["sw"]) + src_c * int(rec["sc"])]


def _views():
    g = torch.Generator().manual_seed(0)
    hwc = torch.randint(0, 256, (37, 53, 3), dtype=torch.uint8, generator=g)
    chw = torch.randint(0, 256, (3, 41, 29), dtype=torch.uint8, generator=g)
    rgba = torch.randint(0, 256, (19, 23, 4), dtype=torch.uint8, generator=g)
    return {"contiguous": hwc, "permute": chw.permute(1, 2, 0), "crop": hwc[5:30, 7:40], "step2": hwc[::2, ::2],
            "crop-step": chw.permute(1, 2, 0)[3:, 1::3], "channel-slice": rgba[..., :3], "width1": hwc[:, 4:5],
            "expanded": hwc[:1, :1].expand(6, 9, 3)}


@pytest.mark.parametrize("order", ["bgr", "rgb"])
def test_records_of_strided_views_gather_the_page(order):
    views = _views()
    recs, shapes, device, pages = page_sources(list(views.values()), order, need_cuda=False)
    assert device == torch.device("cpu") and len(pages) == len(views)
    for rec, (name, t), hw in zip(recs, views.items(), shapes):
        assert hw == tuple(t.shape[:2]), name
        expect = t.numpy()[:, :, ::-1] if order == "rgb" else t.numpy()
        np.testing.assert_array_equal(_gather(rec, t), expect, err_msg=name)


def test_stacked_tensor_is_pages():
    t = torch.arange(2 * 5 * 7 * 3, dtype=torch.uint8).reshape(2, 5, 7, 3)
    recs, shapes, _, _ = page_sources(t, "bgr", need_cuda=False)
    assert shapes == [(5, 7), (5, 7)]
    assert int(recs[1]["data"]) - int(recs[0]["data"]) == 5 * 7 * 3
    np.testing.assert_array_equal(_gather(recs[1], t), t[1].numpy())


def _bad_inputs():
    page = torch.zeros((8, 9, 3), dtype=torch.uint8)
    meta = torch.empty((8, 9, 3), dtype=torch.uint8, device="meta")
    return [
        ("CPU tensor", lambda: device_pages([page]), "cpu"),
        ("CPU stack", lambda: device_pages(page[None]), "cpu"),
        ("float", lambda: page_sources([page.float()], need_cuda=False), "dtype"),
        ("one channel", lambda: page_sources([page[..., :1]], need_cuda=False), "three channels"),
        ("four channels", lambda: page_sources([torch.zeros((8, 9, 4), dtype=torch.uint8)], need_cuda=False),
         "three channels"),
        ("2-d", lambda: page_sources([page[..., 0]], need_cuda=False), "three channels"),
        ("empty page", lambda: page_sources([page[:0]], need_cuda=False), "empty"),
        ("empty width", lambda: page_sources([page[:, :0]], need_cuda=False), "empty"),
        ("mixed devices", lambda: page_sources([page, meta], need_cuda=False), "one device"),
        ("no pages", lambda: page_sources([], need_cuda=False), "no pages"),
        ("numpy page", lambda: page_sources([page.numpy()], need_cuda=False), "not a torch tensor"),
        ("3-d stack", lambda: page_sources(page, need_cuda=False), "(n, H, W, 3)"),
        ("channel order", lambda: page_sources([page], "bgra", need_cuda=False), "channel_order"),
        ("not pages", lambda: device_pages("page.jpg"), "list of"),
    ]


@pytest.mark.parametrize("case", _bad_inputs(), ids=lambda c: c[0])
def test_rejected_inputs_raise_value_error_with_the_reason(case):
    _, call, reason = case
    with pytest.raises(ValueError, match=re.escape(reason)):
        call()


def test_host_pages_stay_on_the_host_path():
    page = np.zeros((8, 9, 3), np.uint8)
    assert as_device_pages(page) is None
    assert as_device_pages([page, page]) is None
    assert as_device_pages(torch.zeros((8, 9, 3), dtype=torch.uint8)) is None
    dp = DevicePages(torch.zeros(8 * 9 * 3, dtype=torch.uint8), *_table([(8, 9)]))
    assert as_device_pages(dp) is dp and len(dp) == 1


def _table(shapes):
    from yomitoku_b200.data import page_table
    return page_table(shapes)[0], shapes


def test_page_views_and_select_follow_the_table():
    shapes = [(4, 5), (3, 7), (2, 2)]
    table, shapes = _table(shapes)
    buf = torch.arange(int(sum(h * w * 3 for h, w in shapes)), dtype=torch.int64).to(torch.uint8)
    dp = DevicePages(buf, table, shapes)
    o = 4 * 5 * 3
    assert torch.equal(dp.page(1).reshape(-1), buf[o:o + 3 * 7 * 3])
    one = dp.select(1)
    assert one.shapes == [(3, 7)] and int(one.table["page_off"][0]) == 0
    assert one.buf.data_ptr() == buf.data_ptr() + o
