"""Times the input preparation of the RT-DETRv2 models on one GPU, host path against device path, and prints one JSON
object.  Cases (seeded random BGR pages of 1200 x 1600, three table boxes per page):

  * layout  16 pages -> 640 x 640, one call for all pages (LayoutParser.parse_pages);
  * table   the 3 table crops of a page -> 640 x 640, one call per page (TableStructureRecognizer);
  * cell    the same crops -> 960 x 960, one call per page (CellDetector).

For each case:
  * host_ms_per_call: the module's `preprocess` (cvtColor, numpy crops, Pillow BILINEAR resize, CHW fp32 / 255) plus the
    H2D copy of the fp32 tensors, host clock, ending in a device synchronise;
  * device_ms_per_call: the upload of the u8 pages (layout case only: the table calls read the pages the parser
    uploaded, as LayoutAnalyzer does) plus the two resize kernels (ytk_op_resize_bilinear_u8), CUDA events;
  * host_pcie_bytes / device_pcie_bytes per call, computed from shapes (records and coefficients, a few KB, left out).
Both paths then write the same NHWC-64 engine input (pack_input_kernel on the host path, the vertical resize kernel on
the device path); that write is in neither number.  The card's name and power limit are read in the same run.

Usage: python scripts/time_rtdetr_prep.py [--steps 10] [--warmup 2] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from yomitoku_b200 import _lib  # noqa: E402
from yomitoku_b200.layout_parser import LayoutParser, rtdetr_sources  # noqa: E402
from yomitoku_b200.table_cell_detector import CellDetector  # noqa: E402
from yomitoku_b200.table_structure_recognizer import TableStructureRecognizer  # noqa: E402

N_PAGES, H, W = 16, 1600, 1200
BOXES = [[60, 100, 1140, 620], [40, 700, 700, 1300], [720, 760, 1180, 1560]]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def host_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3 / steps


def event_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


class DeviceResize:
    """ytk_op_resize_bilinear_u8 for fixed records, scratch and output allocated once."""

    def __init__(self, recs, S):
        self.recs, self.S, self.L = recs, S, _lib.lib()
        self.need = self.L.ytk_op_resize_bilinear_scratch_bytes(recs.ctypes.data, len(recs), S)
        self.scratch = torch.empty(self.need, dtype=torch.uint8, device="cuda")
        self.out = torch.empty((len(recs), S, S, 3), dtype=torch.uint8, device="cuda")

    def __call__(self, pages_dev):
        _lib.check(self.L.ytk_op_resize_bilinear_u8(pages_dev.data_ptr(), pages_dev.numel(), self.recs.ctypes.data,
                                                    len(self.recs), self.S, self.scratch.data_ptr(), self.need,
                                                    self.out.data_ptr(), None))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_rtdetr_prep: needs a GPU")
    rng = np.random.default_rng(0)
    pages = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(N_PAGES)]
    flat = np.concatenate([p.reshape(-1) for p in pages])
    parser = LayoutParser(from_pretrained=False, device="cuda")
    tsr = TableStructureRecognizer(from_pretrained=False, device="cuda")
    cell = CellDetector(from_pretrained=False, device="cuda")
    res = {"card": card(), "pages": [N_PAGES, H, W], "table_boxes_per_page": BOXES, "cases": []}

    # layout: all pages in one call
    recs, _ = rtdetr_sources([p.shape for p in pages], [(i, (0, 0, W, H)) for i in range(N_PAGES)])
    rs = DeviceResize(recs, 640)

    def host_layout():
        torch.cat([parser.preprocess(p) for p in pages]).to("cuda")

    def dev_layout():
        rs(torch.from_numpy(flat).to("cuda"))
    res["cases"].append({"case": "layout", "inputs_per_call": N_PAGES, "size": 640,
                         "host_ms_per_call": host_ms(host_layout, a.steps, a.warmup),
                         "device_ms_per_call": event_ms(dev_layout, a.steps, a.warmup),
                         "host_pcie_bytes": N_PAGES * 3 * 640 * 640 * 4, "device_pcie_bytes": flat.nbytes})

    # tables and cells: one call per page, reading the page the parser uploaded
    page_dev = torch.from_numpy(pages[0].reshape(-1).copy()).to("cuda")
    crop_pixels = sum((b[2] - b[0]) * (b[3] - b[1]) for b in BOXES)
    for name, module, S in (("table", tsr, 640), ("cell", cell, 960)):
        recs, _ = rtdetr_sources([pages[0].shape], [(0, b) for b in BOXES])
        rs = DeviceResize(recs, S)
        if module is cell:
            tables = [type("T", (), {"box": b, "role": None})() for b in BOXES]

            def host_tables():
                torch.cat([d["tensor"] for d in cell.preprocess(pages[0], tables)]).to("cuda")
        else:
            def host_tables():
                torch.cat([d["tensor"] for d in tsr.preprocess(pages[0], BOXES)]).to("cuda")
        res["cases"].append({"case": name, "inputs_per_call": len(BOXES), "size": S,
                             "crop_pixels_per_call": crop_pixels,
                             "host_ms_per_call": host_ms(host_tables, a.steps, a.warmup),
                             "device_ms_per_call": event_ms(lambda: rs(page_dev), a.steps * 10, a.warmup),
                             "host_pcie_bytes": len(BOXES) * 3 * S * S * 4, "device_pcie_bytes": 0})
    res["card_after"] = card()
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
