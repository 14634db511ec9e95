"""Times the table cell detector on one GPU and prints one JSON object:

  * CellDetector's model forward (RT-DETRv2, 960 x 960, 1500 queries, 6 classes, random weights) in images/s for
    batch 1, 4 and 8, inputs and outputs resident in device memory, CUDA events around `--steps` forwards;
  * the query-selection kernel (ytk_op_topk_f32) in microseconds per launch at the layout models' shape (8 images x
    8,400 anchors -> 300) and the cell detector's (8 x 18,900 -> 1,500), CUDA events around `--launches` launches;
  * the card's name and power limit, read in the same run (a number is only worth something with them).

Usage: python scripts/time_cell_detector.py [--steps 20] [--warmup 5] [--launches 500] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from yomitoku_b200 import _lib  # noqa: E402
from yomitoku_b200.config import TableCellParserRTDETRv2Config, to_config  # noqa: E402
from yomitoku_b200.models import RTDETRv2  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def event_ms(fn, n, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def forward_rates(steps, warmup):
    L = _lib.lib()
    m = RTDETRv2(cfg=to_config(TableCellParserRTDETRv2Config())).to("cuda")
    out = []
    for batch in (1, 4, 8):
        x = torch.rand(batch, 3, 960, 960, device="cuda")
        lg = torch.empty((batch, 1500, 6), dtype=torch.float32, device="cuda")
        bx = torch.empty((batch, 1500, 4), dtype=torch.float32, device="cuda")

        def step():
            _lib.check(L.ytk_rtdetr_forward_f32(m._ensure(), x.data_ptr(), 1, batch, lg.data_ptr(), bx.data_ptr(), 1,
                                                None))
        ms = event_ms(step, steps, warmup)
        out.append({"batch": batch, "ms_per_forward": ms, "images_per_s": batch / (ms / 1e3),
                    "gflop_per_image": m.flops(batch) / batch / 1e9})
    return out


def topk_times(launches):
    L = _lib.lib()
    out = []
    for n, anchors, k in ((8, 8400, 300), (8, 18900, 1500)):
        s = torch.randn(n, anchors, device="cuda")
        idx = torch.empty((n, k), dtype=torch.int32, device="cuda")

        def launch():
            _lib.check(L.ytk_op_topk_f32(s.data_ptr(), n, anchors, k, idx.data_ptr(), None))
        ms = event_ms(launch, launches, 20)
        out.append({"images": n, "anchors": anchors, "k": k, "us_per_launch": ms * 1e3})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--launches", type=int, default=500)
    ap.add_argument("--out", default=None, help="also write the JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_cell_detector: needs a GPU")
    res = {"card": card(), "cell_detector_forward": forward_rates(a.steps, a.warmup), "topk": topk_times(a.launches),
           "card_after": card()}
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
