"""Times the packed ragged attention op (ytk_op_attention_f16) on the PARSeq-large encoder shape of the bench step:
3200 sequences (seeded lengths 48..264 tokens), 8 heads of 96, fp16, for the mma.sync kernel (impl 1) and the wgmma
kernel (impl 2), plus the masked refinement shape.  CUDA events over 20 launches after 3 warm-up launches; prints one
JSON line with the GPU name and power limit.

    python scripts/time_attention.py
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from yomitoku_b200 import _lib  # noqa: E402


def _time(fn, reps=20, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    L = _lib.lib()
    hd, heads = 96, 8
    D = hd * heads
    rng = np.random.default_rng(0)
    lens = rng.integers(48, 265, size=3200).tolist()
    T = sum(lens)
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(T, 3 * D, generator=g).cuda().half()
    out = torch.empty(T, D, device="cuda", dtype=torch.float16)
    seqs = (_lib.YtkAttnSeq * len(lens))()
    off = 0
    for i, n in enumerate(lens):
        seqs[i] = _lib.YtkAttnSeq(off, n, off, n, off * 3 * D, n, 0)
        off += n
    seqs_dev = torch.frombuffer(bytearray(bytes(seqs)), dtype=torch.uint8).cuda()

    def run(impl):
        _lib.check(L.ytk_op_attention_f16(qkv.data_ptr(), 3 * D, T, qkv[:, D:].data_ptr(), qkv[:, 2 * D:].data_ptr(),
                                          3 * D, T, out.data_ptr(), D, seqs_dev.data_ptr(), len(lens), max(lens),
                                          heads, hd, 0, impl, None))
    res = {"shape": "%d sequences, %d tokens, %d heads x %d" % (len(lens), T, heads, hd)}
    for impl, name in ((1, "mma_sync_ms"), (2, "wgmma_ms")):
        res[name] = _time(lambda: run(impl))
    # masked refinement shape: S = 101 shared queries against per-sequence key blocks of 101 rows
    S, nseq = 101, 3200
    qm = torch.randn(S, D, generator=g).cuda().half()
    kv = torch.randn(nseq * S, 2 * D, generator=g).cuda().half()
    om = torch.empty(nseq * S, D, device="cuda", dtype=torch.float16)
    ms = (_lib.YtkAttnSeq * nseq)()
    for i in range(nseq):
        ms[i] = _lib.YtkAttnSeq(0, S, i * S, S, i * S * 2 * D, int(rng.integers(8, S + 1)), 0)
    ms_dev = torch.frombuffer(bytearray(bytes(ms)), dtype=torch.uint8).cuda()

    def run_m(impl):
        _lib.check(L.ytk_op_attention_f16(qm.data_ptr(), D, S, kv.data_ptr(), kv[:, D:].data_ptr(), 2 * D, nseq * S,
                                          om.data_ptr(), D, ms_dev.data_ptr(), nseq, S, heads, hd, 1, impl, None))
    for impl, name in ((1, "masked_mma_sync_ms"), (2, "masked_wgmma_ms")):
        res[name] = _time(lambda: run_m(impl))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    res["gpu"] = q or torch.cuda.get_device_name()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
