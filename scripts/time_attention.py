"""Times the packed ragged attention op (ytk_op_attention_f16) for the mma.sync kernel (impl 1) and the wgmma kernel
(impl 2) on three shapes, 8 heads of 96, fp16:

  bench    - the PARSeq-large encoder sequences of one bench step (16 synthetic pages, 3200 crops, N = padded width / 2
             tokens), built on the CPU by the same synth / crop geometry / mini-batch plan calls as bench.py
  uniform  - 3200 sequences of seeded lengths 48..264
  masked   - the refinement self-attention: 101 shared queries against per-sequence key blocks of 101 rows

CUDA events over 20 launches after 3 warm-up launches.  Per kernel and shape: ms per launch, algorithmic GB/s (Q, K, V
read once, O written once), its fraction of the H100 SXM data sheet's 3.35 TB/s, and the tensor-core work the
wgmma kernel issues (64-query x 64-key tiles) over the real work (visible query-key pairs).  Prints one JSON line with
the GPU name and power limit, and the largest difference between the two kernels' outputs.

    python scripts/time_attention.py [--save-outputs FILE]

--save-outputs writes the wgmma kernel's outputs on every shape (torch.save) so that two builds can be compared bit
for bit.
"""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
HD, HEADS = 96, 8
REFINE_S = 101


def bench_encoder_lengths(pages=16):
    """Encoder sequence lengths of one single-GPU bench step, in the order the recognizer packs them."""
    from yomitoku_b200.config import TextRecognizerPARSeqLargeV41Config
    from yomitoku_b200.data import crop_geometry
    from yomitoku_b200.synth import synthetic_page
    from yomitoku_b200.text_recognizer import TextRecognizer, plan_mini_batches

    cfg = TextRecognizerPARSeqLargeV41Config()
    ph, pw = cfg["encoder"]["patch_size"]
    gh = cfg["data"]["img_size"][0] // ph
    lens = []
    for pi in range(pages):
        _, quads = synthetic_page(pi, n_slots=5)
        g, _ = crop_geometry((1200, 1600), quads, cfg["data"]["img_size"], True, page=pi)
        widths = g["canvas_w"].tolist()
        plan = plan_mini_batches(widths, np.argsort(g["cw"]).tolist(), True, cfg["data"]["batch_size"], None, None)
        padded, _ = TextRecognizer._collate_widths(SimpleNamespace(dynamic_width=True), widths, plan)
        lens += [gh * (padded[i] // pw) for b in plan for i in b]
    return lens


def uniform_lengths():
    return np.random.default_rng(0).integers(48, 265, size=3200).tolist()


def masked_keys():
    return np.random.default_rng(1).integers(8, REFINE_S + 1, size=3200).tolist()


def mma_work(q_lens, k_lens, masked, tq=64, tk=64):
    """(issued, real) query-key pairs of one head: issued by tiles of tq queries x tk keys (a tile's key range ends at
    the last key any of its queries sees), real = visible pairs."""
    issued = real = 0
    for nq, nk in zip(q_lens, k_lens):
        qi = np.arange(nq)[:, None]
        kj = np.arange(nk)[None, :]
        vis = ((qi < 2) | (kj <= qi)) if masked else np.ones((nq, nk), bool)
        real += int(vis.sum())
        for q0 in range(0, nq, tq):
            k_end = nk if not masked or q0 < 2 else min(nk, q0 + tq)
            issued += tq * (-(-k_end // tk) * tk)
    return issued, real


def main():
    import torch

    from yomitoku_b200 import _lib

    ap = argparse.ArgumentParser()
    ap.add_argument("--save-outputs", default=None)
    args = ap.parse_args()

    def time_ms(fn, reps=20, warmup=3):
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

    L = _lib.lib()
    D = HD * HEADS
    g = torch.Generator().manual_seed(0)
    res, saved = {}, {}

    def report(name, run, nbytes, work, out):
        r = {"work_issued_over_real": round(work[0] / work[1], 3), "algorithmic_MB": round(nbytes / 1e6, 1)}
        for impl, kern in ((1, "mma_sync"), (2, "wgmma")):
            ms = time_ms(lambda: run(impl))
            r[kern + "_ms"] = round(ms, 4)
            r[kern + "_GBps"] = round(nbytes / ms / 1e6, 1)
            r[kern + "_frac_hbm"] = round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3)
        out.fill_(float("nan"))
        run(1)
        ref = out.clone()
        out.fill_(float("nan"))
        run(2)
        torch.cuda.synchronize()
        r["wgmma_max_abs_diff_vs_mma_sync"] = (out.float() - ref.float()).abs().max().item()
        saved[name] = out.cpu().clone()
        res[name] = r

    for name, lens in (("bench", bench_encoder_lengths()), ("uniform", uniform_lengths())):
        T = sum(lens)
        qkv = torch.randn(T, 3 * D, generator=g).cuda().half()
        out = torch.empty(T, D, device="cuda", dtype=torch.float16)
        seqs = (_lib.YtkAttnSeq * len(lens))()
        off = 0
        for i, n in enumerate(lens):
            seqs[i] = _lib.YtkAttnSeq(off, n, off, n, off * 3 * D, n, 0)
            off += n
        seqs_dev = torch.frombuffer(bytearray(bytes(seqs)), dtype=torch.uint8).cuda()

        def run(impl, qkv=qkv, out=out, T=T, lens=lens, seqs_dev=seqs_dev):
            _lib.check(L.ytk_op_attention_f16(qkv.data_ptr(), 3 * D, T, qkv[:, D:].data_ptr(),
                                              qkv[:, 2 * D:].data_ptr(), 3 * D, T, out.data_ptr(), D,
                                              seqs_dev.data_ptr(), len(lens), max(lens), HEADS, HD, 0, impl, None))
        report(name, run, 8 * T * D, mma_work(lens, lens, False), out)
        res[name]["shape"] = "%d sequences, %d tokens (%d..%d), %d heads x %d" % (len(lens), T, min(lens), max(lens),
                                                                                 HEADS, HD)
        del qkv, out

    # masked refinement shape: S = 101 shared queries against per-sequence key blocks of 101 rows, keys >= kpad hidden
    S, kl = REFINE_S, masked_keys()
    nseq = len(kl)
    qm = torch.randn(S, D, generator=g).cuda().half()
    kv = torch.randn(nseq * S, 2 * D, generator=g).cuda().half()
    om = torch.empty(nseq * S, D, device="cuda", dtype=torch.float16)
    ms = (_lib.YtkAttnSeq * nseq)()
    for i in range(nseq):
        ms[i] = _lib.YtkAttnSeq(0, S, i * S, S, i * S * 2 * D, kl[i], 0)
    ms_dev = torch.frombuffer(bytearray(bytes(ms)), dtype=torch.uint8).cuda()

    def run_m(impl):
        _lib.check(L.ytk_op_attention_f16(qm.data_ptr(), D, S, kv.data_ptr(), kv[:, D:].data_ptr(), 2 * D, nseq * S,
                                          om.data_ptr(), D, ms_dev.data_ptr(), nseq, S, HEADS, HD, 1, impl, None))
    report("masked", run_m, 2 * D * (S + 2 * sum(kl) + nseq * S), mma_work([S] * nseq, kl, True), om)
    res["masked"]["shape"] = "%d x %d shared queries, kpad 8..%d, %d heads x %d" % (nseq, S, S, HEADS, HD)

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    res["gpu"] = q or torch.cuda.get_device_name()
    if args.save_outputs:
        torch.save(saved, args.save_outputs)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
