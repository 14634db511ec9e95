"""The bench-mixture shape of scripts/time_attention.py is the encoder attention of a bench step: its statistics are
pinned here so that the timing shape cannot drift from bench.py unnoticed."""
import importlib.util
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _time_attention():
    spec = importlib.util.spec_from_file_location("time_attention", os.path.join(ROOT, "scripts", "time_attention.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_bench_mixture_statistics():
    lens = np.asarray(_time_attention().bench_encoder_lengths())
    assert len(lens) == 3200
    assert (lens.min(), lens.max()) == (100, 184)
    assert int(lens.sum()) == 424448
    assert round(float(lens.mean()), 2) == 132.64
    assert int((lens < 128).sum()) == 2048
    assert int(((lens >= 128) & (lens < 192)).sum()) == 1152
    assert (lens % 4 == 0).all()    # 4 patch rows of a 32-px crop


def test_issued_work_of_64_query_units():
    mod = _time_attention()
    lens = mod.bench_encoder_lengths()
    issued, real = mod.mma_work(lens, lens, False, tq=64)
    assert round(issued / real, 2) == 1.25
    issued, real = mod.mma_work(lens, lens, False, tq=128)
    assert round(issued / real, 2) == 1.48
