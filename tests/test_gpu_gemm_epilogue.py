"""GPU: the TMA epilogue of gemm_tc_kernel (results stored from the wgmma fragments) against the staged epilogue
(YTK_EPI=staged, row per thread) on the same operands.  Both apply (acc + bias) + residual, the activation and the
rounding in the same order, so the outputs must be bit-identical, sentinel columns past Cout included.  The staged
outputs come from a child process because the epilogue choice is read once per process."""
import os
import subprocess
import sys

import pytest
import torch

from yomitoku_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (M, K, N, act, resid, f32, in_place): the linear cases of test_gpu_kernels.py, the PARSeq encoder's four linears
# (qkv, proj, fc1, fc2 at a slice of the bench's 424,448 rows) and the AR step's at 3200 rows
LINEAR = [
    (128, 64, 64, 0, None, True, False), (300, 128, 200, 0, None, False, False),
    (1000, 768, 2304, 2, None, False, False), (517, 768, 7119, 0, None, True, False),
    (640, 3072, 768, 0, "f32", True, False), (33, 192, 576, 1, "f16", False, False),
    (129, 64, 100, 0, "f16", True, False), (128 * 74 + 5, 768, 2304, 2, None, False, False),
    (128 * 148 + 77, 192, 768, 0, "f32", True, False), (128 * 21 + 1, 768, 7119, 0, None, True, False),
    (128 * 200, 3072, 768, 0, "f32", True, False), (1000, 128, 72, 0, "f16", False, False),
    (4000, 64, 64, 1, "f16", False, False), (128 * 500 + 3, 64, 256, 0, "f32", True, False),
    (128 * 300 + 64, 128, 328, 2, "f16", False, False),
    (128 * 90 + 17, 768, 768, 0, "f32", True, True),
    # encoder
    (128 * 400 + 37, 768, 2304, 0, None, False, False), (128 * 400 + 37, 768, 768, 0, "f32", True, True),
    (128 * 400 + 37, 768, 3072, 2, None, False, False), (128 * 400 + 37, 3072, 768, 0, "f32", True, True),
    # AR step
    (3200, 768, 768, 0, None, False, False), (3200, 768, 768, 0, "f32", True, True),
    (3200, 768, 3072, 2, None, False, False), (3200, 3072, 768, 0, "f32", True, True),
]
# (N, H, W, Cin, Cout, k, s, p, d, act, resid, pad): test_conv and test_conv_tma_epilogue_patch_shapes
CONV = [
    (1, 16, 24, 64, 64, 1, 1, 0, 1, 0, False, 0), (2, 37, 50, 128, 256, 3, 1, 1, 1, 1, False, 0),
    (1, 37, 50, 128, 128, 3, 1, 2, 2, 1, True, 0), (1, 38, 52, 64, 128, 3, 2, 1, 1, 1, False, 0),
    (1, 37, 51, 64, 128, 3, 2, 1, 1, 1, False, 0), (2, 38, 52, 256, 512, 1, 2, 0, 1, 0, False, 0),
    (1, 74, 100, 512, 512, 3, 1, 2, 2, 1, True, 0), (1, 296, 400, 64, 64, 3, 1, 1, 1, 1, False, 0),
    (1, 296, 400, 64, 256, 1, 1, 0, 1, 1, True, 0), (3, 148, 200, 128, 128, 3, 2, 1, 1, 1, False, 0),
    (2, 20, 8, 64, 96, 3, 1, 1, 1, 1, True, 24), (1, 9, 16, 64, 64, 3, 1, 1, 1, 0, True, 24),
    (3, 13, 30, 128, 40, 1, 1, 0, 1, 1, True, 24), (2, 50, 37, 64, 264, 3, 1, 1, 1, 1, False, 24),
]


def _linear(M, K, N, act, resid, f32, in_place):
    L = _lib.lib()
    g = torch.Generator().manual_seed(M * 7 + N + K)
    A = (torch.randn(M, K, generator=g) * 0.5).to(DEV).half()
    W = (torch.randn(N, K, generator=g) * 0.1).to(DEV).half()
    b = torch.randn(N, generator=g).to(DEV)
    ldc = N if in_place else (N + 7) // 8 * 8 + 8
    R = None
    if resid == "f32":
        R = torch.randn(M, ldc, generator=g).to(DEV)
    elif resid == "f16":
        R = torch.randn(M, ldc, generator=g).to(DEV).half()
    out = R if in_place else torch.full((M, ldc), 7.0, device=DEV, dtype=torch.float32 if f32 else torch.float16)
    _lib.check(L.ytk_op_linear_f16(_lib.ptr(A), K, M, K, _lib.ptr(W), N, _lib.ptr(b), _lib.ptr(R),
                                    1 if resid == "f32" else 0, ldc, _lib.ptr(out), 1 if f32 else 0, ldc, act, None))
    torch.cuda.synchronize()
    return out.cpu()


def _conv(N, H, W, Cin, Cout, k, s, p, d, act, resid, pad):
    L = _lib.lib()
    g = torch.Generator().manual_seed(H * W + Cout + 1)
    x = (torch.randn(N, H, W, Cin, generator=g) * 0.5).to(DEV).half()
    w = (torch.randn(Cout, k, k, Cin, generator=g) / (Cin * k * k) ** 0.5).to(DEV).half()
    b = torch.randn(Cout, generator=g).to(DEV)
    Ho = (H + 2 * p - d * (k - 1) - 1) // s + 1
    Wo = (W + 2 * p - d * (k - 1) - 1) // s + 1
    R = torch.randn(N, Ho, Wo, Cout, generator=g).to(DEV).half() if resid else None
    out = torch.full((N, Ho, Wo, Cout + pad), 7.0, device=DEV, dtype=torch.float16)
    _lib.check(L.ytk_op_conv2d_f16(_lib.ptr(x), N, H, W, Cin, Cin, _lib.ptr(w), _lib.ptr(b), k, k, s, p, d, Cout,
                                    _lib.ptr(R), 0, Cout, _lib.ptr(out), 0, Cout + pad, act, 0, None))
    torch.cuda.synchronize()
    return out.cpu()


def _run_all():
    return [_linear(*c) for c in LINEAR] + [_conv(*c) for c in CONV]


@pytest.fixture(scope="module")
def staged(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("staged") / "staged.pt")
    env = dict(os.environ, YTK_EPI="staged", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-s", os.path.abspath(__file__), path], env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return torch.load(path)


def test_tma_epilogue_is_bit_identical_to_staged(staged):
    assert os.environ.get("YTK_EPI", "") == "", "the in-process run must take the default (TMA) epilogue"
    got = _run_all()
    cases = [("linear", c) for c in LINEAR] + [("conv", c) for c in CONV]
    bad = [case for case, a, b in zip(cases, got, staged) if not torch.equal(a, b)]
    assert not bad, bad


if __name__ == "__main__":
    torch.save(_run_all(), sys.argv[1])
