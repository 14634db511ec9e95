"""CPU: the op-level entries of the deformable attention, LayerNorm and single-query attention kernels refuse invalid
arguments on the host - a nonzero status, a message that names the problem, and no kernel launch.  The pointers are
never dereferenced on these paths, so plain addresses stand in for device buffers."""
import ctypes

import pytest

from yomitoku_b200 import _lib, build

P = 0x10000          # 16-byte aligned stand-in for a device pointer


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.lib()


def _refused(lib, status, fragment):
    assert status != 0
    msg = lib.ytk_last_error()
    assert fragment in msg, msg


def _levels(hw, points):
    arr = lambda v: (ctypes.c_int * len(v))(*v)
    return arr([h for h, _ in hw]), arr([w for _, w in hw]), arr(points)


def _deform(lib, ow=P, ref=P, value=P, out=P, hw=((80, 80), (40, 40), (20, 20)), points=(4, 4, 4), n_levels=None,
            n_img=1, K=300, heads=8, head_dim=32, ldo=288, ldv=1536, voff=256, ldout=256, level_arrays=None):
    h, w, p = level_arrays if level_arrays is not None else _levels(hw, points)
    return lib.ytk_op_deform_attn_f16(ow, ldo, ref, value, ldv, voff, h, w, p, len(hw) if n_levels is None else n_levels,
                                      n_img, K, heads, head_dim, 0.5, out, ldout, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(ow=None), b"null argument"), (dict(ref=None), b"null argument"), (dict(value=None), b"null argument"),
    (dict(out=None), b"null argument"), (dict(level_arrays=(None, None, None)), b"null argument"),
    (dict(n_levels=0), b"0 levels unsupported"), (dict(n_levels=5), b"5 levels unsupported"),
    (dict(n_img=0), b"non-positive size"), (dict(K=0), b"non-positive size"), (dict(heads=0), b"non-positive size"),
    (dict(K=-3), b"non-positive size"), (dict(voff=-256), b"non-positive size"),
    (dict(hw=((80, 80), (0, 40), (20, 20))), b"level 1 is 0x40"),
    (dict(points=(4, 0, 4)), b"level 1 is 40x40 with 0 points"),
    (dict(ldo=287), b"pitches too small"), (dict(ldv=1536, voff=1300), b"pitches too small"),
    (dict(ldout=255), b"pitches too small"), (dict(ref=P + 4), b"16-byte aligned"),
    # the kernel's own limits: head_dim 32 and 12 points per head
    (dict(head_dim=64, ldv=4096, ldout=512), b"head_dim 64 / 12 points"),
    (dict(points=(4, 4, 3), ldo=264), b"head_dim 32 / 11 points"),
])
def test_deform_attn_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _deform(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _ln(lib, x=P, M=8, D=384, d_real=368, gamma=P, beta=P, out_f16=P, out_f32=P, addvec=None, period=1, row0_dev=None,
        row0=0, writeback=0):
    return lib.ytk_op_layernorm_f32(x, M, D, d_real, gamma, beta, 1e-5, out_f16, out_f32, addvec, period, row0_dev, row0,
                                    writeback, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(D=1028, d_real=1028), b"D=1028 / d_real=1028 unsupported"),
    (dict(D=384, d_real=366), b"D=384 / d_real=366 unsupported"),
    (dict(D=384, d_real=388), b"D=384 / d_real=388 unsupported"),
    (dict(D=382, d_real=368), b"D=382 / d_real=368 unsupported"), (dict(d_real=0), b"D=384 / d_real=0 unsupported"),
    (dict(x=None), b"null argument"), (dict(gamma=None), b"null argument"), (dict(beta=None), b"null argument"),
    (dict(M=0), b"0 rows"), (dict(addvec=P, period=0), b"period 0"), (dict(addvec=P, row0=-1), b"first row -1"),
    # with a device pointer for the first table row the value is not read, so only the bad width is refused
    (dict(addvec=P, row0_dev=P, row0=-1, D=1028, d_real=1028), b"D=1028 / d_real=1028 unsupported"),
    (dict(x=P + 8), b"aligned"), (dict(out_f32=P + 4), b"aligned"), (dict(addvec=P + 4), b"aligned"),
    (dict(out_f16=P + 2), b"aligned"),
])
def test_layernorm_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _ln(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _crops(ntoks, tok_offs=None):
    arr = (_lib.YtkCrop * len(ntoks))()
    off = 0
    for i, n in enumerate(ntoks):
        arr[i] = _lib.YtkCrop(0, 0, 0, off if tok_offs is None else tok_offs[i], n, 0)
        off += n
    return arr


def _sqa(lib, mode=0, q=P, kv=P, B=4, S=26, D=384, heads=8, step=P, crops=None, out=P):
    return lib.ytk_op_single_query_attn_f16(mode, q, kv, B, S, D, heads, step, crops, out, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(mode=2), b"mode 2 unknown"), (dict(mode=-1), b"mode -1 unknown"),
    (dict(q=None), b"null argument"), (dict(kv=None), b"null argument"), (dict(out=None), b"null argument"),
    (dict(step=None), b"null argument"), (dict(mode=1, crops=None), b"null argument"),
    (dict(B=0), b"B 0"), (dict(heads=0), b"0 heads"), (dict(D=384, heads=7), b"7 heads"),
    (dict(D=128, heads=8), b"head dim"), (dict(D=1024, heads=8), b"head dim"),
    (dict(S=0), b"S 0 unsupported"), (dict(S=801), b"S 801 unsupported"),
    (dict(q=P + 8), b"16-byte aligned"), (dict(kv=P + 2), b"16-byte aligned"), (dict(out=P + 4), b"16-byte aligned"),
    # the engine's memory limit of 800 tokens per crop, and empty crops
    (dict(mode=1, B=3, crops=_crops([100, 801, 5])), b"crop 1 has 801 tokens"),
    (dict(mode=1, B=2, crops=_crops([0, 5])), b"crop 0 has 0 tokens"),
    (dict(mode=1, B=2, crops=_crops([5, 5], [0, -5])), b"crop 1 has 5 tokens from row -5"),
])
def test_single_query_attn_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _sqa(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before
