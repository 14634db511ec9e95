"""CPU: the op-level entries of the deformable attention, LayerNorm and single-query attention kernels, of the DBNet
detector's kernels and of the GEMM (linear / convolution) refuse invalid arguments on the host - a nonzero status, a message that names the problem, and no
kernel launch.  The pointers are never dereferenced on these paths, so plain addresses stand in for device buffers."""
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


# ======================================================================================================== DBNet
W_HOST = (ctypes.c_float * (64 * 64 * 4))()      # host weights: large enough for every entry, never read on refusal


def preprocess_table(lib, src=P, n=1, H0=1200, W0=1600, Hn=1184, Wn=1600, canvas=P, table=True):
    """ytk_op_dbnet_preprocess_table_u8 on a table of n evenly spaced H0 x W0 whole pages (at most 4 records are
    written) in a buffer of n 1200x1600 pages."""
    t = (_lib.YtkRtdetrSrc * 4)()
    for i in range(min(n, 4)):
        t[i] = _lib.YtkRtdetrSrc(i * H0 * W0 * 3, H0, W0, 0, 0, W0, H0)
    return lib.ytk_op_dbnet_preprocess_table_u8(src, n * 1200 * 1600 * 3, t if table else None, n, Hn, Wn, canvas,
                                                None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(src=None), b"null argument"), (dict(canvas=None), b"null argument"),
    (dict(n=0), b"0 page records"), (dict(n=65536), b"65536 page records"), (dict(table=False), b"1 page records"),
    (dict(H0=0), b"page 0 (at 0, 0x1600"), (dict(W0=-1), b"page 0 (at 0, 1200x-1"),
    (dict(Hn=0), b"non-positive input size 0x1600"), (dict(Wn=0), b"non-positive input size 1184x0"),
    (dict(canvas=P + 8), b"16-byte aligned"),
])
def test_dbnet_preprocess_table_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, preprocess_table(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _stem(lib, canvas=P, n=1, Hn=96, Wn=160, w=W_HOST, bias=W_HOST, out=P):
    return lib.ytk_op_dbnet_stem_f16(canvas, n, Hn, Wn, w, bias, out, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(canvas=None), b"null argument"), (dict(w=None), b"null argument"), (dict(bias=None), b"null argument"),
    (dict(out=None), b"null argument"),
    (dict(n=0), b"n 0, input 96x160 unsupported"), (dict(Hn=80), b"input 80x160 unsupported (multiples of 32)"),
    (dict(Wn=100), b"input 96x100 unsupported"), (dict(Hn=0), b"input 0x160 unsupported"),
    (dict(Wn=-32), b"input 96x-32 unsupported"),
    (dict(canvas=P + 8), b"16-byte aligned"), (dict(out=P + 2), b"16-byte aligned"),
])
def test_dbnet_stem_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _stem(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _pool(lib, src=P, n=1, H=320, W=320, C=64, out=P):
    return lib.ytk_op_maxpool3x3s2_f16(src, n, H, W, C, out, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(src=None), b"null argument"), (dict(out=None), b"null argument"),
    (dict(n=0), b"n 0, 320x320, C 64 unsupported"), (dict(H=0), b"0x320"), (dict(W=0), b"320x0"),
    (dict(C=12), b"C 12 unsupported"), (dict(C=0), b"C 0 unsupported"),
    (dict(src=P + 8), b"16-byte aligned"), (dict(out=P + 4), b"16-byte aligned"),
])
def test_maxpool_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _pool(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _up(lib, src=P, n=1, Hs=37, Ws=50, C=64, dst=P, Hd=74, Wd=100, ldd=256, coff=64, acc=0):
    return lib.ytk_op_upsample_bilinear_f16(src, n, Hs, Ws, C, dst, Hd, Wd, ldd, coff, acc, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(src=None), b"null argument"), (dict(dst=None), b"null argument"),
    (dict(n=0), b"n 0, 37x50 -> 74x100"), (dict(Hs=0), b"0x50 -> 74x100"), (dict(Wd=0), b"37x50 -> 74x0"),
    (dict(C=20), b"C 20 unsupported"),
    (dict(coff=200), b"channels [200, 264) do not fit a pitch of 256"),
    (dict(C=64, coff=192, ldd=248), b"channels [192, 256) do not fit a pitch of 248"),
    (dict(coff=4), b"channels [4, 68) do not fit"), (dict(coff=-8), b"channels [-8, 56) do not fit"),
    (dict(ldd=260), b"a pitch of 260"),
    (dict(src=P + 8), b"16-byte aligned"), (dict(dst=P + 2), b"16-byte aligned"),
])
def test_upsample_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _up(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _asf(lib, a=P, fuse=P, n=1, H=296, W=400, w1=P, w2=P, sp3=W_HOST, att=W_HOST):
    return lib.ytk_op_asf_f16(a, fuse, n, H, W, w1, w2, sp3, 0.5, att, None, None, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(a=None), b"null argument"), (dict(fuse=None), b"null argument"), (dict(w1=None), b"null argument"),
    (dict(w2=None), b"null argument"), (dict(sp3=None), b"null argument"), (dict(att=None), b"null argument"),
    (dict(n=0), b"n 0, 296x400 unsupported"), (dict(n=65536), b"n 65536, 296x400 unsupported"),
    (dict(H=0), b"0x400 unsupported"), (dict(W=-1), b"296x-1 unsupported"),
    (dict(H=65536, W=32768), b"65536x32768 unsupported"),
    (dict(a=P + 8), b"16-byte aligned"), (dict(fuse=P + 2), b"16-byte aligned"),
])
def test_asf_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _asf(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _head(lib, x=P, n=1, H=37, W=50, w1=W_HOST, b1=W_HOST, w2=W_HOST, prob=P):
    return lib.ytk_op_dbnet_head_f32(x, n, H, W, w1, b1, w2, 0.1, prob, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(x=None), b"null argument"), (dict(w1=None), b"null argument"), (dict(b1=None), b"null argument"),
    (dict(w2=None), b"null argument"), (dict(prob=None), b"null argument"),
    (dict(n=0), b"non-positive size (n 0, 37x50)"), (dict(H=0), b"non-positive size"), (dict(W=-4), b"non-positive size"),
    (dict(x=P + 8), b"x_dev must be 16-byte"), (dict(prob=P + 4), b"prob_dev 8-byte aligned"),
])
def test_dbnet_head_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _head(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


# ======================================================================================================== PARSeq decoding tail
def _rowmax(lib, A=P, lda=384, M=129, K=384, W=P, N=7119, bias=P, part=P, cap=129 * 2 * 28):
    npart, bn = ctypes.c_int(-1), ctypes.c_int(-1)
    st = lib.ytk_op_linear_rowmax_f16(A, lda, M, K, W, N, bias, 0, part, cap, ctypes.byref(npart), ctypes.byref(bn),
                                      None)
    assert npart.value == -1 and bn.value == -1                       # nothing reported on a refusal
    return st


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(A=None), b"null argument"), (dict(W=None), b"null argument"), (dict(part=None), b"null argument"),
    (dict(M=0), b"M 0, K 384, N 7119"), (dict(N=0), b"N 0"), (dict(K=0, lda=0), b"K 0"),
    (dict(K=100, lda=104), b"K 100"), (dict(lda=320), b"lda 320 unsupported"), (dict(lda=388), b"lda 388"),
    (dict(A=P + 8), b"16-byte aligned"), (dict(W=P + 2), b"16-byte aligned"), (dict(bias=P + 4), b"16-byte aligned"),
    (dict(part=P + 8), b"16-byte aligned"),
    # fewer float4s than M x 2 x ceil(N / 256), the fewest partials any N tile gives
    (dict(cap=129 * 2 * 28 - 1), b"partials_capacity 7223 float4s < 7224"), (dict(cap=0), b"partials_capacity 0"),
    (dict(M=1, N=64, cap=1), b"partials_capacity 1 float4s < 2"),
])
def test_linear_rowmax_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _rowmax(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _smax(lib, logits=P, ldl=7168, C=7119, rows=101, S=101, g_stride=1, g_off=0, rep_cut=None, eos=0, ids=P,
          probs=P):
    return lib.ytk_op_softmax_max_f32(logits, ldl, C, rows, S, g_stride, g_off, rep_cut, eos, ids, probs, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(logits=None), b"null argument"), (dict(ids=None), b"null argument"), (dict(probs=None), b"null argument"),
    (dict(ldl=7118), b"ldl 7118 for C 7119"), (dict(ldl=7122), b"ldl 7122 for C 7119"),
    (dict(logits=P + 4), b"not 16-byte aligned"), (dict(C=0), b"C 0"), (dict(rows=0), b"0 rows"),
    (dict(S=0), b"S 0"), (dict(g_stride=-1), b"g_stride -1"), (dict(g_off=-5), b"g_off -5"),
    (dict(eos=-1), b"eos_id -1"),
])
def test_softmax_max_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _smax(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _fin(lib, part=P, ldp=56, npart=56, C=7119, rows=101, S=101, g_stride=1, g_off=0, eos=0, ids=P, probs=P):
    return lib.ytk_op_rowmax_finalize_f32(part, ldp, npart, C, rows, S, g_stride, g_off, None, eos, ids, probs, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(part=None), b"null argument"), (dict(ids=None), b"null argument"), (dict(probs=None), b"null argument"),
    (dict(npart=57), b"npart 57, ldp 56"), (dict(npart=0), b"npart 0"), (dict(part=P + 8), b"not 16-byte aligned"),
    (dict(rows=0), b"0 rows"), (dict(C=-1), b"C -1"), (dict(S=0), b"S 0"), (dict(g_off=-1), b"g_off -1"),
])
def test_rowmax_finalize_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _fin(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _state(**none):
    names = [n for n, _ in _lib.YtkArState._fields_]
    return _lib.YtkArState(*[None if n in none else P + 64 * i for i, n in enumerate(names)])


def _arc(lib, logits=P, ldl=7168, C=7119, npart=0, B=8, S=101, row_group=P, g0=0, ngroups=2, state=None, eos=0,
         rep_on=1, pmax=8, run_p1=8, reps=3, embed=P, pos_q=P, D=384, d_real=368, g_c=P, b_c=P, cin=P):
    state = _state() if state is None else state
    return lib.ytk_op_ar_control(logits, ldl, C, npart, B, S, row_group, g0, ngroups, ctypes.byref(state), eos, rep_on,
                                 pmax, run_p1, reps, embed, pos_q, D, d_real, g_c, b_c, cin, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(D=1028, d_real=1028), b"D 1028 / d_real 1028 unsupported"), (dict(d_real=385), b"D 384 / d_real 385"),
    (dict(d_real=0), b"d_real 0"), (dict(D=0, d_real=0), b"D 0"),
    (dict(npart=-1), b"npart -1"), (dict(B=0), b"B 0"), (dict(S=0), b"S 0"), (dict(C=0, eos=0), b"C 0"),
    (dict(ldl=7116), b"ldl 7116 too small for C 7119"), (dict(ldl=7121), b"ldl 7121"),
    (dict(npart=56, ldl=55), b"ldl 55 too small for C 7119 / npart 56"), (dict(logits=P + 4), b"not 16-byte aligned"),
    (dict(eos=7119), b"eos_id 7119 outside [0, 7119)"), (dict(eos=-1), b"eos_id -1 outside"),
    (dict(ngroups=0), b"0 groups from g0 0"), (dict(g0=-1), b"2 groups from g0 -1"),
    (dict(pmax=0), b"period_max 0"), (dict(run_p1=0), b"min_run_p1 0"), (dict(reps=0), b"min_repeats 0"),
    (dict(logits=None), b"null argument"), (dict(row_group=None), b"null argument"), (dict(embed=None), b"null argument"),
    (dict(pos_q=None), b"null argument"), (dict(g_c=None), b"null argument"), (dict(b_c=None), b"null argument"),
    (dict(cin=None), b"null argument"),
] + [(dict(state=_state(**{n: 1})), b"null argument") for n, _ in _lib.YtkArState._fields_])
def test_ar_control_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _arc(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _ref(lib, raw=P, row_group=P, glen=P, B=8, S=101, bos=7119, eos=0, embed=P, pos_q=P, D=384, d_real=368, g_c=P,
         b_c=P, cin=P, klen=P, kpad=P):
    return lib.ytk_op_refine_embed(raw, row_group, glen, B, S, bos, eos, embed, pos_q, D, d_real, g_c, b_c, cin, klen,
                                   kpad, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(raw=None), b"null argument"), (dict(row_group=None), b"null argument"), (dict(glen=None), b"null argument"),
    (dict(klen=None), b"null argument"), (dict(kpad=None), b"null argument"), (dict(embed=None), b"null argument"),
    (dict(pos_q=None), b"null argument"), (dict(g_c=None), b"null argument"), (dict(b_c=None), b"null argument"),
    (dict(cin=None), b"null argument"),
    (dict(D=1040, d_real=1040), b"D 1040 / d_real 1040"), (dict(d_real=400), b"D 384 / d_real 400"),
    (dict(B=0), b"B 0"), (dict(B=65536), b"B 65536"), (dict(S=0), b"S 0"), (dict(bos=-1), b"bos_id -1"),
    (dict(eos=-2), b"eos_id -2"),
])
def test_refine_embed_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _ref(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(rep_cut=None), b"null argument"), (dict(ids=None), b"null argument"), (dict(probs=None), b"null argument"),
    (dict(B=0), b"B 0"), (dict(S=0), b"S 0"), (dict(C=0), b"C 0"), (dict(eos=-1), b"eos_id -1"),
])
def test_apply_rep_cut_refusals(lib, kwargs, fragment):
    a = dict(rep_cut=P, B=8, S=101, C=7119, eos=0, ids=P, probs=P)
    a.update(kwargs)
    before = lib.ytk_launch_count()
    _refused(lib, lib.ytk_op_apply_rep_cut(a["rep_cut"], a["B"], a["S"], a["C"], a["eos"], a["ids"], a["probs"], None),
             fragment)
    assert lib.ytk_launch_count() == before


# ======================================================================================================== GEMM entries
def _linear(lib, A=P, lda=256, M=300, K=256, W=P, N=200, bias=P, resid=None, resid_f32=0, ldr=0, out=P, out_f32=0,
            ldc=200, act=0):
    return lib.ytk_op_linear_f16(A, lda, M, K, W, N, bias, resid, resid_f32, ldr, out, out_f32, ldc, act, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(out=None), b"null output"),
    # a misaligned output would take the staged epilogue, whose 16-byte stores fault: refused on the host
    (dict(out=P + 8), b"16-byte aligned"), (dict(out=P + 4, out_f32=1), b"16-byte aligned"),
    (dict(resid=P + 8, ldr=200), b"16-byte aligned"), (dict(bias=P + 4), b"16-byte aligned"),
    (dict(ldc=192), b"ldc=192 is less than the 200 columns"), (dict(ldc=196), b"ldc=196 must keep rows 16-byte"),
    (dict(out_f32=1, ldc=196), b"ldc=196 is less than the 200 columns"),
    (dict(resid=P, ldr=192), b"ldr=192 is less than Cout=200"),
    (dict(resid=P, resid_f32=1, ldr=196), b"ldr=196 is less than Cout=200"),
    (dict(N=0), b"Cout=0"), (dict(N=-8), b"Cout=-8"),
    (dict(act=5), b"act 5 unknown"), (dict(act=-1), b"act -1 unknown"),
    (dict(lda=192), b"lda=192 must be >= K=256"), (dict(lda=260), b"lda=260 must be >= K=256 and a multiple of 8"),
    (dict(K=100, lda=104), b"K=100"), (dict(M=0), b"M=0"),
])
def test_linear_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _linear(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _conv(lib, x=P, N=1, H=37, W=50, Cin=128, in_ld=128, w=P, bias=P, k=3, s=1, p=1, d=1, Cout=256, resid=None,
          resid_f32=0, ldr=0, out=P, out_f32=0, ldc=256, act=1, mode=0):
    return lib.ytk_op_conv2d_f16(x, N, H, W, Cin, in_ld, w, bias, k, k, s, p, d, Cout, resid, resid_f32, ldr, out,
                                 out_f32, ldc, act, mode, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(in_ld=120), b"in_ld 120 < Cin 128"),
    # the fused DBNet head (2) and the row statistics (3) need arguments this entry does not take
    (dict(mode=2), b"mode 2 unsupported"), (dict(mode=3), b"mode 3 unsupported"), (dict(mode=-1), b"mode -1"),
    (dict(out=None), b"null output"),
    (dict(out=P + 8), b"16-byte aligned"), (dict(out=P + 8, out_f32=1), b"16-byte aligned"),
    (dict(resid=P + 8, ldr=256), b"16-byte aligned"), (dict(bias=P + 4), b"16-byte aligned"),
    (dict(ldc=248), b"ldc=248 is less than the 256 columns"),
    # 2x2 pixel shuffle: each of the four column blocks of width Cout / 4 is one output pixel's row
    (dict(mode=1, k=1, p=0, ldc=56), b"ldc=56 is less than the 64 columns"),
    (dict(resid=P, ldr=248), b"ldr=248 is less than Cout=256"),
    (dict(Cout=0), b"Cout=0"), (dict(act=7), b"act 7 unknown"),
])
def test_conv2d_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _conv(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


# ======================================================================================================== RT-DETRv2 glue
def _avgpool(lib, src=P, n=1, H=160, W=160, C=256, out=P):
    return lib.ytk_op_rt_avgpool2_f16(src, n, H, W, C, out, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(src=None), b"null argument"), (dict(out=None), b"null argument"),
    (dict(n=0), b"n 0, 160x160, C 256 unsupported"), (dict(H=7), b"7x160"), (dict(W=161), b"160x161"),
    (dict(H=0, W=0), b"0x0"), (dict(C=12), b"C 12 unsupported"), (dict(C=0), b"C 0 unsupported"),
    (dict(src=P + 8), b"16-byte aligned"), (dict(out=P + 2), b"16-byte aligned"),
])
def test_rt_avgpool2_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _avgpool(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _nearest(lib, src=P, lds=512, n=1, Hs=20, Ws=20, C=256, dst=P, ldd=512, coff=0):
    return lib.ytk_op_rt_upsample_nearest2_f16(src, lds, n, Hs, Ws, C, dst, ldd, coff, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(src=None), b"null argument"), (dict(dst=None), b"null argument"),
    (dict(n=0), b"n 0, 20x20, C 256"), (dict(Hs=0), b"0x20"), (dict(Ws=-1), b"20x-1"),
    (dict(C=252), b"C 252 unsupported"), (dict(C=0), b"C 0 unsupported"),
    # 16-byte vectors: pitches and the column offset in whole groups of 8 fp16
    (dict(lds=516), b"lds 516, ldd 512, coff 0 must be non-negative multiples of 8"),
    (dict(ldd=516), b"lds 512, ldd 516, coff 0 must be"), (dict(coff=4), b"coff 4 must be"),
    (dict(coff=-8), b"coff -8 must be"),
    (dict(lds=248), b"pitches too small (lds 248 for C 256"),
    (dict(coff=264), b"ldd 512 for channels [264, 520))"), (dict(ldd=248), b"ldd 248 for channels [0, 256))"),
    (dict(src=P + 8), b"16-byte aligned"), (dict(dst=P + 2), b"16-byte aligned"),
])
def test_rt_upsample_nearest2_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _nearest(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _add(lib, a=P, b=P, b_f32=None, C=256, period=1, out=P, rows=400):
    return lib.ytk_op_rt_add_f16(a, b, b_f32, C, period, out, rows, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(a=None), b"exactly one of b / b_f32"), (dict(out=None), b"exactly one of b / b_f32"),
    (dict(b=None), b"exactly one of b / b_f32"), (dict(b_f32=P), b"exactly one of b / b_f32"),
    (dict(C=252), b"C 252, period 1 unsupported"), (dict(C=0), b"C 0, period"), (dict(rows=0), b"0 rows"),
    (dict(b=None, b_f32=P, period=0), b"period 0 unsupported"),
    (dict(a=P + 8), b"16-byte aligned"), (dict(b=P + 4), b"16-byte aligned"), (dict(out=P + 2), b"16-byte aligned"),
])
def test_rt_add_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _add(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _lv(hw=((80, 80), (40, 40), (20, 20))):
    return _levels(hw, [1] * len(hw))[:2]


def _level_cases(n_levels_key="n_levels"):
    """refusals of the shared level-table check (the deformable attention entry's, without points)"""
    return [
        (dict(level_arrays=(None, None)), b"null argument"), (dict(**{n_levels_key: 0}), b"0 levels unsupported"),
        (dict(**{n_levels_key: 5}), b"5 levels unsupported"),
        (dict(hw=((80, 80), (40, 0), (20, 20))), b"level 1 is 40x0"), (dict(hw=((-1, 80),)), b"level 0 is -1x80"),
        (dict(hw=((65536, 32768),)), b"levels 0..0 hold more than"),
    ]


def _mask(lib, x=P, D=256, bias=P, invalid=P, n_invalid=100, hw=((80, 80), (40, 40), (20, 20)), level_arrays=None,
          n_levels=None, n_img=2):
    h, w = level_arrays if level_arrays is not None else _lv(hw)
    return lib.ytk_op_rt_mask_invalid_f32(x, D, bias, invalid, n_invalid, h, w, len(hw) if n_levels is None else n_levels,
                                          n_img, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(x=None), b"null argument"), (dict(bias=None), b"null argument"), (dict(invalid=None), b"null argument"),
    (dict(D=0), b"D 0, 100 invalid anchors, n_img 2"), (dict(n_invalid=-1), b"-1 invalid anchors"),
    (dict(n_img=0), b"n_img 0 unsupported"),
] + _level_cases())
def test_rt_mask_invalid_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _mask(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def test_rt_mask_invalid_without_anchors_launches_nothing(lib):
    before = lib.ytk_launch_count()
    assert _mask(lib, invalid=None, n_invalid=0) == 0
    assert lib.ytk_launch_count() == before


def _scores(lib, logits=P, ldl=8, C=6, hw=((80, 80), (40, 40), (20, 20)), level_arrays=None, n_levels=None, n_img=2,
            scores=P):
    h, w = level_arrays if level_arrays is not None else _lv(hw)
    return lib.ytk_op_rt_enc_scores_f32(logits, ldl, C, h, w, len(hw) if n_levels is None else n_levels, n_img, scores,
                                        None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(logits=None), b"null argument"), (dict(scores=None), b"null argument"),
    (dict(C=0), b"C 0, ldl 8, n_img 2 unsupported"), (dict(C=9), b"C 9, ldl 8"), (dict(n_img=0), b"n_img 0"),
] + _level_cases())
def test_rt_enc_scores_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _scores(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


def _gather(lib, om=P, D=256, idx=P, K=300, hw=((80, 80), (40, 40), (20, 20)), level_arrays=None, n_levels=None,
            n_img=2, tgt=P, tgt16=P, anchors=P, asel=P):
    h, w = level_arrays if level_arrays is not None else _lv(hw)
    return lib.ytk_op_rt_gather_queries_f32(om, D, idx, K, h, w, len(hw) if n_levels is None else n_levels, n_img, tgt,
                                            tgt16, anchors, asel, None)


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(om=None), b"null argument"), (dict(idx=None), b"null argument"), (dict(tgt=None), b"null argument"),
    (dict(tgt16=None), b"null argument"), (dict(anchors=None), b"null argument"), (dict(asel=None), b"null argument"),
    (dict(D=0), b"D 0, K 300, n_img 2 unsupported"), (dict(K=0), b"K 0"), (dict(n_img=0), b"n_img 0"),
    (dict(K=1 << 30, n_img=4), b"K 1073741824, n_img 4"),
] + _level_cases())
def test_rt_gather_queries_refusals(lib, kwargs, fragment):
    before = lib.ytk_launch_count()
    _refused(lib, _gather(lib, **kwargs), fragment)
    assert lib.ytk_launch_count() == before


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(delta=None), b"null argument"), (dict(ref=None), b"null argument"),
    (dict(n=0), b"0 boxes"), (dict(n=1 << 29), b"536870912 boxes"), (dict(ldd=3), b"ldd 3 unsupported"),
])
def test_rt_ref_update_refusals(lib, kwargs, fragment):
    a = dict(delta=P, ldd=4, asel=None, ref=P, n=600)
    a.update(kwargs)
    before = lib.ytk_launch_count()
    _refused(lib, lib.ytk_op_rt_ref_update_f32(a["delta"], a["ldd"], a["asel"], a["ref"], a["n"], None), fragment)
    assert lib.ytk_launch_count() == before


@pytest.mark.parametrize("kwargs,fragment", [
    (dict(ref=None), b"null argument"), (dict(W=None), b"null argument"), (dict(b=None), b"null argument"),
    (dict(out=None), b"null argument"), (dict(H1=0), b"H1 0, 600 rows"), (dict(rows=0), b"0 rows"),
    (dict(ref=P + 8), b"16-byte aligned"), (dict(W=P + 4), b"16-byte aligned"),
])
def test_rt_qpos_l0_refusals(lib, kwargs, fragment):
    a = dict(ref=P, W=P, b=P, H1=512, out=P, rows=600)
    a.update(kwargs)
    before = lib.ytk_launch_count()
    _refused(lib, lib.ytk_op_rt_qpos_l0_f32(a["ref"], a["W"], a["b"], a["H1"], a["out"], a["rows"], None), fragment)
    assert lib.ytk_launch_count() == before


# ======================================================================================================== PARSeq patchify
_PATCH_CASES = [
    (dict(pos=None), b"null argument"), (dict(A=None), b"null argument"), (dict(x=None), b"null argument"),
    (dict(n=0), b"0 images"), (dict(n=65536), b"65536 images"),
    (dict(ph=3), b"patch 3x8"), (dict(ph=0), b"patch 0x8"), (dict(pw=0), b"patch 4x0"), (dict(ph=64), b"patch 64x8"),
    (dict(full_gw=0), b"full_gw 0"), (dict(D=0), b"D 0 unsupported"),
    (dict(Kpad=95), b"Kpad 95 < 3 * 4 * 8"), (dict(ph=8, pw=8, Kpad=128), b"Kpad 128 < 3 * 8 * 8"),
]


@pytest.mark.parametrize("kwargs,fragment", _PATCH_CASES + [(dict(src=None), b"null argument"),
                                                             (dict(descs=None), b"null argument")])
def test_patchify_u8_refusals(lib, kwargs, fragment):
    a = dict(src=P, descs=P, n=4, ph=4, pw=8, Kpad=128, pos=P, full_gw=100, D=192, A=P, x=P)
    a.update(kwargs)
    before = lib.ytk_launch_count()
    _refused(lib, lib.ytk_op_patchify_u8(a["src"], a["descs"], a["n"], a["ph"], a["pw"], a["Kpad"], a["pos"],
                                         a["full_gw"], a["D"], a["A"], a["x"], None), fragment)
    assert lib.ytk_launch_count() == before


@pytest.mark.parametrize("kwargs,fragment", _PATCH_CASES + [
    (dict(src=None), b"null argument"),
    (dict(W=100), b"W 100 unsupported"), (dict(W=0), b"W 0 unsupported"), (dict(W=-8), b"W -8 unsupported"),
    (dict(W=808), b"W 808 unsupported (a positive multiple of pw 8, at most full_gw 100"),
])
def test_patchify_f32_refusals(lib, kwargs, fragment):
    a = dict(src=P, n=4, W=128, ph=4, pw=8, Kpad=128, pos=P, full_gw=100, D=192, A=P, x=P)
    a.update(kwargs)
    before = lib.ytk_launch_count()
    _refused(lib, lib.ytk_op_patchify_f32(a["src"], a["n"], a["W"], a["ph"], a["pw"], a["Kpad"], a["pos"],
                                          a["full_gw"], a["D"], a["A"], a["x"], None), fragment)
    assert lib.ytk_launch_count() == before


def test_rtdetr_debug_hooks_refuse_null_arguments(lib):
    """The debug hooks of all three handles (RT-DETRv2, DBNet, PARSeq) refuse a null handle, name or shape4."""
    shape = (ctypes.c_int * 4)()
    _refused(lib, lib.ytk_rtdetr_set_debug(None, 1), b"ytk_rtdetr_set_debug: null handle")
    _refused(lib, lib.ytk_rtdetr_debug_tensor(None, 1, b"c3", None, 0, shape), b"ytk_rtdetr_debug_tensor: null argument")
    _refused(lib, lib.ytk_rtdetr_debug_tensor(P, 1, None, None, 0, shape), b"ytk_rtdetr_debug_tensor: null argument")
    _refused(lib, lib.ytk_rtdetr_debug_tensor(P, 1, b"c3", None, 0, None), b"ytk_rtdetr_debug_tensor: null argument")
    dbnet = b"ytk_dbnet_debug_tensor: null argument"
    _refused(lib, lib.ytk_dbnet_debug_tensor(None, 1, 32, 32, b"stem", None, 0, shape), dbnet)
    _refused(lib, lib.ytk_dbnet_debug_tensor(P, 1, 32, 32, None, None, 0, shape), dbnet)
    _refused(lib, lib.ytk_dbnet_debug_tensor(P, 1, 32, 32, b"stem", None, 0, None), dbnet)
    _refused(lib, lib.ytk_parseq_set_debug(None, 1), b"ytk_parseq_set_debug: null handle")
    parseq = b"ytk_parseq_debug_tensor: null argument"
    _refused(lib, lib.ytk_parseq_debug_tensor(None, b"enc.mem", None, 0, shape), parseq)
    _refused(lib, lib.ytk_parseq_debug_tensor(P, None, None, 0, shape), parseq)
    _refused(lib, lib.ytk_parseq_debug_tensor(P, b"enc.mem", None, 0, None), parseq)
