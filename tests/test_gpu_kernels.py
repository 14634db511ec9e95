"""GPU: kernel-level parity of the wgmma implicit-GEMM convolution / linear op through the C ABI against torch fp32
on the same bf16-rounded operands (tolerance: bf16 output rounding, 2^-8 relative)."""
import pytest
import torch
import torch.nn.functional as F

from yomitoku_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _lib_():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return _lib.lib()


def _check(got, ref, tol=6e-3):
    got, ref = got.float(), ref.float()
    assert not torch.isnan(got).any()
    rel = (got - ref).abs().max().item() / (ref.abs().max().item() + 1e-12)
    assert rel < tol, rel


@pytest.mark.parametrize("M,K,N,act,resid,f32", [
    (128, 64, 64, 0, None, True), (300, 128, 200, 0, None, False), (1000, 768, 2304, 2, None, False),
    (517, 768, 7119, 0, None, True), (640, 3072, 768, 0, "f32", True), (33, 192, 576, 1, "f16", False),
    (257, 192, 200, 3, "f32", False), (129, 64, 100, 0, "f16", True),
    # >= 4 tiles per SM (the persistent CTAs loop over many tiles); 75 / 149 M tiles are odd; N = 2304 has 9 full N
    # tiles, N = 7119 a ragged last one, K = 3072 wraps the stage ring
    (128 * 74 + 5, 768, 2304, 2, None, False), (128 * 148 + 77, 192, 768, 0, "f32", True),
    (128 * 21 + 1, 768, 7119, 0, None, True), (128 * 200, 3072, 768, 0, "f32", True),
    # TMA epilogue (residual boxes by TMA load, results by TMA store): ragged N with a 16-bit residual, one N tile of 64,
    # fp32 in / out over many tiles per CTA (the residual ring wraps), GELU + fp16 residual
    (1000, 128, 72, 0, "f16", False), (4000, 64, 64, 1, "f16", False), (128 * 500 + 3, 64, 256, 0, "f32", True),
    (128 * 300 + 64, 128, 328, 2, "f16", False)])
def test_linear(M, K, N, act, resid, f32):
    L = _lib_()
    g = torch.Generator().manual_seed(M + N)
    A = (torch.randn(M, K, generator=g) * 0.5).to(DEV).half()
    W = (torch.randn(N, K, generator=g) * 0.1).to(DEV).half()
    b = torch.randn(N, generator=g).to(DEV)
    ldc = (N + 7) // 8 * 8 + 8    # pad columns keep a sentinel: nothing is written past Cout
    R = None
    if resid == "f32":
        R = torch.randn(M, ldc, generator=g).to(DEV)
    elif resid == "f16":
        R = torch.randn(M, ldc, generator=g).to(DEV).half()
    out = torch.full((M, ldc), 7.0, device=DEV, dtype=torch.float32 if f32 else torch.float16)
    _lib.check(L.ytk_op_linear_f16(_lib.ptr(A), K, M, K, _lib.ptr(W), N, _lib.ptr(b), _lib.ptr(R),
                                    1 if resid == "f32" else 0, ldc, _lib.ptr(out), 1 if f32 else 0, ldc, act, None))
    torch.cuda.synchronize()
    ref = A.float() @ W.float().t() + b
    if R is not None:
        ref = ref + R[:, :N].float()
    ref = {0: ref, 1: ref.relu(), 2: F.gelu(ref), 3: ref.sigmoid()}[act]
    _check(out[:, :N], ref, 1e-5 if f32 else 6e-3)
    if ldc > N:
        assert (out[:, N:].float() == 7.0).all()       # columns beyond Cout are never written


@pytest.mark.parametrize("N,H,W,Cin,Cout,k,s,p,d,act,resid", [
    (1, 16, 24, 64, 64, 1, 1, 0, 1, 0, False), (2, 37, 50, 128, 256, 3, 1, 1, 1, 1, False),
    (1, 37, 50, 128, 128, 3, 1, 2, 2, 1, True), (1, 38, 52, 64, 128, 3, 2, 1, 1, 1, False),
    (1, 37, 51, 64, 128, 3, 2, 1, 1, 1, False), (2, 38, 52, 256, 512, 1, 2, 0, 1, 0, False),
    (1, 74, 100, 512, 512, 3, 1, 2, 2, 1, True),
    # big maps (>= 4 tiles per SM, odd tile counts): layer-1-like 3x3 and a residual 1x1 on a 296x400 map
    (1, 296, 400, 64, 64, 3, 1, 1, 1, 1, False), (1, 296, 400, 64, 256, 1, 1, 0, 1, 1, True),
    (3, 148, 200, 128, 128, 3, 2, 1, 1, 1, False)])
def test_conv(N, H, W, Cin, Cout, k, s, p, d, act, resid):
    _conv_case(N, H, W, Cin, Cout, k, s, p, d, act, resid)


@pytest.mark.parametrize("N,H,W,Cin,Cout,k,s,p,d,act,resid", [
    # narrow maps: the 128-pixel tile is a 16 x 8 / 8 x 16 / 4 x 32 patch, an epilogue warp's TMA box covers 4 / 2 / 1 rows
    (2, 20, 8, 64, 96, 3, 1, 1, 1, 1, True), (1, 9, 16, 64, 64, 3, 1, 1, 1, 0, True),
    (3, 13, 30, 128, 40, 1, 1, 0, 1, 1, True), (2, 50, 37, 64, 264, 3, 1, 1, 1, 1, False)])
def test_conv_tma_epilogue_patch_shapes(N, H, W, Cin, Cout, k, s, p, d, act, resid):
    _conv_case(N, H, W, Cin, Cout, k, s, p, d, act, resid, pad=24)


def test_linear_residual_in_place_fp32():
    """x += A W^T + b with the residual tensor = the output tensor (PARSeq's residual stream): every box is loaded before
    the same box is stored."""
    L = _lib_()
    g = torch.Generator().manual_seed(5)
    M, K, N = 128 * 90 + 17, 768, 768
    A = (torch.randn(M, K, generator=g) * 0.5).to(DEV).half()
    W = (torch.randn(N, K, generator=g) * 0.05).to(DEV).half()
    b = torch.randn(N, generator=g).to(DEV)
    x = torch.randn(M, N, generator=g).to(DEV)
    ref = x + A.float() @ W.float().t() + b
    _lib.check(L.ytk_op_linear_f16(_lib.ptr(A), K, M, K, _lib.ptr(W), N, _lib.ptr(b), _lib.ptr(x), 1, N, _lib.ptr(x), 1,
                                    N, 0, None))
    torch.cuda.synchronize()
    _check(x, ref, 1e-5)


def _conv_case(N, H, W, Cin, Cout, k, s, p, d, act, resid, pad=0):
    L = _lib_()
    g = torch.Generator().manual_seed(H * W + Cout)
    x = (torch.randn(N, H, W, Cin, generator=g) * 0.5).to(DEV).half()
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).to(DEV).half()
    wp = w.permute(0, 2, 3, 1).contiguous()
    b = torch.randn(Cout, generator=g).to(DEV)
    Ho = (H + 2 * p - d * (k - 1) - 1) // s + 1
    Wo = (W + 2 * p - d * (k - 1) - 1) // s + 1
    R = torch.randn(N, Ho, Wo, Cout, generator=g).to(DEV).half() if resid else None
    # pad > 0: the output lives in a wider buffer (channel pitch Cout + pad) whose extra channels must stay untouched
    out = torch.full((N, Ho, Wo, Cout + pad), 7.0, device=DEV, dtype=torch.float16)
    _lib.check(L.ytk_op_conv2d_f16(_lib.ptr(x), N, H, W, Cin, Cin, _lib.ptr(wp), _lib.ptr(b), k, k, s, p, d, Cout,
                                    _lib.ptr(R), 0, Cout, _lib.ptr(out), 0, Cout + pad, act, 0, None))
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b, stride=s, padding=p, dilation=d).permute(0, 2, 3, 1)
    if R is not None:
        ref = ref + R.float()
    if act == 1:
        ref = ref.relu()
    _check(out[..., :Cout], ref)
    if pad:
        assert (out[..., Cout:].float() == 7.0).all()


def test_conv_transpose_shuffle_epilogue():
    L = _lib_()
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(1, 20, 28, 64, generator=g) * 0.5).to(DEV).half()
    wt = (torch.randn(64, 64, 2, 2, generator=g) * 0.1).to(DEV).half()
    wp = wt.permute(2, 3, 1, 0).reshape(256, 64).contiguous()
    b = torch.randn(64, generator=g).to(DEV)
    out = torch.empty((1, 40, 56, 64), device=DEV, dtype=torch.float16)
    _lib.check(L.ytk_op_conv2d_f16(_lib.ptr(x), 1, 20, 28, 64, 64, _lib.ptr(wp), _lib.ptr(b.repeat(4).contiguous()), 1,
                                    1, 1, 0, 1, 256, None, 0, 0, _lib.ptr(out), 0, 64, 1, 1, None))
    torch.cuda.synchronize()
    ref = F.conv_transpose2d(x.float().permute(0, 3, 1, 2), wt.float(), b, stride=2).relu().permute(0, 2, 3, 1)
    _check(out, ref)


def test_bad_arguments_fail_loudly():
    L = _lib_()
    x = torch.zeros(1, 8, 8, 48, device=DEV, dtype=torch.float16)
    w = torch.zeros(64, 1, 1, 48, device=DEV, dtype=torch.float16)
    out = torch.zeros(1, 8, 8, 64, device=DEV, dtype=torch.float16)
    st = L.ytk_op_conv2d_f16(_lib.ptr(x), 1, 8, 8, 48, 48, _lib.ptr(w), None, 1, 1, 1, 0, 1, 64, None, 0, 0,
                              _lib.ptr(out), 0, 64, 0, 0, None)
    assert st != 0 and b"multiple of 64" in L.ytk_last_error()


# ---------------------------------------------------------------------------------------------------- attention
def _attn_case(hd, heads, lens, masked, impl, seed=0, q_shared=None, kpads=None, qscale=1.0):
    """Packed ragged self-attention (q, k, v = column blocks of one [T, 3D] matrix) or, with q_shared = S, the refinement
    shape (S shared queries, per-sequence key blocks of S rows with k_len / kpad).  Returns (max |d| of O, ref scale)."""
    import ctypes
    L = _lib.lib()
    g = torch.Generator().manual_seed(seed)
    D = hd * heads
    nseq = len(lens)
    if q_shared is None:
        T = sum(lens)
        qkv = torch.randn(T, 3 * D, generator=g)
        qkv[:, :D] *= qscale
        qkv = qkv.to(DEV).half()
        Q, K, V = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
        ldq = ldkv = 3 * D
        q_rows = kv_rows = T
        out = torch.full((T, D), 7.0, device=DEV, dtype=torch.float16)
        seqs = (_lib.YtkAttnSeq * nseq)()
        off = 0
        for i, n in enumerate(lens):
            seqs[i] = _lib.YtkAttnSeq(off, n, off, n, off * 3 * D, n, 0)
            off += n
        max_q = max(lens)
    else:
        S = q_shared
        qm = torch.randn(S, D, generator=g).to(DEV).half()
        kv = torch.randn(nseq * S, 2 * D, generator=g).to(DEV).half()
        Q, K, V = qm, kv[:, :D], kv[:, D:]
        ldq, ldkv = D, 2 * D
        q_rows, kv_rows = S, nseq * S
        out = torch.full((nseq * S, D), 7.0, device=DEV, dtype=torch.float16)
        seqs = (_lib.YtkAttnSeq * nseq)()
        for i, n in enumerate(lens):
            seqs[i] = _lib.YtkAttnSeq(0, S, i * S, n, i * S * 2 * D, kpads[i] if kpads else n, 0)
        max_q = S
    seqs_dev = torch.frombuffer(bytearray(bytes(seqs)), dtype=torch.uint8).to(DEV)
    _lib.check(L.ytk_op_attention_f16(Q.data_ptr(), ldq, q_rows, K.data_ptr(), V.data_ptr(), ldkv, kv_rows,
                                      out.data_ptr(), D, seqs_dev.data_ptr(), nseq, max_q, heads, hd,
                                      1 if masked else 0, impl, None))
    torch.cuda.synchronize()
    worst = 0.0
    for i, n in enumerate(lens):
        if q_shared is None:
            q = Q[seqs[i].q_off: seqs[i].q_off + n].float()
            k = K[seqs[i].q_off: seqs[i].q_off + n].float()
            v = V[seqs[i].q_off: seqs[i].q_off + n].float()
            o = out[seqs[i].o_off: seqs[i].o_off + n].float()
        else:
            S = q_shared
            q = Q.float()
            k = K[i * S: i * S + n].float()
            v = V[i * S: i * S + n].float()
            o = out[i * S: (i + 1) * S].float()
        q = q.reshape(q.shape[0], heads, hd).transpose(0, 1)
        k = k.reshape(n, heads, hd).transpose(0, 1)
        v = v.reshape(n, heads, hd).transpose(0, 1)
        s = (q @ k.transpose(-1, -2)) / hd ** 0.5
        if masked:
            qi = torch.arange(q.shape[1], device=DEV)[:, None]
            kj = torch.arange(n, device=DEV)[None, :]
            vis = ((qi < 2) | (kj <= qi)) & (kj < (kpads[i] if kpads else n))
            s = s.masked_fill(~vis[None], float("-inf"))
        ref = (torch.softmax(s, -1) @ v).transpose(0, 1).reshape(q.shape[1], D)
        worst = max(worst, (o - ref).abs().max().item())
    return worst


@pytest.mark.parametrize("impl", [1, 2])     # 1: mma.sync kernel, 2: wgmma kernel (default)
@pytest.mark.parametrize("hd,heads,lens", [(96, 8, [132, 92, 48, 200, 400, 129, 128, 4]), (32, 6, [800, 320, 64, 8, 72]),
                                           (48, 8, [100, 260]), (64, 8, [160, 96, 31]),
                                           # RT-DETRv2: AIFI at 960 / 640, cell decoder (1500 queries), layout decoder
                                           (32, 8, [900, 900]), (32, 8, [400] * 3), (32, 8, [1500, 1500]),
                                           (32, 8, [300] * 4)])
def test_attention_tc_vs_torch(hd, heads, lens, impl):
    """Both attention kernels (parseq_ops.cu mma.sync, attn_tc.cu wgmma) vs fp32 softmax attention on the same fp16 operands: the only rounding the
    kernel adds is P and O in fp16 (2^-11 relative)."""
    d = _attn_case(hd, heads, lens, False, impl)
    print("[attn] impl %d hd %d max|d| %.5f" % (impl, hd, d))
    assert d < 4e-3, d


@pytest.mark.parametrize("impl", [1, 2])
def test_attention_tc_masked_refinement_shape(impl):
    d = _attn_case(96, 8, [101, 40, 7, 1, 64, 65], True, impl, q_shared=101, kpads=[101, 33, 7, 1, 20, 65])
    print("[attn] impl %d masked max|d| %.5f" % (impl, d))
    assert d < 4e-3, d


def test_attention_tc_many_sequences_long_rescale():
    """Many pairs per worker (the persistent pipeline wraps its barriers many times) and scores with a large spread (the
    lazy rescale of the running max fires)."""
    import ctypes
    d = _attn_case(96, 8, [132] * 300 + [260] * 40, False, 2, seed=3, qscale=3.0)
    assert d < 6e-3, d


def test_attention_legacy_kernel_still_matches():
    assert _attn_case(96, 8, [132, 92, 200], False, 1) < 4e-3
