"""GPU: op-level tests of the recognizer's decoding tail - the kernels that pick every character and score the OCR
returns - through the C ABI against float64 / integer references on the kernel's own operands:

  head statistics   ytk_op_linear_rowmax_f16 (gemm_tc_kernel, EPI_ROWMAX), ytk_op_rowmax_finalize_f32,
                    ytk_op_softmax_max_f32
  AR control        ytk_op_ar_control (ar_control_kernel) driven step by step through whole decodes
  refinement input  ytk_op_refine_embed (refine_embed_kernel), ytk_op_apply_rep_cut

Bounds.
  Exact head operands: A in {-2..2}, W in {-1, 0, 1}, integer bias, K = 704.  Every product and every partial sum is
  an integer below 2^11, so every logit is exact in fp32 in any accumulation order.  Ids must equal the smallest
  index of the float64 maximum on every row.  On a row whose maxima are k columns with every other logit at least
  120 below, each chunk sum is an integer: __expf(0) = ex2.approx(0) = 1 exactly, and __expf(-120) underflows to 0.
  The probability must then be fp32(1/k) bitwise, so a missing or double-counted column cannot hide.  k = C for a
  constant row.
  Random head operands: the fp32 GEMM error per logit is at most E = (K + 2) 2^-23 (sum_k |a_k w_k| + |b|).  This is
  the recursive-summation bound with a factor 2 of slack for the tensor core's accumulation order.  Ids are compared
  where the float64 top-2 margin exceeds 2 E_row (E_row = max of E over the row).  The softmax maximum
  p = 1 / sum_j exp(x_j - m) moves by a factor of at most exp(2 max|dx|) under logit errors dx, so its relative
  error is at most
      2 E_row + 48 2^-21 + 65 2^-24 + 2^-22 sum_j t_j |x_j - m| / sum_j t_j,     t_j = exp(x_j - m).
  Each __expf(x) is ex2.approx(x log2 e) with relative error <= 2^-22 (2^-21 here).  The rounding of x and of
  x log2 e adds |x| 2^-23 (the last term).  A term passes through at most 48 rescales by __expf(m_old - m_new) on
  its way to the total: fewer than 30 online updates per thread of softmax_max plus 12 merges, or 4 chunk merges
  plus 8 partial merges plus 5 shuffles in the fused path.  It also passes through at most 64 fp32 additions (a
  positive sum: the relative error is at most the depth times 2^-24) and one division.  rowmax_finalize and
  softmax_max read the same fp32 logits: they agree within twice the last three terms.
  Content embeddings (cin): the LayerNorm bound of tests/test_gpu_decoder_kernels.py,
  1e-5 (1 + |y|) + 2^-20 |mean| rstd |gamma| (1 + |xhat|), plus one fp16 rounding (2^-11 |y| + 2^-25).  Folding
  sqrt(d_real / D) into the table and multiplying by sqrtf(D) again costs 3 2^-24 relative per feature, which the
  1e-5 term covers.

Repetition stop: with the default knobs (period_max 8, min_run_p1 8, min_repeats 3) period 2 cuts any run of 6
equal tokens, before the period-1 rule can see a run of 8.  So the runs of 7 and 8 are cut by p = 2 there, and the
period-1 threshold (7: no cut, 8: cut) is pinned with min_repeats = 5.  The knobs are kernel arguments.

Wrong variants, each checked against the kernels.  For an exact check the kernel must differ on the named rows; for
a tolerance check it must miss by at least 10 x the tolerance:
  the largest index wins ties (tie rows) / the sum skips the ragged last chunk (constant rows: 1/(C - C % 32), and
  random rows, whose ragged chunk carries +12 of bias) / rep_cut = onset instead of onset + period (cut rows) / the
  largest period is tried first (the "aaaaaa" row with min_run_p1 = 6, where p = 1 and p = 2 fire at the same step:
  with the default 8 / 3 knobs two periods never first fire at one step, so no sequence tells the orders apart) /
  the repetition check skips rows that already hold an EOS (the repeat-after-EOS row) / a group ends when any of
  its rows holds an EOS (the named groups) / cin uses pos_q[j] / LN statistics over D instead of d_real / kpad is
  computed from raw without the BOS shift (rows with an EOS in raw[0 .. L-1]).
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle.parseq import detect_repeat_onset
from yomitoku_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EOS = 0
CHAIN = 48 * 2.0 ** -21 + 65 * 2.0 ** -24        # __expf rescales, fp32 additions and the division (docstring)
LN_EPS = 1e-5


def _p(t, elems=0):
    """device pointer of t advanced by `elems` elements"""
    return ctypes.c_void_p(t.data_ptr() + elems * t.element_size())


def _first_max(x):
    """(max, smallest index of the max, largest index of the max) per row"""
    m = x.max(1, keepdim=True).values
    col = torch.arange(x.shape[1], device=x.device)
    eq = x == m
    first = torch.where(eq, col, x.shape[1]).min(1).values
    last = torch.where(eq, col, -1).max(1).values
    return m[:, 0], first, last


# ======================================================================================================== head kernels
def _rowmax(A, W, bias, argmax_only=0):
    """EPI_ROWMAX partials; returns (float32 [M, npart, 4] on the device, npart, block_n).  Float4 slots after the M
    rows' partials hold NaN and must stay so."""
    L = _lib.lib()
    M, K = A.shape
    N = W.shape[0]
    cap = M * 2 * ((N + 63) // 64)
    buf = torch.full(((cap + 16) * 4,), float("nan"), dtype=torch.float32, device=DEV)
    npart, bn = ctypes.c_int(0), ctypes.c_int(0)
    Ad, Wd = A.to(DEV).contiguous(), W.to(DEV).contiguous()
    bd = None if bias is None else bias.to(DEV).float().contiguous()
    _lib.check(L.ytk_op_linear_rowmax_f16(_p(Ad), K, M, K, _p(Wd), N, _lib.ptr(bd), argmax_only, _p(buf), cap,
                                          ctypes.byref(npart), ctypes.byref(bn), None))
    torch.cuda.synchronize()
    n = npart.value
    assert n == 2 * ((N + bn.value - 1) // bn.value)
    assert torch.isnan(buf[M * n * 4:]).all()                     # nothing past the M x npart partials
    return buf[:M * n * 4].reshape(M, n, 4), n, bn.value


def _linear_f32(A, W, bias, ldl):
    """EPI_NORMAL fp32 logits [M, ldl]; +1e30 in the pad columns and in a row after M, which must stay."""
    L = _lib.lib()
    M, K = A.shape
    N = W.shape[0]
    out = torch.full((M + 1, ldl), 1e30, dtype=torch.float32, device=DEV)
    Ad, Wd, bd = A.to(DEV).contiguous(), W.to(DEV).contiguous(), bias.to(DEV).float().contiguous()
    _lib.check(L.ytk_op_linear_f16(_p(Ad), K, M, K, _p(Wd), N, _p(bd), None, 0, 0, _p(out), 1, ldl, 0, None))
    torch.cuda.synchronize()
    assert (out[:M, N:] == 1e30).all() and (out[M] == 1e30).all()
    return out


def _stats(kind, src, rows, C, S=1, g_stride=1, g_off=0, rep_cut=None, ld=None, npart=None, n_out=None):
    """ids / probs of softmax_max (kind 's', src = logits [*, ld]) or rowmax_finalize (kind 'f', src = partials
    [rows, ld] float4).  The outputs hold -7 / NaN sentinels; returns them whole, on the host."""
    L = _lib.lib()
    n_out = rows * g_stride + g_off + 3 if n_out is None else n_out
    ids = torch.full((n_out,), -7, dtype=torch.int32, device=DEV)
    probs = torch.full((n_out,), float("nan"), dtype=torch.float32, device=DEV)
    rc = None if rep_cut is None else torch.as_tensor(rep_cut, dtype=torch.int32).to(DEV)
    if kind == "s":
        _lib.check(L.ytk_op_softmax_max_f32(_p(src), ld, C, rows, S, g_stride, g_off, _lib.ptr(rc), EOS, _p(ids),
                                            _p(probs), None))
    else:
        _lib.check(L.ytk_op_rowmax_finalize_f32(_p(src), ld, npart, C, rows, S, g_stride, g_off, _lib.ptr(rc), EOS,
                                                _p(ids), _p(probs), None))
    torch.cuda.synchronize()
    return ids.cpu(), probs.cpu()


def _rel_tol(x64, E_row=None):
    """relative bound of the softmax maximum of float64 logits x64 [M, C] (docstring); E_row: GEMM error per row"""
    m = x64.max(1, keepdim=True).values
    t = torch.exp(x64 - m)
    s = t.sum(1)
    chain = CHAIN + 2.0 ** -22 * (t * (x64 - m).abs()).sum(1) / s
    return (1.0 / s), chain, chain + (0 if E_row is None else 2 * E_row)


K_EX = 704                 # 8 planted blocks of 64, the bias-cancelling block, 128 noise dims
BC = 512                   # W[:, BC] = -bias: a row with A[BC] = 1 sees no bias
NOISE0 = 576


def _targets(C):
    """the planted maxima of row kinds 0..7"""
    s = 32 * ((C // 2) // 32)
    return [[0],                                       # column 0
            [C - 1],                                   # last column: the ragged chunk unless C % 32 == 0
            [s + 3, s + 17],                           # tie inside one 32-column chunk
            [5, 37],                                   # tie across the two warp sets of tile 0 (chunks 0 and 1)
            [9, C - 2],                                # tie across N tiles (one tile only when C = 64)
            [1, 65] if C > 65 else [1, 33],            # 64 apart: two tiles at block_n 64, one warp set otherwise
            sorted({0, 31, 32, 63, C - 1}),            # k maxima at chunk edges
            [C - 2, C - 1]]                            # tie inside the ragged chunk


def _exact_operands(C, M, seed):
    """Row kinds r % 10: 0..7 planted maxima (targets 128, every other logit <= 0), 8 constant (all 0), 9 random."""
    g = torch.Generator().manual_seed(seed)
    T = _targets(C)
    W = torch.zeros(C, K_EX)
    for k, t in enumerate(T):
        col = torch.full((C,), -1.0)
        col[t] = 1.0
        W[:, 64 * k:64 * (k + 1)] = col[:, None]
    bias = torch.randint(-1, 2, (C,), generator=g).float()
    W[:, BC] = -bias
    noise = torch.randint(-1, 2, (C, K_EX - NOISE0), generator=g).float()
    noise[sorted({c for t in T for c in t})] = 0.0
    W[:, NOISE0:] = noise
    kind = torch.arange(M) % 10
    A = torch.zeros(M, K_EX)
    planted = kind < 8
    A[planted, BC] = 1.0
    A[planted, NOISE0:] = torch.randint(-1, 2, (int(planted.sum()), K_EX - NOISE0), generator=g).float()
    for k in range(8):
        A[kind == k, 64 * k:64 * (k + 1)] = 2.0
    A[kind == 8, BC] = 1.0
    rnd = kind == 9
    A[rnd] = torch.randint(-2, 3, (int(rnd.sum()), K_EX), generator=g).float()
    return A.half(), W.half(), bias, kind, T


# (C, M): the vocabularies of the catalog (7119 = 7121 - 2, 7310 = 7312 - 2) and small heads; M = 300 / 384 are the
# shapes whose shrink rule lands on block_n 128 (3 M tiles x 28 / 29 N tiles of 256 columns < 132 SMs <= 3 x 56).
EXACT_SHAPES = [(7119, 1), (7119, 7), (7119, 129), (7119, 300), (7119, 3200), (7119, 16384), (7310, 7), (7310, 384),
                (7310, 3200), (64, 1), (64, 129), (64, 3200), (100, 7), (100, 16384), (300, 129), (300, 16384)]


@pytest.mark.parametrize("C,M", EXACT_SHAPES)
def test_head_statistics_exact(C, M):
    A, W, bias, kind, T = _exact_operands(C, M, seed=C * 7 + M)
    x64 = A.to(DEV).double() @ W.to(DEV).double().T + bias.to(DEV).double()
    m64, first, last = _first_max(x64)
    part, npart, bn = _rowmax(A, W, bias)
    part_am, npart_am, _ = _rowmax(A, W, bias, argmax_only=1)
    assert npart_am == npart
    # the sum-free mode: the same max and index, sums 0
    assert torch.equal(part_am[..., 0], part[..., 0])
    assert torch.equal(part_am[..., 2].view(torch.int32), part[..., 2].view(torch.int32))     # bit-cast indices
    assert (part_am[..., 1] == 0).all()
    pd = part.contiguous()
    ids_f, probs_f = _stats("f", pd, M, C, ld=npart, npart=npart)
    assert (ids_f[M:] == -7).all() and torch.isnan(probs_f[M:]).all()
    ldl = (C + 255) // 256 * 256
    logits = _linear_f32(A, W, bias, ldl)
    assert torch.equal(logits[:M, :C].double(), x64)                  # exact integers
    ids_s, probs_s = _stats("s", logits, M, C, ld=ldl)                 # +1e30 in the pad columns C..ldl
    assert (ids_s[M:] == -7).all() and torch.isnan(probs_s[M:]).all()
    ids_f, probs_f, ids_s, probs_s = ids_f[:M], probs_f[:M], ids_s[:M], probs_s[:M]
    first_c, last_c = first.cpu().int(), last.cpu().int()
    assert torch.equal(ids_f, first_c) and torch.equal(ids_s, first_c)
    # ar_control's partials path (both modes) picks the same ids
    assert torch.equal(_ar_ids_from(part, npart, M, C), first_c)
    assert torch.equal(_ar_ids_from(part_am, npart, M, C), first_c)
    # the max of the partials is the logit itself
    pmax = part[..., 0].to(DEV).max(1).values.double()
    assert torch.equal(pmax, m64)
    # exact probabilities where every non-maximal logit is >= 120 below the maxima
    kind_d = kind.to(DEV)
    k_max = (x64 == m64[:, None]).sum(1)
    second = torch.where(x64 == m64[:, None], -1e9, x64).max(1).values
    exact = (kind_d <= 8) & ((m64 - second >= 120) | (k_max == C))
    assert bool(exact[kind_d <= 8].all())                             # the planted design holds
    want = (1.0 / k_max.double()).float().cpu()
    ex = exact.cpu()
    assert torch.equal(probs_f[ex], want[ex]) and torch.equal(probs_s[ex], want[ex])
    # random rows: within the chain bound (no GEMM error: the logits are exact)
    p64, chain, tol = _rel_tol(x64)
    r = ~ex
    worst = 0.0
    if r.any():
        for pk in (probs_f, probs_s):
            d = (pk.to(DEV).double() - p64).abs() / (tol * p64)
            worst = max(worst, d[r.to(DEV)].max().item())
        assert worst <= 1.0, worst
    # wrong variants: the largest index on ties; the sum without the ragged chunk on constant rows
    ties = (k_max >= 2).cpu()
    if M >= 3:
        assert ties[kind == 2].all() and ties.any()
        assert (ids_f[ties] != last_c[ties]).all() and (ids_s[ties] != last_c[ties]).all()
    const = (kind == 8)
    if const.any() and C % 32:
        wrong = torch.tensor(1.0 / (C - C % 32), dtype=torch.float32)
        assert (probs_f[const] != wrong).all() and (probs_s[const] != wrong).all()
    print("[head exact] C %d M %d: block_n %d, npart %d, %d exact-probability rows, random rows worst / tol %.3f"
          % (C, M, bn, npart, int(ex.sum()), worst))


def test_head_shapes_reach_every_block_n():
    """The shrink rule picks 64, 128 and 256 on the exact shapes (zero operands; block_n does not depend on K), and
    a capacity one float4 short of M x npart is refused with nothing launched."""
    L = _lib.lib()
    seen = {}
    for C, M in EXACT_SHAPES:
        A = torch.zeros(M, 64, dtype=torch.float16, device=DEV)
        W = torch.zeros(C, 64, dtype=torch.float16, device=DEV)
        part = torch.zeros(M * 2 * ((C + 63) // 64) * 4, dtype=torch.float32, device=DEV)
        npart, bn = ctypes.c_int(0), ctypes.c_int(0)
        _lib.check(L.ytk_op_linear_rowmax_f16(_p(A), 64, M, 64, _p(W), C, None, 0, _p(part), part.numel() // 4,
                                              ctypes.byref(npart), ctypes.byref(bn), None))
        seen[(C, M)] = bn.value
        before = L.ytk_launch_count()
        short = M * npart.value - 1
        assert L.ytk_op_linear_rowmax_f16(_p(A), 64, M, 64, _p(W), C, None, 0, _p(part), short, None, None, None) != 0
        assert b"partials_capacity %d float4s < %d" % (short, short + 1) in L.ytk_last_error()
        assert L.ytk_launch_count() == before
    torch.cuda.synchronize()
    print("[head exact] block_n per (C, M): %s" % seen)
    assert set(seen.values()) == {64, 128, 256}, seen


def _ar_ids_from(part, npart, M, C):
    """one ar_control step on EPI_ROWMAX partials (S = 2, step 0, one group per row): raw[:, 0]"""
    D = 64
    ar = _ArBufs(M, 2, M)
    rg = torch.arange(M, dtype=torch.int32, device=DEV)
    tabs = _tables(C + 2, 2, D, D, seed=1)
    cin = torch.zeros(M, D, dtype=torch.float16, device=DEV)
    pd = part.to(DEV).contiguous()
    _lib.check(_lib.lib().ytk_op_ar_control(_p(pd), npart, C, npart, M, 2, _p(rg), 0, M, ctypes.byref(ar.state()), EOS,
                                            0, 8, 8, 3, _p(tabs["embed"]), _p(tabs["pos_q"]), D, D, _p(tabs["g"]),
                                            _p(tabs["b"]), _p(cin), None))
    torch.cuda.synchronize()
    return ar.raw[:, 0].cpu()


RANDOM_SHAPES = [(7119, 3200, 384), (7119, 129, 768), (7310, 1000, 512), (300, 1000, 512), (100, 7, 64)]


@pytest.mark.parametrize("C,M,K", RANDOM_SHAPES)
def test_head_statistics_random(C, M, K):
    g = torch.Generator().manual_seed(C + M + K)
    A = torch.randn(M, K, generator=g).half()
    W = (torch.randn(C, K, generator=g) * 3.0 / math.sqrt(K)).half()
    bias = torch.randn(C, generator=g) * 0.5
    rag = C % 32
    if rag:
        bias[C - rag:] += 12.0                     # the ragged chunk carries a large share of every row's sum
    Ad, Wd, bd = A.to(DEV).double(), W.to(DEV).double(), bias.to(DEV).double()
    x64 = Ad @ Wd.T + bd
    E = (K + 2) * 2.0 ** -23 * (Ad.abs() @ Wd.abs().T + bd.abs())
    E_row = E.max(1).values
    ldl = (C + 255) // 256 * 256
    logits = _linear_f32(A, W, bias, ldl)
    l32 = logits[:M, :C].double()
    g_err = ((l32 - x64).abs() / E).max().item()
    assert g_err <= 1.0, g_err
    part, npart, bn = _rowmax(A, W, bias)
    pd = part.contiguous()
    ids_f, probs_f = _stats("f", pd, M, C, ld=npart, npart=npart)
    ids_s, probs_s = _stats("s", logits, M, C, ld=ldl)
    ids_f, probs_f, ids_s, probs_s = ids_f[:M], probs_f[:M], ids_s[:M], probs_s[:M]
    # the same accumulators: ids equal the first arg-max of the EPI_NORMAL fp32 logits, and the partials' max is the
    # fp32 logit at that index bitwise
    m32, first32, _ = _first_max(l32)
    assert torch.equal(ids_f, first32.cpu().int()) and torch.equal(ids_s, ids_f)
    assert torch.equal(part[..., 0].to(DEV).max(1).values.double(), m32)
    assert torch.equal(_ar_ids_from(part, npart, M, C), ids_f)
    # ids against float64 where the decision is not within the GEMM error
    top2 = x64.topk(2, 1).values
    decided = ((top2[:, 0] - top2[:, 1]) > 2 * E_row).cpu()
    _, first64, _ = _first_max(x64)
    assert torch.equal(ids_f[decided], first64.cpu().int()[decided])
    # probabilities
    p64, chain, tol = _rel_tol(x64, E_row)
    r_f = ((probs_f.to(DEV).double() - p64).abs() / (tol * p64)).max().item()
    r_s = ((probs_s.to(DEV).double() - p64).abs() / (tol * p64)).max().item()
    assert r_f <= 1.0 and r_s <= 1.0, (r_f, r_s)
    _, chain32, _ = _rel_tol(l32)
    r_fs = ((probs_f.double() - probs_s.double()).abs().to(DEV) / (2 * chain32 * probs_s.to(DEV).double())).max().item()
    assert r_fs <= 1.0, r_fs
    miss = float("inf")
    if rag:
        # wrong variant: the sum of exp(x - m) skips the ragged chunk (m stays the maximum of the whole row)
        p_wrong = 1.0 / torch.exp(x64[:, :C - rag] - x64.max(1, keepdim=True).values).sum(1)
        miss = min(((pk.to(DEV).double() - p_wrong).abs() / (tol * p64)).min().item() for pk in (probs_f, probs_s))
        assert miss >= 10.0, miss
    print("[head random] C %d M %d K %d: block_n %d; GEMM |d| / E %.3g; probs worst / tol finalize %.3g softmax_max %.3g;"
          " finalize vs softmax_max %.3g; ids decided on %d / %d rows; ragged chunk skipped misses by %.0f x tol"
          % (C, M, K, bn, g_err, r_f, r_s, r_fs, int(decided.sum()), M, miss))
    _rep_patch_forms(logits, part, npart, ldl, C, M, {"s": (ids_s, probs_s), "f": (ids_f, probs_f)})


def _rep_patch_forms(logits, part, npart, ldl, C, M, unpatched):
    """The repetition patch as the AR call passes it (g_stride S, g_off = step) and as the refinement chunking does
    (g_stride 1, g_off = r0 >= 16384): patched positions get EOS and exactly 1.0, the others the unpatched result,
    and nothing outside the call's indices is written."""
    S, i = 26, 7
    rep = np.where(np.arange(M) % 3 == 0, i, np.where(np.arange(M) % 3 == 1, -1, (i + 5) % S)).astype(np.int32)
    for kind, src, ld in (("s", logits, ldl), ("f", part.contiguous(), npart)):
        ids0, probs0 = unpatched[kind]
        ids, probs = _stats(kind, src, M, C, S=S, g_stride=S, g_off=i, rep_cut=rep, ld=ld, npart=npart,
                            n_out=M * S + 5)
        at = torch.arange(M) * S + i
        written = torch.zeros(M * S + 5, dtype=torch.bool)
        written[at] = True
        assert (ids[~written] == -7).all() and torch.isnan(probs[~written]).all()
        cut = torch.from_numpy(rep == i)
        assert (ids[at][cut] == EOS).all() and (probs[at][cut] == 1.0).all()
        assert torch.equal(ids[at][~cut], ids0[~cut]) and torch.equal(probs[at][~cut], probs0[~cut])
        r0 = 16384 + 37
        ncrop = (r0 + M) // S + 1
        rep2 = ((np.arange(ncrop) * 7) % (S + 3) - 1).astype(np.int32)          # -1, positions, and cuts >= S
        ids, probs = _stats(kind, src, M, C, S=S, g_stride=1, g_off=r0, rep_cut=rep2, ld=ld, npart=npart,
                            n_out=r0 + M + 5)
        assert (ids[:r0] == -7).all() and (ids[r0 + M:] == -7).all() and torch.isnan(probs[r0 + M:]).all()
        gidx = torch.arange(M) + r0
        cut = torch.from_numpy(rep2)[gidx // S] == gidx % S
        assert (ids[r0:r0 + M][cut] == EOS).all() and (probs[r0:r0 + M][cut] == 1.0).all()
        assert torch.equal(ids[r0:r0 + M][~cut], ids0[~cut]) and torch.equal(probs[r0:r0 + M][~cut], probs0[~cut])


# ======================================================================================================== AR control
class _ArBufs:
    """Device ArState for R rows and G groups, initialised as the engine does (tgt = PAD with BOS first, raw = a
    -7 sentinel the engine does not have), plus two parts' scalars [n_active, step, ticket, pad] x 2."""

    def __init__(self, R, S, G, bos=7119, pad=7120):
        self.S = S
        tgt = torch.full((R, S), pad, dtype=torch.int32)
        tgt[:, 0] = bos
        self.tgt = tgt.to(DEV)
        self.raw = torch.full((R, S), -7, dtype=torch.int32, device=DEV)
        self.rep_cut = torch.full((R,), -1, dtype=torch.int32, device=DEV)
        self.rep_done = torch.zeros(R, dtype=torch.int32, device=DEV)
        self.has_eos = torch.zeros(R, dtype=torch.int32, device=DEV)
        self.group_len = torch.zeros(G, dtype=torch.int32, device=DEV)
        self.open_rows = torch.zeros(G, dtype=torch.int32, device=DEV)
        self.scal = torch.zeros(8, dtype=torch.int32, device=DEV)

    def state(self, r0=0, part=0):
        S = self.S
        return _lib.YtkArState(_p(self.tgt, r0 * S), _p(self.raw, r0 * S), _p(self.rep_cut, r0), _p(self.rep_done, r0),
                               _p(self.has_eos, r0), _p(self.group_len), _p(self.scal, 4 * part),
                               _p(self.scal, 4 * part + 1), _p(self.open_rows), _p(self.scal, 4 * part + 2))

    def host(self):
        return {k: getattr(self, k).cpu().numpy().copy() for k in
                ("tgt", "raw", "rep_cut", "rep_done", "has_eos", "group_len", "open_rows", "scal")}


def _tables(n_tok, S, D, d_real, seed):
    """Embedding tables in the engine's layout: E [n_tok, d_real] float64-exact fp32, embed = fp32(E sqrt(d_real/D))
    zero padded to D; pos_q [S, D] (one row more than the kernels read, for the pos_q[j] variant); LN_c gamma / beta."""
    g = torch.Generator().manual_seed(seed)
    E = torch.randn(n_tok, d_real, generator=g)
    embed = torch.zeros(n_tok, D)
    embed[:, :d_real] = E * math.sqrt(d_real / D)
    pos_q = torch.zeros(S, D)
    pos_q[:, :d_real] = 0.5 * torch.randn(S, d_real, generator=g)
    gam = torch.zeros(D)
    bet = torch.zeros(D)
    gam[:d_real] = 1.0 + 0.3 * torch.randn(d_real, generator=g)
    bet[:d_real] = 0.3 * torch.randn(d_real, generator=g)
    return {"E": E.double(), "embed": embed.to(DEV), "pos_q": pos_q.to(DEV), "pos_q64": pos_q.double(),
            "g": gam.to(DEV), "b": bet.to(DEV), "g64": gam.double(), "b64": bet.double(), "D": D, "d_real": d_real}


def _content_ref(tabs, tok, pos, shift=0, stats_width=None):
    """float64 LN_c(pos_q[pos - 1 + shift] + sqrt(d_real) E[tok]) (pos 0: no pos_q) -> (y [n, D], tol)"""
    D, dr = tabs["D"], tabs["d_real"]
    tok = torch.as_tensor(tok, dtype=torch.long)
    pos = torch.as_tensor(pos, dtype=torch.long)
    x = torch.zeros(len(tok), D, dtype=torch.float64)
    x[:, :dr] = math.sqrt(dr) * tabs["E"][tok]
    pq = tabs["pos_q64"][(pos - 1 + shift).clamp(min=0)]
    x = x + torch.where((pos > 0)[:, None], pq, torch.zeros_like(pq))
    n = dr if stats_width is None else stats_width
    mean = x[:, :n].mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x[:, :n] - mean) ** 2).mean(1, keepdim=True) + LN_EPS)
    xhat = torch.zeros_like(x)
    xhat[:, :dr] = (x[:, :dr] - mean) * rstd
    y = xhat * tabs["g64"] + tabs["b64"]
    tol = (1e-5 * (1 + y.abs()) + 2.0 ** -20 * mean.abs() * rstd * tabs["g64"].abs() * (1 + xhat.abs())
           + 2.0 ** -11 * y.abs() + 2.0 ** -25)
    return y, tol


class _Restated:
    """oracle/parseq.py:185-204 per row, with the engine's per-group stop (a group ends after the step at which every
    one of its rows holds an EOS, or after the last step).  Wrong variants: 'cut_onset', 'largest_period',
    'skip_eos_rows', 'any_eos'."""

    def __init__(self, R, S, row_group, G, bos, pad, rep_on, knobs, variant=None):
        self.S, self.rg, self.G, self.rep_on, self.knobs, self.variant = S, row_group, G, rep_on, knobs, variant
        self.tgt = np.full((R, S), pad, dtype=np.int64)
        self.tgt[:, 0] = bos
        self.raw = np.full((R, S), -7, dtype=np.int64)
        self.rep_cut = np.full(R, -1)
        self.rep_done = np.zeros(R, dtype=np.int64)
        self.has_eos = np.zeros(R, dtype=np.int64)
        self.group_len = np.zeros(G, dtype=np.int64)
        self.rows_of = [np.nonzero(row_group == g)[0] for g in range(G)]

    def _detect(self, seq):
        pmax, run_p1, reps = self.knobs
        if self.variant == "largest_period":
            n = len(seq)
            for p in range(pmax, 0, -1):
                if n < 2 * p:
                    continue
                cnt, start = 1, n - p
                while start - p >= 0 and seq[start - p:start] == seq[n - p:]:
                    cnt += 1
                    start -= p
                if cnt >= (run_p1 if p == 1 else reps):
                    return start, p
            return None
        return detect_repeat_onset(seq, pmax, run_p1, reps)

    def step(self, i, ids):
        """ids: scripted arg-max per row.  Returns (rows processed, final token per processed row)."""
        S, j = self.S, i + 1
        proc = np.nonzero(self.group_len[self.rg] == 0)[0]
        for r in proc:
            self.raw[r, i] = ids[r]
            if j < S:
                self.tgt[r, j] = ids[r]
                skip = self.variant == "skip_eos_rows" and self.has_eos[r]
                if self.rep_on and not self.rep_done[r] and ids[r] != EOS and not skip:
                    hit = self._detect(self.tgt[r, 1:j + 1].tolist())
                    if hit is not None:
                        self.rep_cut[r] = hit[0] + (0 if self.variant == "cut_onset" else hit[1])
                        self.rep_done[r] = 1
                        self.tgt[r, j] = EOS
                if self.tgt[r, j] == EOS:
                    self.has_eos[r] = 1
        for g in range(self.G):
            if self.group_len[g] == 0 and len(self.rows_of[g]):
                eos = self.has_eos[self.rows_of[g]]
                if j >= S:
                    self.group_len[g] = S
                elif (eos.any() if self.variant == "any_eos" else eos.all()):
                    self.group_len[g] = j
        return proc, self.tgt[proc, j] if j < S else None

    def n_active(self):
        return int(sum(1 for g in range(self.G) if self.group_len[g] == 0 and len(self.rows_of[g])))


S_AR = 32
C_AR = 7119


def _scenarios(rng, S=S_AR, C=C_AR):
    """Scripted arg-max sequences (one token per step) by group; returns (scripts [R][S], groups [R], names).
    Named rows / groups: the ones each wrong variant must be caught on."""
    pool = iter(rng.permutation(np.arange(1, C - 3)).tolist())

    def n(k):
        return [next(pool) for _ in range(k)]

    def row(*parts):
        seq = [t for p in parts for t in p]
        return (seq + n(S - len(seq)))[:S]

    rows, groups, names = [], [], {}

    def add(g, name, seq):
        names[name] = len(rows)
        rows.append(seq)
        groups.append(g)

    a = n(1)
    add(0, "run7", row(n(2), a * 7, n(3), [EOS]))
    b = n(1)
    add(0, "run8", row(n(2), b * 8))
    add(0, "eos_then", row(n(3), [EOS]))
    for p in range(2, 9):
        add(1, "per%d_x2" % p, row(n(2), n(p) * 2, n(2), [EOS]))
    add(1, "tail_tokens", row([C - 1, C - 2, C - 3, C - 1], n(4), [EOS]))        # the kernel's scalar tail (C % 4 = 3)
    for p in range(2, 9):
        add(2, "per%d_x3" % p, row(n(2), n(p) * 3))
    c = n(1)
    add(3, "aaaaaa", row(n(2), c * 6))
    d = n(1)
    add(3, "rep_after_eos", row(n(1), [EOS], n(1), d * 8))
    add(3, "eos_tokens", row(n(4), [EOS], n(3), [EOS]))
    add(3, "late_eos", row(n(20), [EOS]))
    e = n(1)
    add(4, "cut_last", row(n(S - 7), e * 6))                    # the 6th repeat is step S - 2: the cut is at j = S - 1
    add(4, "never_eos", row(n(S)))
    add(5, "early_a", row(n(2), [EOS]))
    add(5, "early_b", row(n(3), [EOS]))
    add(6, "first_step", row([EOS]))
    return rows, np.array(groups), names


def _step_logits(rng, ids, live, C, ldl, fused):
    """fp32 logits [R, ldl] whose first arg-max is ids[r]: N(0, 1) values, 8.0 at the token and at up to two larger
    indices (ties), +1e30 in the pad columns (a read shows), NaN on rows of finished groups.  fused: the EPI_ROWMAX
    partials of those logits at block_n 256 (56 per row) and 8 more slots of +1e30 partials."""
    R = len(ids)
    x = rng.standard_normal((R, ldl)).astype(np.float32)
    x[:, C:] = 1e30
    x[np.arange(R), ids] = 8.0
    for r in range(R):
        if r % 2 == 0 and ids[r] < C - 1:
            x[r, C - 1] = 8.0
        if r % 3 == 0 and ids[r] + 40 < C:
            x[r, ids[r] + 40] = 8.0
    x[~live] = np.nan
    if not fused:
        return torch.from_numpy(x).to(DEV), 0, ldl
    ntile = (C + 255) // 256
    v = np.full((R, ntile * 256), -np.inf, dtype=np.float32)
    v[:, :C] = x[:, :C]
    v = v.reshape(R, ntile, 4, 2, 32).transpose(0, 1, 3, 2, 4).reshape(R, ntile, 2, 128)   # [tile][warp set][cols]
    col = (np.arange(ntile)[:, None, None, None] * 256 + np.arange(4)[None, None, :, None] * 64 +
           np.arange(2)[None, :, None, None] * 32 + np.arange(32)[None, None, None, :]).reshape(ntile, 2, 128)
    mx = v.max(-1)
    am = v.argmax(-1)
    idx = np.take_along_axis(np.broadcast_to(col, v.shape), am[..., None], -1)[..., 0].astype(np.int32)
    with np.errstate(invalid="ignore", over="ignore"):
        sm = np.exp(v.astype(np.float64) - mx[..., None].astype(np.float64)).sum(-1).astype(np.float32)
    empty = ~np.isfinite(mx) & (mx < 0)
    idx[empty] = 0x7fffffff
    sm[empty] = 0.0
    npart = 2 * ntile
    P = np.zeros((R, npart + 8, 4), dtype=np.float32)
    P[:, :npart, 0] = mx.reshape(R, npart)
    P[:, :npart, 1] = sm.reshape(R, npart)
    P[:, :npart, 2] = idx.reshape(R, npart).view(np.float32)
    P[:, npart:, 0] = 1e30
    P[:, npart:, 1] = 1.0
    P[~live] = np.nan
    return torch.from_numpy(P).to(DEV), npart, npart + 8


# (name, fused partials, D, d_real, row order, second-part shape, replicas, rep_on, knobs)
AR_FORMS = [("fused-d384", True, 384, 368, "sorted", False, 1, 1, (8, 8, 3)),
            ("unfused-d768", False, 768, 768, "sorted", False, 1, 1, (8, 8, 3)),
            ("unsorted", False, 384, 368, "shuffled", False, 1, 1, (8, 8, 3)),
            ("part2-fused", True, 384, 368, "sorted", True, 1, 1, (8, 8, 3)),
            ("part2-unfused-unsorted", False, 768, 768, "shuffled", True, 1, 1, (8, 8, 3)),
            ("many-fused", True, 384, 368, "sorted", False, 75, 1, (8, 8, 3)),
            ("many-unfused", False, 384, 368, "shuffled", False, 75, 1, (8, 8, 3)),
            ("rep-off", False, 384, 368, "sorted", False, 1, 0, (8, 8, 3)),
            ("min-run-p1-6", True, 384, 368, "sorted", False, 1, 1, (8, 6, 3)),
            ("min-repeats-5", False, 384, 368, "sorted", False, 1, 1, (8, 8, 5))]


@pytest.mark.parametrize("form", AR_FORMS, ids=[f[0] for f in AR_FORMS])
def test_ar_control_whole_decode(form):
    name, fused, D, d_real, order, part2, reps, rep_on, knobs = form
    S, C, bos, pad = S_AR, C_AR, C_AR, C_AR + 1
    rng = np.random.default_rng(len(name) * 1009 + D)
    base, bgroups, names = _scenarios(rng)
    G0 = int(bgroups.max()) + 1
    scripts, groups = [], []
    for k in range(reps):                                   # replicas: the same structure under a token permutation
        perm = np.concatenate([[EOS], rng.permutation(np.arange(1, C))])
        scripts += [[int(perm[t]) if k else t for t in s] for s in base]
        groups += (bgroups + k * G0).tolist()
    scripts, groups = np.array(scripts), np.array(groups)
    if order == "shuffled":
        p = rng.permutation(len(scripts))
        inv = np.argsort(p)
        scripts, groups = scripts[p], groups[p]
        names = {k: int(inv[v]) for k, v in names.items()}
    B, G = len(scripts), int(groups.max()) + 1
    # second-part shape: this launch's rows start at r0 of a larger state, its groups at g0 (global ids)
    r0, g0 = (11, 3) if part2 else (0, 0)
    ar = _ArBufs(r0 + B, S, g0 + G, bos, pad)
    if part2:
        ar.group_len[:g0] = 5                                # the first part's groups and rows must stay untouched
    rg = torch.from_numpy(np.concatenate([np.zeros(r0), groups + g0]).astype(np.int32)).to(DEV)
    tabs = _tables(C + 2, S, D, d_real, seed=D + d_real)
    cin = torch.full((r0 + B + 1, D), 7.0, dtype=torch.float16, device=DEV)
    ref = _Restated(B, S, groups, G, bos, pad, rep_on, knobs)
    variants = {v: _Restated(B, S, groups, G, bos, pad, rep_on, knobs, v)
                for v in ("cut_onset", "largest_period", "skip_eos_rows", "any_eos")}
    first = ar.host()
    worst, miss_pos, miss_ln = 0.0, float("inf"), float("inf")
    done_at = None
    for i in range(S):
        live = ref.group_len[groups] == 0
        if not live.any():
            done_at = i
            break
        ids = scripts[:, i]
        lg, npart, ldl = _step_logits(rng, ids, live, C, (C + 255) // 256 * 256, fused)
        cin_before = cin.cpu()
        _lib.check(_lib.lib().ytk_op_ar_control(
            _p(lg), ldl, C, npart, B, S, _p(rg, r0), g0, G, ctypes.byref(ar.state(r0, 1 if part2 else 0)), EOS, rep_on,
            knobs[0], knobs[1], knobs[2], _p(tabs["embed"]), _p(tabs["pos_q"]), D, d_real, _p(tabs["g"]),
            _p(tabs["b"]), _p(cin, r0 * D), None))
        torch.cuda.synchronize()
        proc, tok = ref.step(i, ids)
        for v in variants.values():
            v.step(i, ids)
        h = ar.host()
        sl = slice(r0, r0 + B)
        for key in ("tgt", "raw", "rep_cut", "rep_done", "has_eos"):
            assert np.array_equal(h[key][sl], getattr(ref, key)), (name, i, key)
            assert np.array_equal(h[key][:r0], first[key][:r0]), (name, i, key)
        assert np.array_equal(h["group_len"][g0:], ref.group_len), (name, i)
        assert np.array_equal(h["group_len"][:g0], first["group_len"][:g0])
        assert (h["open_rows"] == 0).all()
        k = 4 if part2 else 0
        assert h["scal"][k] == ref.n_active() and h["scal"][k + 1] == i + 1 and h["scal"][k + 2] == 0, (name, i)
        assert (h["scal"][4 - k:4 - k + 3] == 0).all()                     # the other part's scalars
        # cin: written for processed rows when j < S, untouched otherwise
        got = cin.cpu()
        touched = np.zeros(r0 + B + 1, dtype=bool)
        if tok is not None:
            touched[r0 + proc] = True
            y, tol = _content_ref(tabs, tok, np.full(len(proc), i + 1))
            gp = got[r0 + proc].double()
            r = ((gp - y).abs() / tol).max().item()
            worst = max(worst, r)
            assert r <= 1.0, (name, i, r)
            assert (gp[:, d_real:] == 0).all()
            if i + 2 <= S - 1:
                yw, _ = _content_ref(tabs, tok, np.full(len(proc), i + 1), shift=1)
                miss_pos = min(miss_pos, ((gp - yw).abs() / tol).max().item())
            if d_real < D:
                yw, _ = _content_ref(tabs, tok, np.full(len(proc), i + 1), stats_width=D)
                miss_ln = min(miss_ln, ((gp - yw).abs() / tol).max().item())
        assert torch.equal(got[~torch.from_numpy(touched)], cin_before[~torch.from_numpy(touched)]), (name, i)
    assert done_at is not None or ref.n_active() == 0
    # every scenario ran the way the scripts intend (a check of the test itself)
    n = names
    if rep_on:
        assert ref.rep_cut[n["run8"]] >= 0 and ref.rep_cut[n["rep_after_eos"]] >= 0
        if knobs[2] == 3:      # p = 2 cuts a run of 6 equal tokens before the period-1 rule can
            p_run = 1 if knobs[1] <= 6 else 2
            assert ref.rep_cut[n["run7"]] == 2 + p_run and ref.rep_cut[n["aaaaaa"]] == 2 + p_run
            assert all(ref.rep_cut[n["per%d_x3" % p]] == 2 + p and ref.rep_cut[n["per%d_x2" % p]] < 0
                       for p in range(2, 9))
            r = n["cut_last"]
            assert ref.tgt[r, S - 1] == EOS and scripts[r, S - 2] != EOS and ref.rep_cut[r] >= 0
        else:                  # min_repeats 5: the period-1 rule decides the runs of 7 and 8
            assert ref.rep_cut[n["run7"]] < 0 and ref.rep_cut[n["run8"]] == 2 + 1
    else:
        assert (ref.rep_cut < 0).all()
    assert ref.group_len[groups[n["never_eos"]]] == S and ref.group_len[groups[n["first_step"]]] == 1
    # wrong variants, each caught on its named rows / groups
    caught = []
    if rep_on:
        cut_rows = np.nonzero(ref.rep_cut >= 0)[0]
        assert (variants["cut_onset"].rep_cut[cut_rows] != ref.rep_cut[cut_rows]).all()
        r = n["rep_after_eos"]
        assert variants["skip_eos_rows"].rep_cut[r] != ref.rep_cut[r]
        caught += ["rep_cut = onset on %d rows" % len(cut_rows), "EOS rows skipped on rep_after_eos"]
        if knobs[1] == 2 * knobs[2]:     # p = 1 and p = 2 first fire at the same step on a run
            r = n["aaaaaa"]
            assert variants["largest_period"].rep_cut[r] != ref.rep_cut[r]
            caught.append("largest period first on aaaaaa")
    any_eos = [g for g in range(G) if variants["any_eos"].group_len[g] != ref.group_len[g]]
    assert set(groups[[n["run7"], n["eos_then"], n["late_eos"], n["early_b"]]]) <= set(any_eos)
    caught.append("any-EOS group end on %d groups" % len(any_eos))
    assert miss_pos >= 10.0, miss_pos
    if d_real < D:
        assert miss_ln >= 10.0, miss_ln
    print("[ar_control] %s: B %d, %d groups, steps %s; cin worst / tol %.3f; pos_q[j] misses by %.0f x, LN over D by %s;"
          " caught: %s" % (name, B, G, done_at or S, worst, miss_pos,
                           "%.0f x" % miss_ln if d_real < D else "-", ", ".join(caught)))


# ======================================================================================================== refinement
@pytest.mark.parametrize("D,d_real", [(384, 368), (768, 768)])
def test_refine_embed_vs_reference(D, d_real):
    """t_in = [BOS, raw[:L-1]], pad_mask = cumsum(t_in == EOS) > 0 (oracle/parseq.py:216-217): klen = L, kpad = the
    first EOS of t_in (L if none), cin = LN_c of each context position (positions >= L hold EOS)."""
    S, C = 51, C_AR
    bos = C
    rng = np.random.default_rng(D)
    raw = rng.integers(1, C, size=(12, S)).astype(np.int32)
    L = np.array([S, S, S, S, 1, 1, 17, 17, 17, 2, S, 30])
    raw[0, 0] = EOS                      # EOS at raw[0]: kpad 1
    raw[1, S - 2] = EOS                  # EOS at raw[L-2]: the last context position
    raw[2, S - 1] = EOS                  # EOS at raw[L-1] only: not in t_in, kpad = L
    raw[4, 0] = EOS                      # L = 1: the context is BOS alone
    raw[6, 15] = EOS                     # L-2
    raw[7, 16] = EOS                     # L-1
    raw[8, 3] = EOS
    raw[8, 9] = EOS                      # two EOS: the first one counts
    raw[9, 0] = EOS                      # L = 2, EOS at raw[0]
    raw[11, 29] = EOS                    # beyond L - 1: ignored
    B = len(L)
    # groups: rows share a group when they share L (the kernel reads group_len[row_group[row]])
    uniq = sorted(set(L.tolist()))
    row_group = np.array([uniq.index(v) for v in L], dtype=np.int32)
    group_len = np.array(uniq, dtype=np.int32)
    tabs = _tables(C + 2, S, D, d_real, seed=D + 3)
    cin = torch.full((B + 1, S, D), 7.0, dtype=torch.float16, device=DEV)
    klen = torch.full((B + 1,), -7, dtype=torch.int32, device=DEV)
    kpad = torch.full((B + 1,), -7, dtype=torch.int32, device=DEV)
    rd, rgd, gld = (torch.from_numpy(a).to(DEV) for a in (raw, row_group, group_len))
    _lib.check(_lib.lib().ytk_op_refine_embed(_p(rd), _p(rgd), _p(gld), B, S, bos, EOS, _p(tabs["embed"]),
                                              _p(tabs["pos_q"]), D, d_real, _p(tabs["g"]), _p(tabs["b"]), _p(cin),
                                              _p(klen), _p(kpad), None))
    torch.cuda.synchronize()
    klen, kpad, cin = klen.cpu().numpy(), kpad.cpu().numpy(), cin.cpu()
    assert klen[B] == -7 and kpad[B] == -7 and (cin[B] == 7.0).all()
    want_kpad, wrong_kpad = [], []
    for r in range(B):
        t_in = np.concatenate([[bos], raw[r, :L[r] - 1]])
        pad_mask = np.cumsum(t_in == EOS) > 0
        want_kpad.append(int(np.argmax(pad_mask)) if pad_mask.any() else int(L[r]))
        hit = np.nonzero(raw[r, :L[r]] == EOS)[0]               # the variant without the BOS shift
        wrong_kpad.append(int(hit[0]) if len(hit) else int(L[r]))
    assert np.array_equal(klen[:B], L)
    assert np.array_equal(kpad[:B], want_kpad), (kpad[:B], want_kpad)
    assert [want_kpad[r] for r in (0, 1, 2, 4)] == [1, S - 1, S, 1]
    named = [r for r in range(B) if wrong_kpad[r] != want_kpad[r]]
    assert set(named) >= {0, 1, 2, 6, 7, 8, 9}
    worst, miss = 0.0, float("inf")
    for r in range(B):
        pos = np.arange(S)
        tok = np.where(pos == 0, bos, np.where(pos < L[r], raw[r, np.maximum(pos - 1, 0)], EOS))
        y, tol = _content_ref(tabs, tok, pos)
        g = cin[r].double()
        rr = ((g - y).abs() / tol).max().item()
        worst = max(worst, rr)
        assert rr <= 1.0, (r, rr)
        assert (g[:, d_real:] == 0).all()
        yw, _ = _content_ref(tabs, tok[:S - 1], pos[:S - 1], shift=1)
        miss = min(miss, ((g[1:S - 1] - yw[1:]).abs() / tol[1:S - 1]).max().item())
    assert miss >= 10.0, miss
    print("[refine_embed] D %d d_real %d: cin worst / tol %.3f; pos_q[pos] misses by %.0f x tol; kpad without the BOS "
          "shift differs on rows %s" % (D, d_real, worst, miss, named))


def test_apply_rep_cut_exact():
    S, C = 26, C_AR
    cut = np.array([-1, S - 1, S, S + 40, 0, 7, -5], dtype=np.int32)
    B = len(cut)
    g = torch.Generator().manual_seed(5)
    ids0 = torch.randint(1, C, (B + 1, S), generator=g, dtype=torch.int32)
    probs0 = torch.rand(B + 1, S, generator=g)
    ids, probs = ids0.to(DEV), probs0.to(DEV)
    cd = torch.from_numpy(cut).to(DEV)
    _lib.check(_lib.lib().ytk_op_apply_rep_cut(_p(cd), B, S, C, EOS, _p(ids), _p(probs), None))
    torch.cuda.synchronize()
    want_i, want_p = ids0.clone(), probs0.clone()
    for r, c in enumerate(cut):
        if 0 <= c < S:
            want_i[r, c] = EOS
            want_p[r, c] = 1.0
    assert torch.equal(ids.cpu(), want_i) and torch.equal(probs.cpu(), want_p)
