"""GPU: the wgmma attention kernel (impl 2) against fp32 softmax attention on the same fp16 operands, at the lengths
where its 64-query units and 64-key tiles change shape (1, 63 / 64 / 65, ...), with more (sequence, head) pairs than
SMs x consumer warpgroups so that every Q buffer and the K/V ring wrap many times.  Covers all four head dims, the
masked refinement self-attention (kpad, causal rows from query 2 on), the refinement cross-attention over per-row key
blocks of a shared memory, and run-to-run determinism."""
import pytest
import torch

from yomitoku_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 4e-3
EDGE_LENS = [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 400]


def _launch(Q, ldq, q_rows, K, V, ldkv, kv_rows, out, seqs, max_q, heads, hd, masked):
    seqs_dev = torch.frombuffer(bytearray(bytes(seqs)), dtype=torch.uint8).to(DEV)
    _lib.check(_lib.lib().ytk_op_attention_f16(Q.data_ptr(), ldq, q_rows, K.data_ptr(), V.data_ptr(), ldkv, kv_rows,
                                               out.data_ptr(), out.shape[1], seqs_dev.data_ptr(), len(seqs), max_q,
                                               heads, hd, 1 if masked else 0, 2, None))
    torch.cuda.synchronize()


def _ref(q, k, v, heads, hd, vis=None):
    """fp32 softmax(q k^T / sqrt(hd)) v per head; q [nq, D], k / v [nk, D], vis [nq, nk] or None."""
    q = q.float().reshape(q.shape[0], heads, hd).transpose(0, 1)
    k = k.float().reshape(k.shape[0], heads, hd).transpose(0, 1)
    v = v.float().reshape(v.shape[0], heads, hd).transpose(0, 1)
    s = (q @ k.transpose(-1, -2)) / hd ** 0.5
    if vis is not None:
        s = s.masked_fill(~vis[None], float("-inf"))
    return (torch.softmax(s, -1) @ v).transpose(0, 1).reshape(q.shape[1], heads * hd)


def _self_attention(lens, heads, hd, seed=0):
    """Packed ragged self-attention: q, k, v are column blocks of one [T, 3D] matrix.  Returns (out, max |d|)."""
    g = torch.Generator().manual_seed(seed)
    D = heads * hd
    T = sum(lens)
    qkv = torch.randn(T, 3 * D, generator=g).to(DEV).half()
    Q, K, V = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    out = torch.full((T, D), 7.0, device=DEV, dtype=torch.float16)
    seqs = (_lib.YtkAttnSeq * len(lens))()
    off = 0
    for i, n in enumerate(lens):
        seqs[i] = _lib.YtkAttnSeq(off, n, off, n, off * 3 * D, n, 0)
        off += n
    _launch(Q, 3 * D, T, K, V, 3 * D, T, out, seqs, max(lens), heads, hd, False)
    worst, off = 0.0, 0
    for n in lens:
        r = slice(off, off + n)
        worst = max(worst, (out[r].float() - _ref(Q[r], K[r], V[r], heads, hd)).abs().max().item())
        off += n
    return out, worst


@pytest.mark.parametrize("hd,heads", [(96, 8), (64, 8), (48, 8), (32, 6)])
def test_unit_edges_all_head_dims(hd, heads):
    lens = EDGE_LENS * 12      # 132 sequences: 792..1056 pairs, more than 132 SMs x 3 warpgroups
    _, d = _self_attention(lens, heads, hd)
    print("[attn units] hd %d max|d| %.5f" % (hd, d))
    assert d < TOL, d


def test_two_launches_identical():
    lens = EDGE_LENS * 6 + [132, 100, 184] * 100
    a, _ = _self_attention(lens, 8, 96, seed=5)
    b, _ = _self_attention(lens, 8, 96, seed=5)
    assert torch.equal(a, b)


def test_masked_refinement_shape():
    """S = 101 shared queries against per-sequence key blocks of S rows: key j visible to query i iff
    (i < 2 or j <= i) and j < kpad.  kpads straddle the 64-key tiles and the second 64-query unit (q0 = 64)."""
    S, heads, hd = 101, 8, 96
    D = heads * hd
    base = [(101, 101), (101, 100), (101, 65), (101, 64), (101, 63), (101, 2), (40, 33), (7, 7), (1, 1), (101, 128 - 27)]
    cases = base * 12
    g = torch.Generator().manual_seed(2)
    qm = torch.randn(S, D, generator=g).to(DEV).half()
    kv = torch.randn(len(cases) * S, 2 * D, generator=g).to(DEV).half()
    K, V = kv[:, :D], kv[:, D:]
    out = torch.full((len(cases) * S, D), 7.0, device=DEV, dtype=torch.float16)
    seqs = (_lib.YtkAttnSeq * len(cases))()
    for i, (n, kp) in enumerate(cases):
        seqs[i] = _lib.YtkAttnSeq(0, S, i * S, n, i * S * 2 * D, kp, 0)
    _launch(qm, D, S, K, V, 2 * D, len(cases) * S, out, seqs, S, heads, hd, True)
    qi = torch.arange(S, device=DEV)[:, None]
    worst = 0.0
    for i, (n, kp) in enumerate(cases):
        kj = torch.arange(n, device=DEV)[None, :]
        vis = ((qi < 2) | (kj <= qi)) & (kj < kp)
        ref = _ref(qm, K[i * S: i * S + n], V[i * S: i * S + n], heads, hd, vis)
        worst = max(worst, (out[i * S: (i + 1) * S].float() - ref).abs().max().item())
    print("[attn units] masked max|d| %.5f" % worst)
    assert worst < TOL, worst


def test_cross_attention_refinement_shape():
    """Refinement cross-attention: row i's S queries attend to its own ntok_i keys of the packed encoder memory
    (K / V = column blocks of one [T, 2D] matrix)."""
    S, heads, hd = 101, 8, 96
    D = heads * hd
    ntok = EDGE_LENS * 10
    T = sum(ntok)
    g = torch.Generator().manual_seed(3)
    Q = torch.randn(len(ntok) * S, D, generator=g).to(DEV).half()
    kv = torch.randn(T, 2 * D, generator=g).to(DEV).half()
    K, V = kv[:, :D], kv[:, D:]
    out = torch.full((len(ntok) * S, D), 7.0, device=DEV, dtype=torch.float16)
    seqs = (_lib.YtkAttnSeq * len(ntok))()
    off = 0
    for i, n in enumerate(ntok):
        seqs[i] = _lib.YtkAttnSeq(i * S, S, i * S, n, off * 2 * D, n, 0)
        off += n
    _launch(Q, D, len(ntok) * S, K, V, 2 * D, T, out, seqs, S, heads, hd, False)
    worst, off = 0.0, 0
    for i, n in enumerate(ntok):
        r = slice(i * S, (i + 1) * S)
        ref = _ref(Q[r], K[off: off + n], V[off: off + n], heads, hd)
        worst = max(worst, (out[r].float() - ref).abs().max().item())
        off += n
    print("[attn units] cross max|d| %.5f" % worst)
    assert worst < TOL, worst
