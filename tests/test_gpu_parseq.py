"""GPU: PARSeq engine against the CPU oracle.

Stated tolerances (fp16 operands, fp32 accumulation): logits of rows that took the same token path max |d| < 0.5 % of
the logit standard deviation + 0.01; decoded strings CHARACTER-IDENTICAL for every row whose greedy decisions are not
coin flips - a row may differ from the oracle only if the oracle's own top-2 margin at some decision of that row is
below TAU = 0.05 logits (logit std ~6), and every other row MUST match; scores within 0.05 in the log domain.
tests/test_gpu_parseq_identity.py repeats the identity check on 2 x 2048 crops and records the margin histogram."""
import os

import numpy as np
import pytest
import torch

from oracle import parseq as ops
from oracle import pipeline as opipe
from oracle import weights
from yomitoku_b200 import TextRecognizer
from yomitoku_b200.synth import synthetic_page

pytestmark = pytest.mark.gpu
TAU = 0.05  # logit units; the peaked test weights have a logit std of ~6
LOGIT_TOL = (0.005, 0.01)   # max |d| < 0.5 % of the logit std + 0.01 on rows that took the same token path
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _rec(name, sd=None, **kw):
    r = TextRecognizer(model_name=name, from_pretrained=False, device="cuda", dynamic_width=True, batch_bucketing=True,
                       **kw)
    if sd is not None:
        r.model.load_state_dict(sd)
    return r


def _margin_aware_equal(ids_gpu, logits_ref, aux, tag):
    ids_ref = logits_ref.argmax(-1).numpy()
    ref_margin = logits_ref.topk(2, -1).values
    ref_margin = (ref_margin[..., 0] - ref_margin[..., 1]).numpy()
    n_same = n_low = 0
    for b in range(ids_ref.shape[0]):
        # compare up to and including the first EOS (what the tokenizer reads)
        row = ids_ref[b].tolist()
        n = row.index(0) + 1 if 0 in row else len(row)
        low = min(float(aux["ar_margin"][b].min()), float(ref_margin[b, :n].min()))
        n_low += low < TAU
        if np.array_equal(ids_gpu[b, :n], ids_ref[b, :n]):
            n_same += 1
            continue
        assert low < TAU, "%s row %d differs although every decision margin >= %.2f (min %.3f)" % (tag, b, TAU, low)
    # every row outside the coin-flip set matched (asserted above); inside it most still do
    assert n_same >= ids_ref.shape[0] - n_low
    return n_same


@pytest.mark.parametrize("name,B,W,seed", [("parseq-tiny-dynw-v4", 16, 320, 3), ("parseq-tiny-dynw-v4", 5, 104, 3),
                                           ("parseq-large-v4_1", 8, 160, 4), ("parseq-large-v4_1", 3, 800, 4),
                                           # the rest of the catalog; parseq-tiny (D 368, 8 heads of 46) runs as the
                                           # zero-padded D 384 / head-dim 48 model (csrc/parseq_engine.cu)
                                           ("parseq-tiny", 6, 208, 5), ("parseq-tiny", 2, 400, 5),
                                           ("parseq-small", 4, 160, 6), ("parseq", 4, 240, 7)])
def test_model_seam_vs_oracle(name, B, W, seed):
    spec = ops.SPECS[name]
    sd = weights.make_parseq_state_dict(spec, seed=seed, peaked=True)
    rec = _rec(name, sd)
    img = torch.rand(B, 3, 32, W, generator=torch.Generator().manual_seed(5)) * 2 - 1
    got = rec.model(img)
    ref, aux = ops.parseq_forward(sd, spec, img, return_aux=True)
    assert got.shape == ref.shape == (B, spec.max_label_length + 1, spec.num_classes)
    n_same = _margin_aware_equal(got.argmax(-1).numpy(), ref, aux, name)
    # rows whose AR decisions all had real margins took the same token path: their refined logits agree closely
    # (a row with a near-tie may emit a different token and still be "repaired" to the same ids by the refinement)
    safe = [b for b in range(B) if float(aux["ar_margin"][b].min()) >= TAU and
            torch.equal(got[b].argmax(-1), ref[b].argmax(-1))]
    if safe:
        d = (got[safe] - ref[safe]).abs().max().item()
        assert d < LOGIT_TOL[0] * ref.std().item() + LOGIT_TOL[1], d


@pytest.mark.parametrize("over", [{"decode_ar": 0}, {"decode_ar": 0, "refine_iters": 0}, {"refine_iters": 2},
                                  {"decode_ar": 0, "refine_iters": 2}])
def test_decoder_switches_vs_oracle(over):
    """cfg.decode_ar / cfg.refine_iters (reference parseq.py:192,252-299): non-autoregressive first pass, repeated
    refinement.  The oracle is pinned against the reference for the same switches (oracle/refcheck.py)."""
    import dataclasses
    name = "parseq-tiny-dynw-v4"
    spec = dataclasses.replace(ops.SPECS[name], **over)
    sd = weights.make_parseq_state_dict(spec, seed=3, peaked=True)
    rec = _rec(name)
    rec.model.decode_ar = spec.decode_ar
    rec.model.refine_iters = spec.refine_iters
    rec.model.load_state_dict(sd)
    img = torch.rand(6, 3, 32, 200, generator=torch.Generator().manual_seed(5)) * 2 - 1
    got = rec.model(img)
    ref, aux = ops.parseq_forward(sd, spec, img, return_aux=True)
    assert got.shape == ref.shape
    n_same = _margin_aware_equal(got.argmax(-1).numpy(), ref, aux, str(over))
    same = [b for b in range(6) if torch.equal(got[b].argmax(-1), ref[b].argmax(-1)) and
            float(aux["ar_margin"][b].min()) >= TAU]
    if same:
        assert (got[same] - ref[same]).abs().max().item() < LOGIT_TOL[0] * ref.std().item() + LOGIT_TOL[1]


def test_reference_fixture_strings(charset_v2):
    for tag, kw in (("peaked", dict(peaked=True)), ("repeat", dict(peaked=True, degenerate_repeat=True))):
        z = np.load(os.path.join(G, "parseq_ref_%s.npz" % tag), allow_pickle=True)
        spec = ops.SPECS["parseq-tiny-dynw-v4"]
        sd = weights.make_parseq_state_dict(spec, seed=int(z["weight_seed"]), **kw)
        rec = _rec("parseq-tiny-dynw-v4", sd)
        p = rec.model(torch.from_numpy(z["img"])).softmax(-1)
        strings, scores = rec.tokenizer.decode(p)
        assert strings == list(z["strings"]), tag
        # a score is a product of ~10 probabilities: compare in the log domain (the orientation fallback thresholds on it)
        assert np.allclose(np.log(scores), np.log(z["scores"]), atol=0.05), tag


def test_repetition_stop_and_refine_off():
    spec = ops.SPECS["parseq-tiny-dynw-v4"]
    sd = weights.make_parseq_state_dict(spec, seed=3, peaked=True, degenerate_repeat=True)
    rec = _rec("parseq-tiny-dynw-v4", sd)
    img = torch.rand(4, 3, 32, 200, generator=torch.Generator().manual_seed(1)) * 2 - 1
    ref = ops.parseq_forward(sd, spec, img)
    got = rec.model(img)
    assert torch.equal(got.argmax(-1), ref.argmax(-1))
    assert (got[:, 2, 0] == 30.0).all() and (got[:, 2, 1] == -30.0).all()     # the logit patch at rep_cut
    # refine_iters = 0 (the reference's tests/yaml/text_recognizer.yaml): output length = AR steps run
    rec.model.refine_iters = 0
    spec0 = ops.ParseqSpec(**{**spec.__dict__, "refine_iters": 0})
    ref0 = ops.parseq_forward(sd, spec0, img)
    got0 = rec.model(img)
    assert got0.shape == ref0.shape
    assert torch.equal(got0.argmax(-1), ref0.argmax(-1))


def test_ragged_crops_match_reference_batching(charset_v2):
    """Packed ragged call (many mini-batches, per-crop padded widths) == the reference's batch-by-batch loop."""
    name = "parseq-tiny-dynw-v4"
    spec = ops.SPECS[name]
    sd = weights.make_parseq_state_dict(spec, seed=7, peaked=True)
    rec = _rec(name, sd)
    page, quads = synthetic_page(5)
    quads = quads[:70]
    out, _ = rec(page, quads)
    preds, scores, dirs, aux = opipe.recognize(sd, spec, ops.Tokenizer(charset_v2), page, quads, dynamic_width=True,
                                               batch_bucketing=True, batch_size=10, width_budget=8000,
                                               max_batch_size=64, return_aux=True)
    assert len(aux["plan"]) > 1                       # several reference mini-batches with different padded widths
    assert out.directions == dirs and out.points == quads
    for a, b, m in zip(out.contents, preds, aux["min_margin"]):
        assert a == b or m < TAU, (a, b, m)           # identical unless the oracle's own decision was a coin flip
    same = sum(a == b for a, b in zip(out.contents, preds))
    assert same >= len(quads) - sum(m < TAU for m in aux["min_margin"])
    dl = [abs(np.log(max(sa, 1e-30)) - np.log(max(sb, 1e-30)))
          for a, b, sa, sb in zip(out.contents, preds, out.scores, scores) if a == b]
    assert max(dl) < 0.05, (np.median(dl), max(dl))


def test_large_model_ragged_vs_seam_consistency():
    """Exactness on the device: a crop's result must not depend on what else is packed with it, as long as its
    padded width and group stay the same (SURVEY.md Appendix A9)."""
    name = "parseq-large-v4_1"
    spec = ops.SPECS[name]
    sd = weights.make_parseq_state_dict(spec, seed=9, peaked=True)
    rec = _rec(name, sd)
    rng = np.random.default_rng(0)
    canv = [rng.integers(0, 256, size=(32, w, 3), dtype=np.uint8) for w in (96, 120, 160, 160, 200, 320)]
    ids_a, probs_a, _ = rec.model.recognize_crops(canv, [160, 160, 160, 160, 320, 320], [0, 0, 0, 0, 1, 1], 2)
    ids_b, probs_b, _ = rec.model.recognize_crops(canv[:4], [160] * 4, [0] * 4, 1)
    assert np.array_equal(ids_a[:4], ids_b)
    assert np.allclose(probs_a[:4], probs_b, atol=1e-6)


def test_engine_reuse_smaller_batch_after_larger():
    """State of a previous (larger) call must not leak into the next one on the same handle."""
    name = "parseq-tiny-dynw-v4"
    spec = ops.SPECS[name]
    sd = weights.make_parseq_state_dict(spec, seed=13, peaked=True)
    rec = _rec(name, sd)
    rng = np.random.default_rng(1)
    big = [rng.integers(0, 256, size=(32, 8 * int(w), 3), dtype=np.uint8) for w in rng.integers(9, 40, size=40)]
    small = big[:5]
    fresh = _rec(name, sd)
    ids_ref, probs_ref, glen_ref = fresh.model.recognize_crops(small, [320] * 5, [0] * 5, 1)
    rec.model.recognize_crops(big, [320] * 40, [i // 10 for i in range(40)], 4)
    ids, probs, glen = rec.model.recognize_crops(small, [320] * 5, [0] * 5, 1)
    assert np.array_equal(ids, ids_ref) and np.array_equal(glen, glen_ref)
    assert np.allclose(probs, probs_ref, atol=1e-6)


def _engine_crops(n=200, n_groups=4, seed=21):
    """~200 crops in sorted groups of different padded widths (the layout the two-part AR loop splits)"""
    rng = np.random.default_rng(seed)
    per = n // n_groups
    groups = [min(i // per, n_groups - 1) for i in range(n)]
    widths = [8 * int(w) for w in rng.integers(6, 40, size=n)]
    canv = [rng.integers(0, 256, size=(32, w, 3), dtype=np.uint8) for w in widths]
    padded = [max(widths[j] for j in range(n) if groups[j] == g) for g in groups]
    return canv, padded, groups, n_groups


def test_two_part_ar_loop_matches_one_part(monkeypatch):
    """YTK_AR_SPLIT_MIN=1 runs the AR loop as two row ranges on two streams (second part: g0 > 0, offset state
    pointers, global group ids).  Ids and group lengths must be those of the one-part loop, probabilities within
    1e-6 (test_large_model_ragged_vs_seam_consistency's standard)."""
    name = "parseq-tiny-dynw-v4"
    sd = weights.make_parseq_state_dict(ops.SPECS[name], seed=11, peaked=True)
    rec = _rec(name, sd)
    canv, padded, groups, ng = _engine_crops()
    monkeypatch.delenv("YTK_AR_SPLIT_MIN", raising=False)
    ids_a, probs_a, glen_a = rec.model.recognize_crops(canv, padded, groups, ng)
    monkeypatch.setenv("YTK_AR_SPLIT_MIN", "1")
    ids_b, probs_b, glen_b = rec.model.recognize_crops(canv, padded, groups, ng)
    assert np.array_equal(glen_a, glen_b)
    assert np.array_equal(ids_a, ids_b)
    assert np.allclose(probs_a, probs_b, atol=1e-6)


def test_unfused_head_matches_fused(monkeypatch):
    """YTK_NO_FUSED_HEAD=1 materialises the head logits and runs softmax_max / the logits path of ar_control instead
    of the row-max epilogue.  Both read the same fp32 logits (same plan, same accumulators), so the ids are equal and
    the probabilities agree within the fp32 chain bound of tests/test_gpu_parseq_decode_kernels.py, taken at its
    worst over a row: twice 48 2^-21 + 65 2^-24 + (C - 1) 2^-22 / e."""
    name = "parseq-tiny-dynw-v4"
    spec = ops.SPECS[name]
    sd = weights.make_parseq_state_dict(spec, seed=12, peaked=True)
    rec = _rec(name, sd)
    canv, padded, groups, ng = _engine_crops(seed=22)
    monkeypatch.delenv("YTK_NO_FUSED_HEAD", raising=False)
    ids_a, probs_a, glen_a = rec.model.recognize_crops(canv, padded, groups, ng)
    monkeypatch.setenv("YTK_NO_FUSED_HEAD", "1")
    ids_b, probs_b, glen_b = rec.model.recognize_crops(canv, padded, groups, ng)
    assert np.array_equal(glen_a, glen_b) and np.array_equal(ids_a, ids_b)
    rel = 2 * (48 * 2.0 ** -21 + 65 * 2.0 ** -24 + (spec.num_classes - 1) * 2.0 ** -22 / np.e)
    d = np.abs(probs_a.astype(np.float64) - probs_b) / (rel * probs_b)
    print("[engine] fused vs unfused head: worst |dp| / (rel p) %.3g (rel %.3g)" % (d.max(), rel))
    assert d.max() <= 1.0, d.max()
