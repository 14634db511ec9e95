"""GPU: greedy PARSeq strings against the fp32 CPU oracle AT SCALE (north_star: "greedy-decoded strings
character-identical").

2048 crops per model (16 reference mini-batches of 128, ragged widths) through the product's packed path
(`recognize_crops` -> ytk_parseq_forward_crops) and through the oracle batch by batch.  With fp16 operands / fp32
accumulation the worst logit error is ~1e-3 of the logit spread (std ~6), so a row may differ from the oracle only where
the ORACLE'S OWN top-2 margin is below TAU = 0.05 logits at some decision of that row (a coin flip at any precision short
of fp32).  The test counts every differing row, records the margin histogram of all rows and of the differing ones
(printed; also written to $YTK_REPORT_DIR/identity_<model>.json when that is set), and asserts: no differing row whose
smallest decision margin is >= TAU, and |log score - log score_ref| <= 0.05 on the rows above TAU (the orientation fallback thresholds on that score).
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import parseq as ops
from oracle import weights
from yomitoku_b200 import TextRecognizer

pytestmark = pytest.mark.gpu
TAU = 0.05
SCORE_ATOL = 0.05
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _oracle_group(sd, spec, canv, wp):
    x = torch.full((len(canv), 3, 32, wp), -1.0)
    for i, c in enumerate(canv):
        t = torch.from_numpy(c.astype(np.float32)).permute(2, 0, 1)
        x[i, :, :, : c.shape[1]] = (t / 255.0 - 0.5) / 0.5
    logits, aux = ops.parseq_forward(sd, spec, x, return_aux=True)
    p = logits.softmax(-1)
    prob, ids = p.max(-1)
    top2 = logits.topk(2, -1).values
    return ids.numpy(), prob.numpy(), (top2[..., 0] - top2[..., 1]).numpy(), aux["ar_margin"].numpy()


CASES = [
    ("parseq-tiny-dynw-v4", 16, 128, 64, 320, 21),
    ("parseq-large-v4_1", 16, 128, 64, 200, 22),
]
GOLDEN = os.path.join(ROOT, "tests", "golden")


def make_inputs(n_groups, gsize, wlo, whi, seed):
    """The seeded crop set: n_groups reference mini-batches of gsize ragged canvases (numpy PCG64: the same bytes on
    every machine)."""
    rng = np.random.default_rng(seed)
    canv, padded, groups = [], [], []
    for g in range(n_groups):
        ws = 8 * rng.integers(wlo // 8, whi // 8 + 1, size=gsize)
        wp = int(ws.max())
        for w in ws:
            # smooth random strokes on a light background: non-trivial, crop-dependent encoder features
            base = rng.integers(120, 256, size=(1, int(w) // 4 + 1, 3))
            img = np.repeat(base, 4, axis=1)[:, : int(w)] + rng.integers(-40, 40, size=(32, int(w), 3))
            canv.append(np.clip(img, 0, 255).astype(np.uint8))
            padded.append(wp)
            groups.append(g)
    return canv, padded, groups


def oracle_all(name, n_groups, gsize, wlo, whi, seed):
    """fp32 oracle over the whole crop set, group by group: ids, max-probabilities, top-2 logit margins of the final
    logits and the smallest AR-decision margin per row."""
    spec = ops.SPECS[name]
    sd = weights.make_parseq_state_dict(spec, seed=seed, peaked=True)
    canv, padded, _ = make_inputs(n_groups, gsize, wlo, whi, seed)
    out = [[], [], [], []]
    for g in range(n_groups):
        sl = slice(g * gsize, (g + 1) * gsize)
        r = _oracle_group(sd, spec, canv[sl], padded[g * gsize])
        out[0].append(r[0])
        out[1].append(r[1])
        out[2].append(r[2])
        out[3].append(r[3].min(-1) if r[3].ndim > 1 else r[3])
    return [np.concatenate(o, 0) for o in out]


def _reference(name, n_groups, gsize, wlo, whi, seed):
    """Oracle outputs for the case: the committed fixture (tests/golden/identity_<model>.npz, written by
    tests/golden/make_golden_identity.py = oracle_all() above on the build container's CPU) or, without it or with
    YTK_IDENTITY_LIVE=1, the oracle run here (minutes of host time for the large model)."""
    path = os.path.join(GOLDEN, "identity_%s.npz" % name)
    if os.path.exists(path) and os.environ.get("YTK_IDENTITY_LIVE") != "1":
        z = np.load(path)
        assert tuple(int(v) for v in z["case"]) == (n_groups, gsize, wlo, whi, seed), "fixture made for another case"
        return z["ids"].astype(np.int64), z["prob"], z["margin"], z["ar_margin_min"], "fixture"
    torch.set_num_threads(max(1, min(64, os.cpu_count() or 1)))
    return (*oracle_all(name, n_groups, gsize, wlo, whi, seed), "live")


@pytest.mark.parametrize("name,n_groups,gsize,wlo,whi,seed", CASES)
def test_greedy_strings_identical_at_scale(name, n_groups, gsize, wlo, whi, seed):
    spec = ops.SPECS[name]
    sd = weights.make_parseq_state_dict(spec, seed=seed, peaked=True)
    rec = TextRecognizer(model_name=name, from_pretrained=False, device="cuda", dynamic_width=True,
                         batch_bucketing=True)
    rec.model.load_state_dict(sd)
    canv, padded, groups = make_inputs(n_groups, gsize, wlo, whi, seed)
    R_ids, R_prob, R_margin, R_armin, ref_src = _reference(name, n_groups, gsize, wlo, whi, seed)
    ids, probs, glen = rec.model.recognize_crops(canv, padded, groups, n_groups)
    n = len(canv)
    differing, all_low, score_d, score_low = [], [], [], []
    for g in range(n_groups):
        sl = slice(g * gsize, (g + 1) * gsize)
        r_ids, r_prob, r_margin, ar_min = R_ids[sl], R_prob[sl], R_margin[sl], R_armin[sl]
        for b in range(gsize):
            i = g * gsize + b
            row = r_ids[b].tolist()
            m = row.index(0) + 1 if 0 in row else len(row)      # positions the tokenizer reads (incl. the EOS)
            low = min(float(ar_min[b]), float(r_margin[b, :m].min()))
            all_low.append(low)
            if np.array_equal(ids[i, :m], r_ids[b, :m]):
                # scores are compared on rows without coin-flip decisions: a flipped AR token that the refinement
                # repairs leaves the string identical but legitimately changes the context the probabilities saw
                s_gpu = float(np.log(np.maximum(probs[i, :m], 1e-30)).sum())
                s_ref = float(np.log(np.maximum(r_prob[b, :m], 1e-30)).sum())
                (score_d if low >= TAU else score_low).append(abs(s_gpu - s_ref))
            else:
                first = int(np.nonzero(ids[i, :m] != r_ids[b, :m])[0][0])
                differing.append({"row": i, "first_diff_pos": first, "min_margin": low,
                                  "margin_at_diff": float(r_margin[b, first])})
    all_low = np.asarray(all_low)
    edges = [0.0, 0.01, 0.03, 0.1, 0.3, 1.0, 3.0, np.inf]
    hist = {("[%g,%g)" % (a, b)): int(((all_low >= a) & (all_low < b)).sum()) for a, b in zip(edges[:-1], edges[1:])}
    rep = {"model": name, "rows": n, "oracle": ref_src, "differing_rows": len(differing), "differing": differing[:50],
           "min_margin_histogram_all_rows": hist, "rows_below_tau": int((all_low < TAU).sum()), "tau": TAU,
           "max_abs_log_score_diff": float(max(score_d)) if score_d else None,
           "median_abs_log_score_diff": float(np.median(score_d)) if score_d else None,
           "max_abs_log_score_diff_coin_flip_rows": float(max(score_low)) if score_low else None,
           "mean_decoded_len": float(np.mean([(r.tolist().index(0) if 0 in r.tolist() else len(r)) for r in ids])),
           "ar_steps_per_group": [int(v) for v in glen]}
    print("\n[identity] " + json.dumps(rep))
    if os.environ.get("YTK_REPORT_DIR"):
        os.makedirs(os.environ["YTK_REPORT_DIR"], exist_ok=True)
        json.dump(rep, open(os.path.join(os.environ["YTK_REPORT_DIR"], "identity_%s.json" % name), "w"), indent=1)
    bad = [d for d in differing if d["min_margin"] >= TAU]
    assert not bad, "rows differ from the fp32 oracle although every decision margin >= %.2f: %s" % (TAU, bad[:5])
    assert max(score_d) <= SCORE_ATOL, max(score_d)
