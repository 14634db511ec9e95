"""Python restatement of the word-to-element assignment in reference TableSemanticParser.aggregate
(src/yomitoku/table_semantic_parser.py:683-701) with utils/misc.py calc_overlap_ratio / calc_intersection (:35-91):
the loop the CUDA kernel (yomitoku_b200/csrc/table_ops.cu) replaces, kept as the kernel tests' reference.  Not a
product path."""


def overlap_ratio(elem, word):
    """(share of the word's raw area inside the element, computed on int-truncated boxes), 0 without overlap."""
    ax1, ay1, ax2, ay2 = (int(v) for v in elem)
    bx1, by1, bx2, by2 = (int(v) for v in word)
    iw, ih = max(0, min(ax2, bx2) - max(ax1, bx1)), max(0, min(ay2, by2) - max(ay1, by1))
    if iw == 0 or ih == 0:
        return 0
    return (iw * ih) / ((word[2] - word[0]) * (word[3] - word[1]))


def assign_best_overlap(word_boxes, elem_boxes, elem_skip, groups, overlap_th=0.2):
    """Same arguments and results as yomitoku_b200.models.assign_best_overlap: per group (w0, w1, e0, e1) and word,
    (best element index or -1, best ratio), as two lists."""
    best, ratios = [], []
    for w0, w1, e0, e1 in groups:
        for w in range(int(w0), int(w1)):
            word = [float(v) for v in word_boxes[w]]
            b, r = -1, 0
            for e in range(int(e0), int(e1)):
                if elem_skip[e]:
                    continue
                ratio = overlap_ratio([float(v) for v in elem_boxes[e]], word)
                if ratio > r:
                    b, r = e, ratio
            best.append(-1 if b < 0 or r < overlap_th else b)
            ratios.append(float(r))
    return best, ratios


def canonical_kv(dump):
    """A TableSemanticParserSchema.model_dump() with each table's key-value items in a fixed order and without their
    ids.  The reference sorts the items by the top edge of their value cell and leaves items with equal top edges in
    the order its depth-first walk met them, which starts from a Python set of cell ids and so follows the
    per-process string hash; the ids kv0, kv1, ... follow that order.  Everything else is compared as it is."""
    out = dict(dump, tables=[])
    for t in dump["tables"]:
        items = sorted(t["kv_items"], key=lambda kv: (t["cells"][kv["value"]]["box"][1], list(kv["key"]), kv["value"]))
        out["tables"].append(dict(t, kv_items=[dict(kv, id=None) for kv in items]))
    return out
