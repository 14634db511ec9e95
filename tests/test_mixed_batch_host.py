"""CPU: batches of pages of different sizes on the host side of the OCR path - the page table and detector plan of a
batch (pipeline.BatchPlan), the capacity-sized staging ring, and BatchedOCR over mixed batches with the device calls
replaced by stand-ins: every page must come out as it does from a batch of its own."""
import ctypes

import numpy as np
import pytest
import torch

from yomitoku_b200 import TextDetector, TextRecognizer
from yomitoku_b200 import data as D
from yomitoku_b200.pipeline import BatchedOCR, BatchPlan
from yomitoku_b200.synth import synthetic_page

SHAPES = [(1200, 1600), (900, 1200), (1600, 1200), (600, 800), (1000, 1000), (1200, 1600), (480, 3000), (900, 1200),
          (2339, 1654), (1500, 2000)]


def _input_size(h, w):
    return D.shortest_edge_size(h, w, 1280, 1600)


def test_batch_plan_groups_chunks_and_offsets():
    plan = BatchPlan(SHAPES, _input_size, 2)
    sizes = np.array([h * w * 3 for h, w in SHAPES])
    assert plan.table["page_off"].tolist() == (np.cumsum(sizes) - sizes).tolist()
    assert plan.page_bytes == int(sizes.sum())
    assert plan.table["x1"].tolist() == [w for _, w in SHAPES] and plan.table["y1"].tolist() == [h for h, _ in SHAPES]
    assert plan.inputs == [_input_size(h, w) for h, w in SHAPES]
    # groups by detector input size in order of first appearance, chunks of det_batch, submission order inside
    assert [(hn, wn, idx) for hn, wn, idx in plan.chunks] == [
        (1184, 1600, [0, 1]), (1184, 1600, [3, 5]), (1184, 1600, [7, 9]), (1600, 1184, [2]), (1280, 1280, [4]),
        (256, 1600, [6]), (1600, 1120, [8])]
    assert sorted(i for _, _, idx in plan.chunks for i in idx) == list(range(len(SHAPES)))
    # every chunk's maps are contiguous in the map buffer, in chunk order
    off = 0
    for hn, wn, idx in plan.chunks:
        assert [plan.prob_off[i] for i in idx] == [off + k * hn * wn for k in range(len(idx))]
        off += len(idx) * hn * wn
    assert plan.prob_len == off
    buf = np.arange(plan.prob_len, dtype=np.float32)
    for ch in plan.chunks:
        maps = plan.chunk_maps(buf, ch)
        for j, i in enumerate(ch[2]):
            assert np.array_equal(maps[j], plan.prob_map(buf, i))


def test_same_size_batch_is_one_group_with_the_stacked_layout():
    n, (h, w) = 5, (1200, 1600)
    plan = BatchPlan([(h, w)] * n, _input_size, 2)
    hn, wn = _input_size(h, w)
    assert [c[2] for c in plan.chunks] == [[0, 1], [2, 3], [4]]
    assert plan.table["page_off"].tolist() == [i * h * w * 3 for i in range(n)]
    assert plan.prob_off == [i * hn * wn for i in range(n)]
    det = TextDetector(from_pretrained=False, device="cpu")
    rec = TextRecognizer(model_name="parseq-tiny-dynw-v4", from_pretrained=False, device="cpu")
    ocr = BatchedOCR(det, rec, workers=1, det_batch=2, device_crops=False)
    rng = np.random.default_rng(0)
    pages = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(n)]
    try:
        for shared in (False, True):
            stage, out, _ = ocr._stage(pages, shared)
            assert stage.numpy().tobytes() == np.stack(pages).tobytes()
            assert out.numel() == n * hn * wn
    finally:
        ocr.close()


def test_staging_ring_keeps_one_buffer_per_kind_and_slot():
    """Batches whose byte totals differ reuse (or grow) their slot's buffer instead of adding one per total."""
    det = TextDetector(from_pretrained=False, device="cpu")
    rec = TextRecognizer(model_name="parseq-tiny-dynw-v4", from_pretrained=False, device="cpu")
    ocr = BatchedOCR(det, rec, workers=1, device_crops=False)
    rng = np.random.default_rng(1)
    made = []
    real = BatchedOCR._shared.__globals__["_SharedBuf"]

    class Counting(real):
        def __init__(self, nbytes):
            made.append(nbytes)
            super().__init__(nbytes)

    BatchedOCR._shared.__globals__["_SharedBuf"] = Counting
    try:
        sizes = [[(300, 400)], [(200, 300), (300, 200)], [(64, 64)] * 3, [(300, 400)] * 2, [(100, 500)], [(320, 320)]]
        for k in range(12):
            ocr._slot = k % 3
            pages = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes[k % len(sizes)]]
            stage, _, plan = ocr._stage(pages, shared=True)
            assert stage.numel() == plan.page_bytes
            got = stage.numpy()
            for p, off in zip(pages, plan.table["page_off"]):
                assert np.array_equal(got[int(off):int(off) + p.size].reshape(p.shape), p)
            for kind, ring in ocr._prob_ring.items():
                assert set(ring) <= {0, 1, 2}, kind
        assert sorted(ocr._prob_ring) == ["pages", "prob"]
        assert all(len(ring) <= 3 for ring in ocr._prob_ring.values())
        # 12 batches in 3 slots: buffers are only created when a slot first needs one or needs a larger one
        assert len(made) < 12
    finally:
        BatchedOCR._shared.__globals__["_SharedBuf"] = real
        ocr.close()


def _mixed_pages():
    """Pages cut from synthetic pages to sizes that map to different detector inputs, with the quads inside them."""
    out = []
    for k, (h, w) in enumerate([(1200, 1600), (900, 1200), (1199, 1597), (1000, 1000), (600, 800), (1200, 1600)]):
        page, quads = synthetic_page(140 + k)
        inside = [q for q in quads if max(x for x, _ in q) < w - 1 and max(y for _, y in q) < h - 1]
        out.append((np.ascontiguousarray(page[:h, :w]), inside[:30]))
    return out


class _FakeDev:         # stands for the flat uint8 cuda tensor of canvases
    def __init__(self, arr):
        self.arr = arr

    def data_ptr(self):
        return self.arr.ctypes.data


def _stub_models(monkeypatch, source_downscale=False):
    from oracle import build_crop_host
    from yomitoku_b200 import models as M
    host = ctypes.CDLL(build_crop_host.build())
    vp = ctypes.c_void_p

    def pages_of(pages_dev):                    # (flat buffer, page table)
        flat, table = pages_dev
        assert table.dtype == D.PAGE_DTYPE
        f = flat.numpy()
        return [f[int(t["page_off"]):int(t["page_off"]) + int(t["H"]) * int(t["W"]) * 3].reshape(t["H"], t["W"], 3)
                for t in table]

    def fake_extract(pages_dev, geoms, stream=None):
        sb, cb = D.layout_crop_buffers(geoms)
        scratch, canv = np.zeros(max(sb, 1), np.uint8), np.full(max(cb, 1), 99, np.uint8)
        pg = pages_of(pages_dev)
        for i in sorted(set(geoms["page"].tolist())):
            sel = np.ascontiguousarray(geoms[geoms["page"] == i])
            sel["page"] = 0
            p = np.ascontiguousarray(pg[i])
            host.crop_host_extract(p.ctypes.data_as(vp), p.shape[0], p.shape[1], sel.ctypes.data_as(vp), len(sel),
                                   scratch.ctypes.data_as(vp), canv.ctypes.data_as(vp))
        return _FakeDev(canv), cb

    def fake_halve(pages_dev, stream=None):
        out = []
        for p in pages_of(pages_dev):
            p = np.ascontiguousarray(p)
            H, W = p.shape[:2]
            dH, dW = int(np.rint(H * 0.5)), int(np.rint(W * 0.5))
            d = np.zeros((dH, dW, 3), np.uint8)
            host.crop_host_halve(p.ctypes.data_as(vp), W, H, dW, dH, d.ctypes.data_as(vp))
            out.append(d)
        table, total = D.page_table([d.shape[:2] for d in out])
        return torch.from_numpy(np.concatenate([d.reshape(-1) for d in out])), table

    monkeypatch.setattr(M, "extract_crops_device", fake_extract)
    monkeypatch.setattr(M, "halve_pages_device", fake_halve)
    monkeypatch.setattr(M, "concat_device_buffers",
                        lambda parts, stream=None: parts[0][0] if len(parts) == 1 else
                        _FakeDev(np.concatenate([t.arr[:n] for t, n in parts])))
    det = TextDetector(from_pretrained=False, device="cpu")
    calls = []

    def fake_table(flat, table, out=None, stream=None):
        calls.append([(int(t["H"]), int(t["W"])) for t in table])
        assert len({_input_size(int(t["H"]), int(t["W"])) for t in table}) == 1
        return out

    det.model.detect_pages_table = fake_table
    rec = TextRecognizer(model_name="parseq-tiny-dynw-v4", from_pretrained=False, device="cpu", dynamic_width=True,
                         batch_bucketing=True, source_downscale=source_downscale)
    S = rec.model.max_label_length + 1

    def fake_ptr(ptr, on_device, total, descs, n, n_groups, stream=None):
        raw = np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_uint8)), shape=(total,))
        ids = np.zeros((n, S), np.int32)
        for r, d in enumerate(descs):
            c = raw[int(d["pix_off"]):int(d["pix_off"]) + 32 * int(d["w"]) * 3].astype(np.int64)
            ids[r, 0] = 1 + int((c * (1 + np.arange(c.size) % 251)).sum()) % 7000
            ids[r, 1] = 1 + int(d["wp"]) % 7000
        return ids, np.full((n, S), 0.5, np.float32), np.full((n_groups,), S, np.int32)

    rec.model.run_packed_ptr = fake_ptr
    return det, rec, calls


def _words(results):
    return [[(w.points, w.content, w.det_score, w.rec_score) for w in r.words] for r in results]


@pytest.mark.parametrize("device_crops,workers,source_downscale", [(True, 2, False), (False, 2, False),
                                                                   (True, 1, False), (True, 2, True),
                                                                   (False, 1, False)])
def test_mixed_batch_equals_batches_of_one_through_tables(monkeypatch, device_crops, workers, source_downscale):
    det, rec, calls = _stub_models(monkeypatch, source_downscale)
    mixed = _mixed_pages()
    pages, quads = [p for p, _ in mixed], [q for _, q in mixed]
    ocr = BatchedOCR(det, rec, workers=workers, det_batch=2, device_crops=device_crops)
    ocr._upload_pages = lambda stage, stream=None: stage.clone()
    try:
        got = ocr(pages, quads_override=quads)
        mixed_calls = list(calls)
        single = [ocr([p], quads_override=[q])[0] for p, q in zip(pages, quads)]
        batches = [pages[:3], pages[3:], pages[1:5]]
        qb = [quads[:3], quads[3:], quads[1:5]]
        streamed = list(ocr.stream(batches, lookahead=2, quads_override=qb))
    finally:
        ocr.close()
    assert all(len(r.words) == len(q) > 5 for r, q in zip(got, quads))
    assert _words(got) == _words(single)
    assert [_words(s) for s in streamed] == [_words([single[i] for i in ix]) for ix in ([0, 1, 2], [3, 4, 5],
                                                                                       [1, 2, 3, 4])]
    # one detector call per chunk of pages that share an input size, with the chunk's pages in the table
    plan = BatchPlan([p.shape[:2] for p in pages], _input_size, 2)
    expect = [[pages[i].shape[:2] for i in idx] for _, _, idx in plan.chunks]
    assert mixed_calls == expect and len(plan.chunks) >= 4
    assert any(len(set(c)) > 1 for c in expect)          # a chunk of pages of different sizes


def test_same_size_batch_calls_one_table_per_chunk(monkeypatch):
    det, rec, calls = _stub_models(monkeypatch)
    page, quads = synthetic_page(150)
    ocr = BatchedOCR(det, rec, workers=1, det_batch=2, device_crops=True)
    ocr._upload_pages = lambda stage, stream=None: stage.clone()
    try:
        ocr([page] * 5, quads_override=[quads[:10]] * 5)
    finally:
        ocr.close()
    assert calls == [[(1200, 1600)] * 2, [(1200, 1600)] * 2, [(1200, 1600)]]
