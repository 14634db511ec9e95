"""Host-side cost of BatchedOCR.collect with the device calls stubbed out (runs without a GPU):
python scripts/profile_host_collect.py [pages] [workers]"""
import cProfile
import pstats
import sys
import time

import numpy as np

sys.path.insert(0, ".")


def main():
    P = int(sys.argv[1]) if len(sys.argv) > 1 else 16
    W = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    from yomitoku_b200.pipeline import BatchedOCR
    from yomitoku_b200.synth import synthetic_page, synthetic_prob_map
    from yomitoku_b200.text_detector import TextDetector
    from yomitoku_b200.text_recognizer import TextRecognizer
    det = TextDetector(from_pretrained=False, device="cpu")
    rec = TextRecognizer(from_pretrained=False, device="cpu")
    pages, quads = zip(*[synthetic_page(i) for i in range(P)])
    pages = list(pages)
    Hn, Wn = 1184, 1600
    probs = [synthetic_prob_map(q, (Hn, Wn), (1200, 1600)) for q in quads]

    def fake_run_packed(buf, total, descs, n, n_groups, stream=None):
        S = rec.model.max_label_length + 1
        ids = np.random.randint(1, 7000, size=(n, S)).astype(np.int32)
        ids[:, 12] = 0
        return ids, np.full((n, S), 0.9, np.float32), np.full((n_groups,), 13, np.int32)

    rec.model.run_packed = fake_run_packed
    rec.model.run_packed_ptr = lambda ptr, on_device, total, descs, n, n_groups, stream=None: \
        fake_run_packed(None, total, descs, n, n_groups)
    ocr = BatchedOCR(det, rec, det_batch=8, workers=W)
    det.model.detect_pages_table = lambda *a, **k: None      # no GPU here: the maps come from prob_override
    det.model.input_size = lambda h, w: (Hn, Wn)
    for _ in range(4):
        h = ocr.submit(pages, prob_override=probs)
        ocr.collect(h)
    t0 = time.perf_counter()
    h = ocr.submit(pages, prob_override=probs)
    t1 = time.perf_counter()
    host = [f.result() for f in h.futures]
    t2 = time.perf_counter()
    pr = cProfile.Profile()
    pr.enable()
    res = ocr.collect(h)
    pr.disable()
    t3 = time.perf_counter()
    print("submit %.1f ms, wait host %.1f ms, collect %.1f ms, words %d" %
          ((t1 - t0) * 1e3, (t2 - t1) * 1e3, (t3 - t2) * 1e3, sum(len(r.words) for r in res)))
    pstats.Stats(pr).sort_stats("cumulative").print_stats(22)
    ocr.close()


if __name__ == "__main__":
    main()
