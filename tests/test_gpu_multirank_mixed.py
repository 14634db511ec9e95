"""GPU, world_size 2 over NCCL (skipped on single-GPU boxes): the crop scatter for a batch of pages of different sizes.
Each rank holds its pages as one flat device buffer with a page table; the groups that leave a rank are cut from that
table before the all_to_all, and every rank must get back, for each of its own groups, exactly the ids / probabilities a
single-rank run (`_run_groups_dev_local` on the same records and pages) produces."""
import os
import sys

import numpy as np
import pytest
import torch

from test_gpu_multirank import _free_port

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(1200, 1600), (900, 1200), (1000, 1000)]


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from yomitoku_b200 import TextRecognizer
        from yomitoku_b200 import parallel as par
        from yomitoku_b200.data import crop_geometry, page_table
        from yomitoku_b200.pipeline import BatchedOCR
        from yomitoku_b200.synth import peaked_parseq_state_dict, synthetic_page
        from yomitoku_b200.text_recognizer import plan_mini_batches
        rec = TextRecognizer(model_name="parseq-tiny-dynw-v4", from_pretrained=False, device="cuda:%d" % rank,
                             dynamic_width=True, batch_bucketing=True)
        rec.model.load_state_dict(par.broadcast_state_dict(peaked_parseq_state_dict(rec.model.state_dict()), "cuda"))
        ocr = BatchedOCR(None, rec, workers=1, device_crops=True)
        pages, geoms, groups, base = [], [], [], 0
        for i, (h, w) in enumerate(SHAPES):
            page, quads = synthetic_page(60 + 3 * rank + i, height=h, width=w)
            quads = quads[:60] if rank == 0 else quads[:5]          # skew: groups must move from rank 0 to rank 1
            g, _ = crop_geometry(page.shape, quads, rec._cfg.data.img_size, True, page=i)
            widths = g["canvas_w"].tolist()
            plan = plan_mini_batches(widths, np.argsort(g["cw"]).tolist(), True, 16, None, None)
            padded, _ = rec._collate_widths(widths, plan)
            groups += [([widths[k] for k in b], [padded[k] for k in b], base + np.asarray(b, np.int64)) for b in plan]
            pages.append(page)
            geoms.append(g)
            base += len(g)
        geoms = np.concatenate(geoms)
        table, _ = page_table([p.shape[:2] for p in pages])
        flat = torch.from_numpy(np.concatenate([p.reshape(-1) for p in pages])).cuda()
        pages_dev = (flat, table)
        ref = ocr._run_groups_dev_local(groups, geoms, pages_dev, None)
        x0 = dict(par.STATS)
        got = ocr._run_groups_dev(groups, geoms, pages_dev, None)
        moved = par.STATS["exchange_bytes_sent"] - x0["exchange_bytes_sent"]
        recvd = par.STATS["exchange_bytes_received"] - x0["exchange_bytes_received"]
        assert len(got) == len(ref) == len(groups)
        for (ids, probs, glen), (rid, rp, rg) in zip(got, ref):
            assert np.array_equal(ids, rid) and np.array_equal(probs, rp) and glen == rg
        assert (moved > 0) if rank == 0 else (recvd > 0), (rank, moved, recvd)
        q.put((rank, "ok", moved))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, "fail: " + traceback.format_exc(), None))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_mixed_batch_crop_scatter_over_nccl_equals_single_rank():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for rank, status, _ in out:
        assert status == "ok", status
