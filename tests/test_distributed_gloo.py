"""CPU, world_size 2 over gloo: the multi-GPU plumbing (weight broadcast, group balancing, crop scatter, result
gather) with a stand-in recognizer - the exchange logic is independent of the model.  Every crop source (records cut
"on the device", the crop arena, packed host canvases) takes the same planned exchange."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _fake_recognise(canvases):
    """Deterministic function of the crop pixels only: ids[i, :] = checksum-derived, probs = mean pixel."""
    S = 101
    ids = np.zeros((len(canvases), S), np.int32)
    probs = np.zeros((len(canvases), S), np.float32)
    for i, c in enumerate(canvases):
        ids[i, :] = (int(c.astype(np.int64).sum()) + np.arange(S)) % 7119
        probs[i, :] = float(c.mean()) / 255.0
    return ids, probs


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from yomitoku_b200 import parallel as par
    try:
        # ---- weight broadcast
        g = torch.Generator().manual_seed(100 + rank)
        sd = {"a.weight": torch.randn(4, 3, generator=g), "b.bias": torch.randn(5, generator=g),
              "n": torch.tensor(7, dtype=torch.long)}
        out = par.broadcast_state_dict(sd)
        ref = torch.randn(4, 3, generator=torch.Generator().manual_seed(100))
        assert torch.equal(out["a.weight"], ref) and out["n"].item() == 7
        # ---- unbalanced groups: rank 0 owns 6 groups, rank 1 owns 1
        rng = np.random.default_rng(rank)
        n_groups = 6 if rank == 0 else 1
        groups = []
        for gi in range(n_groups):
            n = int(rng.integers(1, 5))
            widths = (rng.integers(9, 40, size=n) * 8).tolist()
            canv = [rng.integers(0, 256, size=(32, w, 3), dtype=np.uint8) for w in widths]
            groups.append((canv, [max(widths)] * n))
        costs = [sum(4 * (p // 8) for p in g[1]) for g in groups]
        all_costs = par.all_gather_objects(costs, "plan")
        assert all_costs[rank] == costs and len(all_costs) == world
        assign = par.balance_groups(all_costs, world)
        loads = [0.0] * world
        for r in range(world):
            for gi, d in enumerate(assign[r]):
                loads[d] += all_costs[r][gi]
        before = max(sum(c) for c in all_costs)
        assert max(loads) < before            # balancing helped
        q.put((rank, "ok", loads))
    except Exception as e:  # pragma: no cover
        import traceback
        q.put((rank, "fail: " + traceback.format_exc(), None))
    finally:
        dist.destroy_process_group()


class _StubModel:
    """Stands in for models.PARSeq's packed device entry, computed from the crop pixels on the host."""
    refine_iters = 1
    max_label_length = 100

    def __init__(self, cfg):
        self.cfg = cfg
        self.calls = 0

    def run_packed_ptr(self, ptr, on_device, total, descs, n, n_groups, stream=None):
        import ctypes
        self.calls += 1
        raw = np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_uint8)), shape=(total,))
        canv = [raw[int(d["pix_off"]):int(d["pix_off"]) + 32 * int(d["w"]) * 3].reshape(32, int(d["w"]), 3)
                for d in descs]
        ids, probs = _fake_recognise(canv)
        return ids, probs, np.full((n_groups,), 101, np.int32)


def _exchange_spy(par_mod, moved):
    """Wraps parallel.exchange_canvases_planned: records the split sizes of every crop scatter."""
    orig = par_mod.exchange_canvases_planned

    def spy(canv, send_splits, recv_splits, out=None):
        assert isinstance(canv, torch.Tensor) and canv.dtype == torch.uint8     # one flat buffer, never host lists
        # the receive buffer is the tail of the recognizer's work buffer: own and received crops go through ONE
        # packed recognizer call
        assert out is not None and out.numel() == sum(recv_splits)
        moved.append(([int(b) for b in send_splits], [int(b) for b in recv_splits]))
        return orig(canv, send_splits, recv_splits, out=out)

    par_mod.exchange_canvases_planned = spy


def _check_one_scatter(par_mod, moved, rank):
    """Rank 0 hands several groups to rank 1 as one buffer (the balancer may send a small group of rank 1 the other
    way); what one rank sends is what the other receives."""
    assert len(moved) == 1
    send, recv = moved[0]
    assert send[rank] == 0 and recv[rank] == 0
    assert (send[1] > 0) if rank == 0 else (recv[0] > 0)
    assert par_mod.STATS["exchange_calls"] == 1
    assert par_mod.STATS["exchange_bytes_sent"] == sum(send) and par_mod.STATS["exchange_bytes_received"] == sum(recv)


def _worker_pipeline(rank, world, port, q):
    """BatchedOCR._run_groups across 2 ranks with crops that live in the shared page-locked arena (stub recognizer):
    the leaving canvases are gathered from the arena and take the planned exchange."""
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from yomitoku_b200 import parallel as par_mod
        from yomitoku_b200 import pipeline as pl
        from yomitoku_b200.config import TextRecognizerPARSeqLargeV41Config, to_config
        cfg = to_config(TextRecognizerPARSeqLargeV41Config())

        class Rec:
            _cfg = cfg
            model = _StubModel(cfg)

        ocr = pl.BatchedOCR(None, Rec(), workers=1)
        rng = np.random.default_rng(10 + rank)
        arena = pl._SharedBuf(1 << 20)
        n_groups = 7 if rank == 0 else 1
        groups, expect, offs, sizes = [], [], [], []
        for gi in range(n_groups):
            n = int(rng.integers(1, 5))
            widths = (rng.integers(9, 30, size=n) * 8).tolist()
            canv = []
            for w in widths:
                c = rng.integers(0, 256, size=(32, w, 3), dtype=np.uint8)
                off = (offs[-1] + sizes[-1] + 96 * 3) if offs else 0      # gaps: canvases need not be back to back
                arena.np[off:off + c.size] = c.reshape(-1)
                offs.append(off)
                sizes.append(c.size)
                canv.append(c)
            groups.append((widths, [max(widths)] * n, np.arange(len(offs) - n, len(offs))))
            expect.append(_fake_recognise(canv))
        moved = []
        _exchange_spy(par_mod, moved)
        calls0 = Rec.model.calls
        res = ocr._run_groups(groups, pl._FlatCrops(arena.torch, offs, sizes))
        assert Rec.model.calls - calls0 == 1          # own + received groups: one packed call
        for (ids, probs, glen), (eid, ep) in zip(res, expect):
            assert np.array_equal(ids, eid) and np.array_equal(probs, ep) and glen == 101
        _check_one_scatter(par_mod, moved, rank)
        arena.close()
        q.put((rank, "ok", None))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, "fail: " + traceback.format_exc(), None))
    finally:
        dist.destroy_process_group()


def _worker_pipeline_dev(rank, world, port, q):
    """BatchedOCR._run_groups_dev across 2 ranks: crops that exist only as records are cut "on the device" (stand-in:
    the product's crop arithmetic compiled for the host, tensors on the CPU under gloo); the groups the balancer moves
    travel as ONE flat uint8 tensor per rank through parallel.exchange_canvases_planned (all_to_all_single, split sizes agreed on by the planners over gloo) and are
    recognised straight from the receive buffer."""
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import ctypes

        from oracle import build_crop_host
        from yomitoku_b200 import data as D
        from yomitoku_b200 import models as M
        from yomitoku_b200 import parallel as par_mod
        from yomitoku_b200 import pipeline as pl
        from yomitoku_b200.config import TextRecognizerPARSeqLargeV41Config, to_config
        from yomitoku_b200.synth import synthetic_page
        cfg = to_config(TextRecognizerPARSeqLargeV41Config())
        host = ctypes.CDLL(build_crop_host.build())

        class Rec:
            _cfg = cfg
            model = _StubModel(cfg)

        def fake_extract(pages_dev, geoms, stream=None):
            sb, cb = D.layout_crop_buffers(geoms)
            scratch, canv = np.zeros(max(sb, 1), np.uint8), np.zeros(max(cb, 1), np.uint8)
            vp = ctypes.c_void_p
            host.crop_host_extract(pages_dev.ctypes.data_as(vp), pages_dev.shape[1], pages_dev.shape[2],
                                   geoms.ctypes.data_as(vp), len(geoms), scratch.ctypes.data_as(vp),
                                   canv.ctypes.data_as(vp))
            return torch.from_numpy(canv), cb          # the "device" of this test is the CPU (gloo)

        M.extract_crops_device = fake_extract
        ocr = pl.BatchedOCR(None, Rec(), workers=1, device_crops=True)
        page, quads = synthetic_page(30 + rank)
        quads = quads[:40] if rank == 0 else quads[:6]         # unbalanced: groups must move from rank 0 to rank 1
        geoms, keep = D.crop_geometry(page.shape, quads, cfg.data.img_size, True, page=0)
        ds = D.ParseqDataset(cfg, page, quads, num_workers=1, dynamic_width=True)
        order = np.argsort(geoms["cw"]).tolist()
        groups, expect = [], []
        for s in range(0, len(order), 5):
            b = order[s:s + 5]
            widths = [int(geoms["canvas_w"][i]) for i in b]
            groups.append((widths, [max(widths)] * len(b), np.asarray(b, np.int64)))
            expect.append(_fake_recognise([ds.data[i] for i in b]))
        moved = []
        _exchange_spy(par_mod, moved)
        # the three phases separately, as stream() runs them (planner / recognizer / assembly thread)
        src = pl._RecordCrops(geoms, None, np.ascontiguousarray(page)[None])
        dplan = ocr._plan_groups_dist(groups, src)
        assert isinstance(dplan, dict) and (rank != 0 or len(dplan["send"]) > 0)   # rank 0 (8 groups) hands some over
        calls0 = Rec.model.calls
        pending = ocr._run_planned(dplan, src)
        assert Rec.model.calls - calls0 == 1          # own + received groups: one packed call
        res = ocr._finish_results(pending)
        for (ids, probs, glen), (eid, ep) in zip(res, expect):
            assert np.array_equal(ids, eid) and np.array_equal(probs, ep) and glen == 101
        _check_one_scatter(par_mod, moved, rank)
        # and the one-call wrapper gives the same
        res2 = ocr._run_groups_dev(groups, geoms, np.ascontiguousarray(page)[None], None)
        for (ids, probs, glen), (eid, ep) in zip(res2, expect):
            assert np.array_equal(ids, eid) and np.array_equal(probs, ep) and glen == 101
        q.put((rank, "ok", None))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, "fail: " + traceback.format_exc(), None))
    finally:
        dist.destroy_process_group()


def test_pipeline_groups_device_crops_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker_pipeline_dev, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=30)
    for rank, status, _ in out:
        assert status == "ok", status


def _worker_pipeline_balanced(rank, world, port, q):
    """Balanced ranks: every rank derives "nothing moves" from the gathered costs and skips the scatter / gather rounds."""
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from yomitoku_b200 import parallel as par
        from yomitoku_b200 import pipeline as pl
        from yomitoku_b200.config import TextRecognizerPARSeqLargeV41Config, to_config
        from yomitoku_b200.models import pack_canvases
        cfg = to_config(TextRecognizerPARSeqLargeV41Config())

        class Rec:
            _cfg = cfg
            model = _StubModel(cfg)

        def forbidden(*a, **k):
            raise AssertionError("no exchange expected for balanced ranks")

        par.exchange_canvases_planned = forbidden
        par.exchange_results_planned = forbidden
        ocr = pl.BatchedOCR(None, Rec(), workers=1)
        rng = np.random.default_rng(5)                    # same widths on both ranks: equal costs
        groups, expect = [], []
        for gi in range(4):
            widths = (rng.integers(9, 30, size=3) * 8).tolist()
            canv = [np.random.default_rng(100 * rank + 10 * gi + j).integers(0, 256, size=(32, w, 3), dtype=np.uint8)
                    for j, w in enumerate(widths)]
            groups.append((canv, [max(widths)] * 3, np.arange(3 * gi, 3 * gi + 3)))
            expect.append(_fake_recognise(canv))
        # host canvases, packed into one buffer as prepare_pooled does
        canvases = [c for g in groups for c in g[0]]
        buf, _, offs = pack_canvases(canvases)
        groups = [([c.shape[1] for c in g[0]], g[1], g[2]) for g in groups]
        res = ocr._run_groups(groups, pl._FlatCrops(buf, offs, [c.size for c in canvases]))
        for (ids, probs, glen), (eid, ep) in zip(res, expect):
            assert np.array_equal(ids, eid) and np.array_equal(probs, ep) and glen == 101
        q.put((rank, "ok", None))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, "fail: " + traceback.format_exc(), None))
    finally:
        dist.destroy_process_group()


def test_pipeline_groups_balanced_world2_skips_exchange():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker_pipeline_balanced, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=30)
    for rank, status, _ in out:
        assert status == "ok", status


def test_pipeline_groups_arena_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker_pipeline, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=30)
    for rank, status, _ in out:
        assert status == "ok", status


def test_broadcast_and_balance_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=30)
    for rank, status, _ in out:
        assert status == "ok", status


def test_balance_groups_properties():
    from yomitoku_b200.parallel import balance_groups
    # balanced input: nothing moves
    a = balance_groups([[100, 100], [100, 100]], 2)
    assert a == [[0, 0], [1, 1]]
    # everything on rank 0 of 4: spreads out, deterministic
    costs = [[50, 40, 30, 20, 10, 10, 10, 10], [], [], []]
    a1, a2 = balance_groups(costs, 4), balance_groups(costs, 4)
    assert a1 == a2
    loads = [0] * 4
    for g, d in enumerate(a1[0]):
        loads[d] += costs[0][g]
    assert max(loads) <= 60 and sum(loads) == 180
    assert balance_groups([[5, 5]], 1) == [[0, 0]]
