"""Batched multi-page OCR: the new surface this repo adds on top of the reference's one-page-per-call modules
(SURVEY.md section 0: "there is no multi-page or multi-GPU batching in the reference").

    ocr = BatchedOCR(TextDetector(...), TextRecognizer(...), workers=16)
    results = ocr(pages)            # list of BGR pages, of any sizes -> list of OCRSchema

Per page the results are what `OCR.__call__` (reference ocr.py:51-63) returns: the pages of a batch sit back to back in
one buffer described by a page table (data.page_table), detection runs in one device launch sequence per group of pages
that share a detector input size (in chunks of `det_batch`; a same-size batch is one group), the host stages the
reference also has (contours/unclip, crop extraction: SURVEY.md R3/R4) fan out over a process pool, and ALL crops of ALL
pages go to the recognizer as one packed ragged call in which every crop keeps the padded width and mini-batch group its
own page would have given it - so per-page outputs do not depend on how many pages are batched, or of which sizes.
"""
import os
from concurrent.futures import ProcessPoolExecutor

import numpy as np

from .data import CROP_GEOM_DTYPE, ParseqDataset, crop_records, page_table
from .device_pages import as_device_pages, require_device
from .models import dbnet_post_front
from .postprocessor import DBnetPostProcessor
from .schemas import OCRSchema
from .text_recognizer import plan_mini_batches

_W = {}
# Cost of a mini-batch group for the cross-rank balancer, in encoder-token units: the encoder and the attention over the
# encoder memory scale with the group's tokens, the AR steps / refinement / head with its rows; with 101 AR steps one
# row costs about as much as 40 tokens.
ROW_COST_TOKENS = 40
TRACE = None     # set to a list to collect (stage, thread name, t0, t1) tuples (scripts/gpu_trace_e2e.py)


class _span:
    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if TRACE is not None:
            import time
            self.t0 = time.perf_counter()

    def __exit__(self, *a):
        if TRACE is not None:
            import threading
            import time
            TRACE.append((self.name, threading.current_thread().name, self.t0, time.perf_counter()))


class BatchPlan:
    """Layout and detector plan of one batch, pages in submission order.
      table / page_bytes  the pages back to back in one flat uint8 buffer (data.page_table)
      inputs              detector input size (Hn, Wn) per page
      chunks              detector calls: (Hn, Wn, page indices), grouped by input size in order of first appearance,
                          at most det_batch pages each, pages in submission order inside a group
      prob_off / prob_len float offset of each page's probability map in the map buffer (maps in chunk order, so every
                          chunk's maps are contiguous) and the buffer's length in floats
    A same-size batch is one group: its chunks, offsets and byte layout are those of the (n, H, W, 3) stack."""

    def __init__(self, shapes, input_size, det_batch):
        self.shapes = [(int(s[0]), int(s[1])) for s in shapes]
        self.table, self.page_bytes = page_table(self.shapes)
        self.inputs = [tuple(int(v) for v in input_size(h, w)) for h, w in self.shapes]
        groups = {}
        for i, hw in enumerate(self.inputs):
            groups.setdefault(hw, []).append(i)
        self.chunks = [(hn, wn, idx[s:s + det_batch]) for (hn, wn), idx in groups.items()
                       for s in range(0, len(idx), det_batch)]
        self.prob_off = [0] * len(self.shapes)
        off = 0
        for hn, wn, idx in self.chunks:
            for i in idx:
                self.prob_off[i] = off
                off += hn * wn
        self.prob_len = off

    def prob_map(self, buf, i):
        """Page i's (Hn, Wn) map in a flat map buffer (numpy array or tensor)."""
        hn, wn = self.inputs[i]
        return buf[self.prob_off[i]:self.prob_off[i] + hn * wn].reshape(hn, wn)

    def chunk_maps(self, buf, chunk):
        hn, wn, idx = chunk
        o = self.prob_off[idx[0]]
        return buf[o:o + len(idx) * hn * wn].reshape(len(idx), hn, wn)


class _SharedBuf:
    """A file in /dev/shm mapped into this process and page-locked for DMA.  Worker processes map the same file once
    (by path, `_attach`) and keep it mapped, so a job carries a tiny (path, offset, shape) descriptor instead of a
    pickled array or a per-job file-descriptor hand-over."""

    def __init__(self, nbytes):
        import mmap
        import tempfile
        import torch
        self.nbytes = int(nbytes)
        fd, self.path = tempfile.mkstemp(prefix="ytk_b200_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
        try:
            os.ftruncate(fd, self.nbytes)
            self.mm = mmap.mmap(fd, self.nbytes)
        finally:
            os.close(fd)
        self.np = np.frombuffer(self.mm, dtype=np.uint8)
        self.torch = torch.from_numpy(self.np)
        self.registered = False
        if torch.cuda.is_available():
            err = torch.cuda.cudart().cudaHostRegister(self.np.ctypes.data, self.nbytes, 0)
            if int(err) != 0:
                self.close()
                raise RuntimeError("cudaHostRegister failed: %s" % err)
            self.registered = True

    def view(self, offset, shape, dtype):
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        return self.np[offset:offset + n].view(dtype).reshape(shape)

    def desc(self, offset, shape, dtype):
        return ("shm", self.path, self.nbytes, int(offset), tuple(int(v) for v in shape), np.dtype(dtype).str)

    def close(self):
        if self.registered:
            import torch
            torch.cuda.cudart().cudaHostUnregister(self.np.ctypes.data)
            self.registered = False
        try:
            os.unlink(self.path)
        except OSError:
            pass


_ATTACHED = {}


def _attach(desc):
    """Worker side of _SharedBuf.desc: numpy view into the (cached) mapping."""
    import mmap
    _, path, nbytes, offset, shape, dtype = desc
    arr = _ATTACHED.get(path)
    if arr is None:
        if len(_ATTACHED) > 64:
            _ATTACHED.clear()
        fd = os.open(path, os.O_RDWR)
        try:
            arr = np.frombuffer(mmap.mmap(fd, nbytes), dtype=np.uint8)
        finally:
            os.close(fd)
        _ATTACHED[path] = arr
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    return arr[offset:offset + n].view(dtype).reshape(shape)


def _worker_init(post_kwargs, rec_cfg, dynamic_width, source_downscale):
    import cv2
    cv2.setNumThreads(1)
    _W["post"] = DBnetPostProcessor(**post_kwargs)
    _W["cfg"] = rec_cfg
    _W["dyn"] = dynamic_width
    _W["sd"] = source_downscale


def _host_stage(args):
    """Post-process one probability map and cut that page's crops (runs in a worker process).  With an `arena`
    (shared page-locked uint8 tensor slice owned by this page) the canvases are written back to back into it and only
    their widths travel back; canvases that do not fit are returned as arrays (`spill`)."""
    import time
    t0 = time.perf_counter()
    page, prob, quads_override = args[:3]
    arena = args[3] if len(args) > 3 else None
    geom_only = len(args) > 4 and args[4] == "geom"
    if geom_only:
        # device-side crop extraction: only the page SHAPE is needed here; the pixels never reach this process
        page = np.empty((page[1], page[2], 0), np.uint8)
    if isinstance(page, tuple):
        page = _attach(page)         # zero-copy views of the parent's shared staging buffers
    if isinstance(prob, tuple):
        prob = _attach(prob)
    if isinstance(arena, tuple):
        arena = _attach(arena)
    if quads_override is None:
        if isinstance(prob, _Runs):
            # front half done on the device (csrc/dbpost_ops.cu): only the components' row runs arrived
            quads, scores = _W["post"].boxes_from_runs(prob.runs, prob.width, prob.height, page.shape[1], page.shape[0])
        else:
            quads, scores = _W["post"]({"binary": prob[None, None]}, page.shape[:2])
    else:
        quads, scores = quads_override, [1.0] * len(quads_override)
    t1 = time.perf_counter()
    if geom_only:
        if not len(quads):
            return quads, scores, (np.zeros(0, CROP_GEOM_DTYPE), np.zeros(0, np.int64)), [], 0
        geoms, levels, _ = crop_records(page.shape, quads, _W["cfg"].data.img_size, _W["dyn"], _W["sd"])
        return quads, scores, (geoms, levels), geoms["cw"].tolist(), len(geoms), (t0, t1, time.perf_counter())
    ds = ParseqDataset(_W["cfg"], page, quads if len(quads) else [], num_workers=1, dynamic_width=_W["dyn"],
                       source_downscale=_W["sd"]) if len(quads) else None
    if ds is None:
        return quads, scores, [], [], 0
    if arena is None:
        return quads, scores, ds.data, ds.content_widths, len(ds)
    an = arena
    cap, off, widths, spill = an.shape[0], 0, [], []
    for c in ds.data:
        nb = c.size
        if not spill and off + nb <= cap:
            an[off:off + nb] = c.reshape(-1)
            off += nb
            widths.append(c.shape[1])
        else:
            spill.append(c)
    return quads, scores, _ArenaRef(widths, spill), ds.content_widths, len(ds), \
        (t0, t1, time.perf_counter())


class _Runs:
    """A page's probability map reduced on the device to the row runs of its components (models.dbnet_post_front)."""

    def __init__(self, runs, height, width):
        self.runs, self.height, self.width = runs, height, width


class _ArenaRef:
    """What a worker sends back instead of canvases: the widths of the crops it wrote into its arena slice."""

    def __init__(self, widths, spill):
        self.widths, self.spill = widths, spill


class _PageCrops:
    """Crops of one page living in the shared arena at absolute byte offsets `offs` (list-like over canvases)."""

    def __init__(self, arena_np, base, widths, height):
        self.arena_np = arena_np
        self.height = height
        self.widths = list(widths)
        sizes = np.asarray(self.widths, dtype=np.int64) * (3 * height)
        self.offs = base + np.cumsum(sizes) - sizes

    def __len__(self):
        return len(self.widths)

    def __getitem__(self, i):
        w = self.widths[i]
        o = int(self.offs[i])
        return self.arena_np[o:o + self.height * w * 3].reshape(self.height, w, 3)


class _PageGeoms:
    """Crops of one page that exist only as ytk_crop_geom records (device-side extraction): `widths` are the canvas
    widths the crops will have, `base` the index of the page's first record in the step's record array."""

    def __init__(self, geoms, base, levels=None):
        self.geoms = geoms
        self.levels = levels if levels is not None else np.zeros(len(geoms), np.int64)   # source_downscale pyramid level
        self.base = base
        self.widths = geoms["canvas_w"].tolist()

    def __len__(self):
        return len(self.widths)


# Where the pixels of a packed recognizer call come from.  Groups of crops are (widths, padded widths, crop indices
# into a source); a source gives, for crop indices `idx` in packing order, the byte layout of their canvases
# (`layout(idx) -> (bytes, offsets)`, host only, so a chunk is planned ahead of the GPU) and a flat buffer holding them
# there (`fill(idx, stream)`).  `pack_layout` / `pack` do the same with the canvases back to back on the compute
# device: what the crop scatter sends.

class _FlatCrops:
    """Canvases already sitting in one flat uint8 tensor at byte offsets `offs` (`nbytes` each): the page-locked crop
    arena, a batch's host canvases packed by `prepare_pooled`, or the receive buffer of the crop scatter.  A chunk is
    read in place: the recognizer gets the span from its first to its last byte."""

    def __init__(self, buf, offs, nbytes):
        self.buf = buf
        self.offs = np.asarray(offs, np.int64)
        self.nbytes = np.asarray(nbytes, np.int64)

    @property
    def on_device(self):
        return 1 if self.buf.is_cuda else 0

    def _span(self, idx):
        o = self.offs[idx]
        return int(o.min()), int((o + self.nbytes[idx]).max())

    def layout(self, idx):
        lo, hi = self._span(idx)
        return hi - lo, self.offs[idx] - lo

    def fill(self, idx, stream=None):
        lo, hi = self._span(idx)
        return self.buf[lo:hi]

    def pack_layout(self, idx):
        size = self.nbytes[idx]
        return int(size.sum()), np.cumsum(size) - size

    def pack(self, idx, stream=None):
        """Gathers the canvases on the host and uploads them once (the buffer is a host one here)."""
        import torch
        from . import parallel as par
        host = self.buf.numpy()
        flat = np.concatenate([host[o:o + n] for o, n in zip(self.offs[idx].tolist(), self.nbytes[idx].tolist())])
        return torch.from_numpy(flat).to(par._dev(), non_blocking=True)


class _RecordCrops:
    """Crops that exist only as ytk_crop_geom records (+ source_downscale levels) of the pages in HBM: the canvases of
    a chunk are cut on the device, one extraction per pyramid level (models.extract_crops_pyramid)."""
    on_device = 1

    def __init__(self, geoms, levels=None, pages_dev=None):
        self.geoms = geoms
        self.levels = levels if levels is not None else np.zeros(len(geoms), np.int64)
        # pyramid level -> pages; the levels above 0 are built on first use
        self.pages = pages_dev if isinstance(pages_dev, dict) or pages_dev is None else {0: pages_dev}

    def layout(self, idx):
        from .models import plan_crop_offsets
        return plan_crop_offsets(self.geoms[idx], self.levels[idx])

    def fill(self, idx, stream=None):
        from . import models
        with _span("recognize.crops_device"):
            return models.extract_crops_pyramid(self.pages, self.geoms[idx], self.levels[idx], stream)[0]

    pack_layout, pack = layout, fill


def _multi_rank():
    import torch.distributed as dist
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


class BatchedOCR:
    def __init__(self, detector, recognizer, workers=None, det_batch=8, max_tokens=1_000_000, device_crops=None):
        self.detector = detector
        self.recognizer = recognizer
        # device-side crop extraction (csrc/crop_ops.cu): pages stay in HBM after detection, the host stage only
        # produces quads + per-crop records, the canvases are cut on the GPU (bit-exact with the OpenCV path; with
        # source_downscale the pyramid levels are built there too)
        if device_crops is None:
            # default ON (round 2): the host stage then only post-processes probability maps; YTK_DEVICE_CROPS=0 selects
            # the OpenCV host path (the reference's way) for A/B runs
            import torch
            device_crops = os.environ.get("YTK_DEVICE_CROPS", "1") != "0" and torch.cuda.is_available()
        self.device_crops = bool(device_crops)
        self.det_batch = det_batch
        self.max_tokens = max_tokens
        self.workers = workers if workers is not None else max(1, min(32, (os.cpu_count() or 2) - 2))
        self._pool = None
        self._prob_ring = {}
        self._slot = 0              # ring slot (pages + probability maps + crop arena) of the batch being submitted
        self._ring = 3              # number of ring slots
        self._slot_busy = {}        # slot -> (host-stage futures, handle) of the batch that last used it
        self._last_shared = None
        self.crop_cap = 8 << 20     # arena bytes per page; doubled when a page spills
        self.post_front_pages = 0   # pages post-processed from device runs / through the downloaded map (holes)
        self.post_host_pages = 0
        self.post_d2h_bytes = 0     # bytes the detector stage brought back (runs + meta, or whole maps)

    # ------------------------------------------------------------------------------------------ host pool
    def _get_pool(self):
        if self._pool is None and self.workers > 1:
            import multiprocessing as mp
            r = self.recognizer
            # forkserver: workers descend from a clean server process, never from this CUDA-initialised,
            # multi-threaded one (forking that is undefined behaviour for the CUDA runtime and OpenCV's thread pool)
            import sys
            mf = getattr(sys.modules.get("__main__"), "__file__", None)
            if mf is None or os.path.exists(mf):
                ctx = mp.get_context("forkserver")
                try:
                    ctx.set_forkserver_preload(["yomitoku_b200.pipeline"])
                except Exception:
                    pass
            else:  # `python -` / `python -c`: the spawn machinery cannot re-import __main__
                ctx = mp.get_context("fork")
            self._pool = ProcessPoolExecutor(
                max_workers=self.workers, mp_context=ctx, initializer=_worker_init,
                initargs=(dict(self.detector._cfg.post_process), r._cfg, r.dynamic_width, r.source_downscale))
        return self._pool

    def close(self):
        if self._pool is not None:
            self._pool.shutdown(wait=True, cancel_futures=True)
            self._pool = None
        for ring in self._prob_ring.values():
            for buf in ring.values():
                buf.close()
        self._prob_ring = {}
        self._slot_busy = {}

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _host_map(self, jobs):
        pool = self._get_pool()
        if pool is None:
            r = self.recognizer
            _worker_init(dict(self.detector._cfg.post_process), r._cfg, r.dynamic_width, r.source_downscale)
            return [_host_stage(j) for j in jobs]
        return list(pool.map(_host_stage, jobs, chunksize=1))

    # ------------------------------------------------------------------------------------------ stages
    def _shared(self, kind, nbytes):
        """Shared + page-locked staging buffer of the current ring slot (pages, probability maps or crop arena).  One
        buffer per (kind, slot), sized by capacity: it is reused while it is large enough and replaced by a larger one
        otherwise (the slot's previous batch is finished by then, see `submit`), so batches with different byte totals
        do not accumulate /dev/shm files and page-locked registrations."""
        ring = self._prob_ring.setdefault(kind, {})
        buf = ring.get(self._slot)
        if buf is None or buf.nbytes < nbytes:
            if buf is not None:
                buf.close()
            buf = ring[self._slot] = _SharedBuf(max(int(nbytes), 1))
        return buf

    def _stage(self, pages, shared):
        """Host staging of a batch: (stage flat u8 tensor holding the pages back to back, out flat f32 tensor for the
        probability maps, BatchPlan).  For same-size pages the stage is byte for byte their (n, H, W, 3) stack.  With
        `shared` both live in the shared page-locked ring - the H2D/D2H copies are plain DMAs and the workers read both
        without a copy; `self._last_shared` then holds the two buffers."""
        import torch
        plan = BatchPlan([p.shape[:2] for p in pages], self.detector.model.input_size, self.det_batch)
        out, ob = self._prob_out(plan, shared)
        if shared:
            pb = self._shared("pages", plan.page_bytes)
            with _span("detect.stage_pages"):
                for (h, w), off, p in zip(plan.shapes, plan.table["page_off"], pages):
                    np.copyto(pb.view(int(off), (h, w, 3), np.uint8), p)
            stage = pb.torch[:plan.page_bytes]
            self._last_shared = (pb, ob)
        else:
            stage = torch.from_numpy(np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in pages]))
        return stage, out, plan

    def _prob_out(self, plan, shared):
        """The host buffer of a batch's probability maps (flat f32 tensor) and, with `shared`, the ring buffer holding it
        (`self._last_shared` is then (pages buffer or None, that buffer))."""
        import torch
        self._last_shared = None
        if shared:
            ob = self._shared("prob", plan.prob_len * 4)
            self._last_shared = (None, ob)
            return ob.torch[:plan.prob_len * 4].view(torch.float32), ob
        return torch.empty(plan.prob_len, dtype=torch.float32), None

    def _detect_chunk(self, stage, plan, chunk, maps, stream=None):
        """One detector call: the chunk's pages of the flat stage (host or device) -> maps (n, Hn, Wn)."""
        self.detector.model.detect_pages_table(stage, plan.table[chunk[2]], out=maps, stream=stream)

    def detect_prob(self, pages, shared=False, stream=None):
        """Device stage 1: probability maps float32 on the host, per page in submission order (an (n, Hn, Wn) array when
        all pages share the detector input size)."""
        stage, out, plan = self._stage(pages, shared)
        for ch in plan.chunks:
            self._detect_chunk(stage, plan, ch, plan.chunk_maps(out, ch), stream)
        maps = [plan.prob_map(out.numpy(), i) for i in range(len(pages))]
        return np.stack(maps) if len(set(plan.inputs)) == 1 else maps

    def _group_tokens(self, g):
        """Encoder tokens of one group (widths, padded widths, ...): what the chunking counts against max_tokens."""
        cfg = self.recognizer._cfg
        ph, pw = cfg.encoder.patch_size
        return (cfg.data.img_size[0] // ph) * (int(np.sum(g[1])) // pw)

    def _plan_chunks(self, groups, src):
        """Host-only plan of the packed recognizer calls for `groups` (crop indices into `src`): <= max_tokens chunks
        ending on group boundaries, each with its crop indices, canvas bytes and ytk_crop descriptors.
        `BatchedOCR.stream` runs this for batch i + 1 in its own thread while batch i is on the GPU."""
        from .models import crop_descriptors
        gtok = [self._group_tokens(g) for g in groups]
        chunks, start = [], 0
        while start < len(groups):
            end, tok = start, 0
            while end < len(groups) and not (end > start and tok + gtok[end] > self.max_tokens):
                tok += gtok[end]
                end += 1
            sel = groups[start:end]
            sizes = [len(g[1]) for g in sel]
            idx = np.concatenate([np.asarray(g[2], np.int64) for g in sel])
            total, pix_off = src.layout(idx)
            descs = crop_descriptors(self.recognizer._cfg, pix_off, np.concatenate([g[0] for g in sel]),
                                     np.concatenate([g[1] for g in sel]), np.repeat(np.arange(end - start), sizes))
            chunks.append({"idx": idx, "total": total, "descs": descs, "sizes": sizes})
            start = end
        return chunks

    def _run_chunks(self, chunks, src, stream=None):
        """One packed recognizer call per planned chunk, its pixels taken from `src`.  Returns per group
        (ids, probs, group_len)."""
        model = self.recognizer.model
        out = []
        for ch in chunks:
            canv = src.fill(ch["idx"], stream)
            with _span("recognize.device"):
                ids, probs, glen = model.run_packed_ptr(canv.data_ptr(), src.on_device, ch["total"], ch["descs"],
                                                        len(ch["descs"]), len(ch["sizes"]), stream=stream)
            del canv
            off = 0
            for k, m in enumerate(ch["sizes"]):
                out.append((ids[off:off + m], probs[off:off + m], int(glen[k])))
                off += m
        return out

    def _plan_groups_dev(self, groups, geoms, levels=None):
        """`_plan_chunks` for groups whose crops exist only as records; `_run_groups_dev` takes the result as `plan`."""
        return self._plan_chunks(groups, _RecordCrops(geoms, levels))

    def _run_groups_dev(self, groups, geoms, pages_dev, stream=None, levels=None, plan=None):
        """`_run_groups` for groups whose crops exist only as records: groups = (widths, padded widths, record indices
        into `geoms`), the canvases are cut on the device and never touch the host.  `plan`: `_plan_groups_dev(groups,
        geoms, levels)` on one rank, prepared ahead of time."""
        return self._run_groups(groups, _RecordCrops(geoms, levels, pages_dev), stream, plan)

    def _run_groups(self, groups, src, stream=None, plan=None):
        """Recognise groups whose pixels come from `src`; results come back in `groups` order.  One rank: the chunks of
        `_plan_chunks`.  With torch.distributed the call has three phases that `stream()` runs in three different
        threads - `_plan_groups_dist` (host: costs, balancing and layouts over a gloo group), `_run_planned` (device:
        the leaving groups are packed into one buffer ordered by destination and travel GPU-to-GPU with ONE
        all_to_all_single over NCCL / NVLink; own and received groups are recognised in one packed call) and
        `_finish_results` (host: ids / probabilities of groups recognised elsewhere come back over a second gloo
        group).  This runs the three back to back."""
        if plan is None:
            plan = self._plan_groups_dist(groups, src) if _multi_rank() else self._plan_chunks(groups, src)
        return self._finish_results(self._run_planned(plan, src, stream))

    def _plan_groups_dist(self, groups, src):
        """Phase 1 (host only; collectives on the "plan" gloo group): every rank learns all group costs, derives the
        same assignment, and tells the others what it will send - after this no rank needs another control message
        before its device work.  When nothing moves this is the single-rank chunk plan."""
        import torch.distributed as dist
        from . import parallel as par
        world, rank = dist.get_world_size(), dist.get_rank()
        costs = [self._group_tokens(g) + ROW_COST_TOKENS * len(g[1]) for g in groups]
        assign_all = par.balance_groups(par.all_gather_objects(costs, "plan"), world)
        if all(dst == r for r, row in enumerate(assign_all) for dst in row):
            return self._plan_chunks(groups, src)
        assign = assign_all[rank]
        height = self.recognizer._cfg.data.img_size[0]

        def packed(ks):
            """Crop indices of groups ks and the layout `src.pack` gives them: (idx, bytes, rows (k, w, wp, offs))."""
            idx = np.concatenate([groups[k][2] for k in ks])
            total, offs = src.pack_layout(idx)
            rows, j = [], 0
            for k in ks:
                m = len(groups[k][1])
                rows.append((k, np.asarray(groups[k][0], np.int64), np.asarray(groups[k][1], np.int64), offs[j:j + m]))
                j += m
            return idx, total, rows

        send, outgoing, send_splits = [], {}, [0] * world
        for dst in range(world):
            ks = [k for k in range(len(groups)) if assign[k] == dst and dst != rank]
            if ks:       # ascending destination = the order of the split sizes
                idx, send_splits[dst], rows = packed(ks)
                send.append((idx, send_splits[dst]))
                outgoing[dst] = {"bytes": send_splits[dst], "groups": rows}
        everyone = par.all_gather_objects(outgoing, "plan")
        # ONE packed recognizer call for own + received groups: a single work buffer [own canvases | received canvases]
        # (two calls would run the 101-step decode loop twice, and its cost is mostly per step, not per row)
        mine = [k for k in range(len(groups)) if assign[k] == rank]
        mine_idx, mine_total, rows = packed(mine) if mine else (None, 0, [])
        work = [(w, wp, offs) for _, w, wp, offs in rows]
        owner = [(rank, k) for k in mine]
        recv_splits, base = [0] * world, mine_total
        for src_rank in range(world):
            d = everyone[src_rank].get(rank) if src_rank != rank else None
            if d is None:
                continue
            recv_splits[src_rank] = int(d["bytes"])
            work += [(w, wp, base + offs) for _, w, wp, offs in d["groups"]]
            owner += [(src_rank, int(gid)) for gid, _, _, _ in d["groups"]]
            base += int(d["bytes"])
        # the work buffer's canvases, numbered in group order: the groups become (widths, padded widths, indices)
        offs = np.concatenate([g[2] for g in work]) if work else np.zeros(0, np.int64)
        widths = np.concatenate([g[0] for g in work]) if work else np.zeros(0, np.int64)
        starts = np.cumsum([0] + [len(g[0]) for g in work])
        work = [(w, wp, np.arange(starts[i], starts[i + 1])) for i, (w, wp, _) in enumerate(work)]
        work_src = _FlatCrops(None, offs, widths * (3 * height))
        # phase 3 is planned here too: a group's result is m rows of (S int32 ids, S float32 probabilities) + its int32
        # decode length, so every rank knows the byte counts of the result exchange before anything runs
        S = int(self.recognizer.model.max_label_length) + 1
        back_splits, expect_splits, expect = [0] * world, [0] * world, {}
        for (src_rank, _), (w, _, _) in zip(owner, work):
            if src_rank != rank:
                back_splits[src_rank] += len(w) * S * 8 + 4
        for k in range(len(groups)):
            if assign[k] != rank:
                expect.setdefault(assign[k], []).append((k, len(groups[k][1])))
                expect_splits[assign[k]] += len(groups[k][1]) * S * 8 + 4
        return {"mine_idx": mine_idx, "mine_total": mine_total, "send": send, "send_splits": send_splits,
                "recv_splits": recv_splits, "work_offs": work_src.offs, "work_bytes": work_src.nbytes,
                "chunks": self._plan_chunks(work, work_src), "owner": owner, "n_groups": len(groups),
                "results": {"S": S, "back_splits": back_splits, "expect_splits": expect_splits, "expect": expect}}

    def _run_planned(self, plan, src, stream=None):
        """Phase 2 (device).  plan: a chunk list (one rank, or nothing moves) -> the group results; a
        `_plan_groups_dist` dict -> a `_PendingResults` (own groups done, results of foreign groups to hand back)."""
        if not isinstance(plan, dict):
            return self._run_chunks(plan, src, stream)
        import contextlib

        import torch
        import torch.distributed as dist
        from . import models
        from . import parallel as par
        device = par._dev()
        with torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext():
            parts = [(src.pack(idx, stream), total) for idx, total in plan["send"]]
            if parts:
                canv = models.concat_device_buffers(parts, stream)
                if len(parts) == 1:
                    canv = canv[: parts[0][1]]
            else:
                canv = torch.empty(0, dtype=torch.uint8, device=device)
            mine_total = plan["mine_total"]
            work = torch.empty(mine_total + int(sum(plan["recv_splits"])), dtype=torch.uint8, device=device)
            if mine_total:
                own = src.pack(plan["mine_idx"], stream)
                work[:mine_total].copy_(own[:mine_total], non_blocking=True)
                del own
            par.exchange_canvases_planned(canv, plan["send_splits"], plan["recv_splits"], out=work[mine_total:])
        res = self._run_chunks(plan["chunks"], _FlatCrops(work, plan["work_offs"], plan["work_bytes"]), stream)
        rank = dist.get_rank()
        out, back = [None] * plan["n_groups"], []
        for (src_rank, gid), r in zip(plan["owner"], res):
            if src_rank == rank:
                out[gid] = r
            else:
                back.append((src_rank, gid) + r)
        return _PendingResults(out, back, plan["results"])

    def _finish_results(self, pending):
        """Phase 3 (host; collectives on the "results" gloo group): results of the groups this rank sent away."""
        if isinstance(pending, list):
            return pending
        from . import parallel as par
        rp = pending.plan
        S = rp["S"]
        parts = []
        for src, gid, ids, probs, glen in pending.back:           # grouped by source rank, ascending (the plan's order)
            if ids.shape[1] != S:
                raise RuntimeError("result exchange: rows of %d positions, the plan says %d" % (ids.shape[1], S))
            parts += [np.ascontiguousarray(ids, np.int32).reshape(-1).view(np.uint8),
                      np.ascontiguousarray(probs, np.float32).reshape(-1).view(np.uint8),
                      np.array([glen], np.int32).view(np.uint8)]
        send = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
        recv = par.exchange_results_planned(send, rp["back_splits"], rp["expect_splits"])
        off = 0
        for dst in sorted(rp["expect"]):
            for k, m in rp["expect"][dst]:
                nb = m * S * 4
                ids = recv[off:off + nb].view(np.int32).reshape(m, S)
                probs = recv[off + nb:off + 2 * nb].view(np.float32).reshape(m, S)
                glen = int(recv[off + 2 * nb:off + 2 * nb + 4].view(np.int32)[0])
                pending.out[k] = (ids, probs, glen)
                off += 2 * nb + 4
        missing = [k for k, r in enumerate(pending.out) if r is None]
        if missing:
            raise RuntimeError("crop scatter: no result came back for groups %s" % missing[:8])
        return pending.out

    def _crop_source(self, per_page, arena, pages_dev):
        """The pixel source of a batch's crops: records cut on the device, the arena the workers wrote, or - for host
        canvas lists (no worker pool, or a page whose arena slice spilled) - one page-locked buffer packed here."""
        pages = [p[0] for p in per_page]
        if pages_dev is not None and all(isinstance(p, _PageGeoms) for p in pages):
            if not pages:
                return _RecordCrops(np.zeros(0, CROP_GEOM_DTYPE), None, pages_dev)
            return _RecordCrops(np.concatenate([p.geoms for p in pages]), np.concatenate([p.levels for p in pages]),
                                pages_dev)
        height = self.recognizer._cfg.data.img_size[0]
        if arena is not None and all(isinstance(p, _PageCrops) for p in pages):
            widths = np.asarray([w for p in pages for w in p.widths], np.int64)
            offs = np.concatenate([p.offs for p in pages]) if pages else np.zeros(0, np.int64)
            return _FlatCrops(arena.torch, offs, widths * (3 * height))
        from .models import pack_canvases
        canvases = [c for p in pages for c in p]
        buf, _, offs = pack_canvases(canvases)
        return _FlatCrops(buf, offs, [c.size for c in canvases])

    def prepare_pooled(self, per_page, arena=None, pages_dev=None):
        """Host-only half of `recognize_pooled`: the reference grouping of every page (bucketing order, mini-batch plan,
        padded widths) flattened into the group list of the batch, the batch's pixel source and the plan of its packed
        recognizer calls (over all ranks with torch.distributed).  No device call, so it can run ahead of the GPU."""
        rec = self.recognizer
        cfg = rec._cfg
        groups, owner, orders, base = [], [], [], 0
        for pi, (canv, cw, n_quads) in enumerate(per_page):
            order = None
            if rec.batch_bucketing and len(canv) == n_quads and len(canv) > 1:
                order = np.argsort(cw).tolist()
            widths = canv.widths if isinstance(canv, (_PageCrops, _PageGeoms)) else [c.shape[1] for c in canv]
            plan = plan_mini_batches(widths, order, rec.dynamic_width, cfg.data.batch_size,
                                     getattr(cfg.data, "width_budget", None),
                                     getattr(cfg.data, "max_batch_size", None))
            padded, _ = rec._collate_widths(widths, plan)
            for b in plan:
                groups.append(([widths[i] for i in b], [padded[i] for i in b], base + np.asarray(b, np.int64)))
                owner.append(pi)
            orders.append(order)
            base += len(widths)
        src = self._crop_source(per_page, arena, pages_dev)
        plan = self._plan_groups_dist(groups, src) if _multi_rank() else self._plan_chunks(groups, src)
        return {"groups": groups, "owner": owner, "orders": orders, "n_pages": len(per_page), "src": src,
                "plan": plan}

    def run_prepared(self, prep, stream=None, arena=None, pages_dev=None, finish=True):
        """Device half of `recognize_pooled` (`arena` / `pages_dev`: those given to `prepare_pooled`, whose source
        holds them).  finish=True: returns per page (ids, probs, order) with rows in the page's *plan* order, exactly
        like TextRecognizer._run_plan.  finish=False (`stream()` with several ranks): returns the raw group results,
        possibly pending on other ranks - `finish_prepared` completes them in another thread."""
        raw = self._run_planned(prep["plan"], prep["src"], stream)
        return self.finish_prepared(prep, raw) if finish else raw

    def finish_prepared(self, prep, raw):
        pages = self._gather_pages(self._finish_results(raw), prep["owner"], prep["n_pages"])
        return [(ids, probs, order) for (ids, probs), order in zip(pages, prep["orders"])]

    def _gather_pages(self, res, owner, n_pages):
        """Group results + the page of every group -> per page (ids, probs), rows in plan order, the positions a
        `refine_iters == 0` model never produced filled like the host path does."""
        rec = self.recognizer
        S = rec._cfg.max_label_length + 1
        out = []
        for pi in range(n_pages):
            mine = [r for r, o in zip(res, owner) if o == pi]
            if not mine:
                out.append((np.zeros((0, S), np.int32), np.zeros((0, S), np.float32)))
                continue
            ids = np.concatenate([m[0] for m in mine])
            probs = np.concatenate([m[1] for m in mine])
            rec._eos_tail(ids, probs, np.repeat([m[2] for m in mine], [len(m[0]) for m in mine]))
            out.append((ids, probs))
        return out

    def recognize_pooled(self, per_page, stream=None, arena=None, pages_dev=None):
        """Device stage 2: per_page = list of (canvases, content_widths, n_quads); canvases is a list of arrays, a
        `_PageCrops` view of `arena` or a `_PageGeoms` (records only, cut on the device)."""
        return self.run_prepared(self.prepare_pooled(per_page, arena, pages_dev), stream, arena, pages_dev)

    # ------------------------------------------------------------------------------------------ whole path
    def submit(self, pages, prob_override=None, quads_override=None, stream=None, wait_recognized=False):
        """Stage 1 (device, synchronous: a few ms per page) + hand the host stage to the worker pool.  Returns a handle
        for `collect`.  Submitting batch i+1 before collecting batch i overlaps its host stage (contours, unclip, crop
        extraction) with the recognition of batch i on the GPU."""
        pool = self._get_pool()
        # staging ring (pages, probability maps, crop arena): a slot is reused only after the host stage of its
        # previous batch has finished AND that batch has been recognised (the recognizer's H2D copy reads the arena).
        # stream() waits for that; with manual submit()/collect() an unrecognised batch keeps its slot and the ring grows
        self._slot = (self._slot + 1) % self._ring
        with _span("submit.wait_slot"):
            prev = self._slot_busy.pop(self._slot, None)
            if prev is not None:
                for f in prev[0]:
                    f.result()
                if not prev[1].done.is_set():
                    if wait_recognized:
                        prev[1].done.wait()
                    else:
                        self._slot_busy[self._slot] = prev
                        self._slot = self._ring
                        self._ring += 1
        dp = as_device_pages(pages)
        if dp is not None:
            # pages already in HBM: no staging copy and no upload; the packed buffer is what the detector and the crop
            # kernels read, so the host stage sees page shapes only (the device-crops jobs)
            require_device(dp, self.detector.model.cuda_device(), "BatchedOCR")
            dp.ready(stream)
            plan = BatchPlan(dp.shapes, self.detector.model.input_size, self.det_batch)
            stage, pages_dev = None, dp.buf
            out, _ = self._prob_out(plan, shared=pool is not None)
        else:
            stage, out, plan = self._stage(pages, shared=pool is not None)
            pages_dev = None
        n = len(plan.shapes)
        prob = out.numpy()
        sh = self._last_shared if pool is not None else None
        arena, cap = None, self.crop_cap
        if pages_dev is None and (self.device_crops or getattr(self.recognizer, "rec_orientation_fallback", False)):
            # (the orientation fallback's second look is implemented on the device-crops path only: its crops are the
            # same records with one bit set, no rectified images have to come back from the workers)
            # the pages stay in HBM for the crop kernels of this batch; the tensor belongs to the handle (no ring slot
            # to guard) and the detector reads the same copy
            with _span("submit.pages_h2d"):
                pages_dev = self._upload_pages(stage, stream)
        if sh is not None:
            pb, ob = sh
            if pages_dev is None:
                arena = self._shared("crops", n * cap)
        if pool is None:
            r = self.recognizer
            _worker_init(dict(self.detector._cfg.post_process), r._cfg, r.dynamic_width, r.source_downscale)
        # device front half of the post-processing: the maps stay in HBM, a page's row runs (~100 KB) come back instead
        # of its 7.6 MB map; a page with a hole in a component (or too many runs) downloads its map and takes OpenCV
        dev_post = (pages_dev is not None and quads_override is None and getattr(self.detector, "device_post", False))
        if dev_post:
            import torch
            out_dev = torch.empty(out.shape, dtype=torch.float32, device=pages_dev.device)
        futs = [None] * n       # submission order, whatever order the detector groups run in
        # detection per chunk of pages that share a detector input size (plan.chunks); a chunk's host jobs start while
        # the next chunk is on the device
        for ch in plan.chunks:
            hn, wn, idx = ch
            maps = plan.chunk_maps(out_dev if dev_post else out, ch)
            with _span("submit.detect"):
                self._detect_chunk(stage if pages_dev is None else pages_dev, plan, ch, maps, stream)
            runs = [None] * len(idx)
            if dev_post:
                with _span("submit.post_front"):
                    if prob_override is not None:      # benchmarks with random detector weights: replace the maps
                        for j, i in enumerate(idx):
                            self._override_prob(maps[j], prob_override[i], stream)
                    runs, _ = dbnet_post_front(maps, self.detector.post_processor.thresh, stream)
                    self.post_front_pages += sum(r is not None for r in runs)
                    self.post_host_pages += sum(r is None for r in runs)
                    self.post_d2h_bytes += 16 * len(idx) + sum(r.nbytes for r in runs if r is not None)
                    for j, i in enumerate(idx):
                        if runs[j] is None:
                            plan.prob_map(out, i).copy_(maps[j])      # pageable or pinned host map; synchronous
                            self.post_d2h_bytes += hn * wn * 4
            else:
                self.post_d2h_bytes += maps.numel() * 4
            for j, i in enumerate(idx):
                h0, w0 = plan.shapes[i]
                pm = plan.prob_map(prob, i)
                qo = None if quads_override is None else quads_override[i]
                if runs[j] is not None:
                    job = (("shape", h0, w0), _Runs(runs[j], hn, wn), qo, None, "geom")
                elif sh is None:
                    pm_in = pm if (prob_override is None or dev_post) else prob_override[i]
                    job = (pages[i], pm_in, qo) if pages_dev is None else (("shape", h0, w0), pm_in, qo, None, "geom")
                elif pages_dev is not None:
                    if prob_override is not None and not dev_post:
                        np.copyto(pm, prob_override[i])
                    job = (("shape", h0, w0), ob.desc(plan.prob_off[i] * 4, pm.shape, np.float32), qo, None, "geom")
                else:
                    if prob_override is not None:   # benchmarks with random detector weights: overwrite the D2H result
                        np.copyto(pm, prob_override[i])
                    # descriptors only: the workers map the three buffers themselves
                    job = (pb.desc(int(plan.table["page_off"][i]), (h0, w0, 3), np.uint8),
                           ob.desc(plan.prob_off[i] * 4, pm.shape, np.float32), qo,
                           arena.desc(i * cap, (cap,), np.uint8))
                futs[i] = _Done(_host_stage(job)) if pool is None else pool.submit(_host_stage, job)
        if pages_dev is not None:
            pages_dev = (pages_dev, plan.table)     # what the crop kernels read
        if pool is None:
            return _Handle(futs, None, 0, pages_dev)
        handle = _Handle(futs, arena, cap, pages_dev)
        self._slot_busy[self._slot] = (futs, handle)
        return handle

    @staticmethod
    def _override_prob(dst, src, stream=None):
        """dst (Hn, Wn) fp32 cuda <- src (numpy array or tensor on either side), asynchronous on `stream`."""
        import torch
        t = src if isinstance(src, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(src, dtype=np.float32))
        if stream is not None:
            with torch.cuda.stream(stream):
                dst.copy_(t, non_blocking=True)
        else:
            dst.copy_(t, non_blocking=True)

    def _upload_pages(self, stage, stream=None):
        """Flat uint8 staging tensor (the pages back to back) -> the same bytes in HBM of the detector's device (asynchronous on
        `stream`)."""
        import torch
        dev = self.detector.model.cuda_device() if hasattr(self.detector.model, "cuda_device") else "cuda"
        if stream is not None:
            with torch.cuda.stream(stream):
                return stage.to(dev, non_blocking=True)
        return stage.to(dev, non_blocking=True)

    def collect(self, handle, stream=None):
        """Waits for the host stage of a submitted batch, recognises all its crops in one packed device call and
        assembles per-page OCRSchema results."""
        return self._assemble(*self._recognize_handle(handle, stream))

    def _recognize_handle(self, handle, stream=None):
        try:
            return self._run_handle(handle, self._prepare_handle(handle), stream)
        finally:
            handle.done.set()       # the staging slot of this batch may be reused

    def _prepare_handle(self, handle):
        """Waits for the host stage of a batch and plans its recognizer call (host only; `stream()` runs this one batch
        ahead of the GPU in its own thread)."""
        with _span("collect.wait_host"):
            host = [f.result() for f in handle.futures]
        arena = handle.arena
        if handle.pages_dev is not None:
            fixed, base = [], 0
            for i, h in enumerate(host):
                g, lv = h[2]
                g["page"] = i
                if TRACE is not None and len(h) > 5:
                    TRACE.append(("worker.post", "worker", h[5][0], h[5][1]))
                    TRACE.append(("worker.geometry", "worker", h[5][1], h[5][2]))
                fixed.append((h[0], h[1], _PageGeoms(g, base, lv), h[3], h[4]))
                base += len(g)
            host = fixed
        elif arena is not None:
            an = arena.np
            fixed = []
            for i, h in enumerate(host):
                ref = h[2]
                if isinstance(ref, _ArenaRef):
                    crops = _PageCrops(an, i * handle.cap, ref.widths, self.recognizer._cfg.data.img_size[0])
                    if ref.spill:       # arena slice too small for this page: generic path now, larger slices next time
                        crops = [crops[k] for k in range(len(crops))] + list(ref.spill)
                        self.crop_cap = max(self.crop_cap, 2 * handle.cap)
                        arena = None
                    if TRACE is not None and len(h) > 5:
                        TRACE.append(("worker.post", "worker", h[5][0], h[5][1]))
                        TRACE.append(("worker.crops", "worker", h[5][1], h[5][2]))
                    h = (h[0], h[1], crops, h[3], h[4])
                fixed.append(h)
            host = fixed
        rec_in = [(h[2], h[3], len(h[0])) for h in host]
        with _span("collect.prepare"):
            prep = self.prepare_pooled(rec_in, arena=arena, pages_dev=handle.pages_dev)
        return host, prep, arena

    def _run_handle(self, handle, prepared, stream=None, defer=False):
        """defer=True (`stream()`): the device work of this batch only; what other ranks still owe is collected by
        `_finish_handle` in the assembly thread, so the GPU goes straight into the next batch."""
        host, prep, arena = prepared
        fallback = handle.pages_dev is not None and getattr(self.recognizer, "rec_orientation_fallback", False)
        with _span("collect.recognize"):
            if defer and not fallback:
                return host, (prep, self.run_prepared(prep, stream, arena=arena, pages_dev=handle.pages_dev, finish=False))
            rec_out = self.run_prepared(prep, stream, arena=arena, pages_dev=handle.pages_dev)
            if fallback:
                self._orientation_fallback_dev([h[2] for h in host], rec_out, handle.pages_dev, stream)
        return host, rec_out

    def _finish_handle(self, item):
        host, rec = item
        if isinstance(rec, tuple):
            rec = self.finish_prepared(*rec)
        return host, rec

    def _orientation_fallback_dev(self, page_geoms, rec_out, pages_dev, stream=None):
        """The recognizer's optional 180-degree second look (reference text_recognizer.py:319-350) for a whole batch:
        per page, the crops whose score is below the threshold - in detection order, in chunks of `batch_size` like
        TextRecognizer._apply_orientation_fallback - are cut again on the GPU rotated by 180 degrees on the fixed-width
        canvas (record bit `rot & 2`); a row of (ids, probs) is replaced when the second look scores higher and reaches
        the threshold.  rec_out rows are in plan order and are updated in place."""
        rec = self.recognizer
        cfg = rec._cfg
        thresh = rec.rec_orientation_fallback_thresh
        bs = cfg.data.batch_size
        groups, owner, retries, geoms2, levels2, base = [], [], [], [], [], 0
        for pi, (pg, (ids, probs, order)) in enumerate(zip(page_geoms, rec_out)):
            n = len(pg)
            retry, pos = [], None
            if n:
                _, scores = rec.tokenizer.decode_ids(ids, probs)
                pos = np.argsort(order) if order is not None else np.arange(n)    # plan position of detection index i
                retry = [i for i in range(n) if scores[int(pos[i])] < thresh]
                retries.append((retry, pos, scores))
            else:
                retries.append(([], None, []))
            if not retry:
                continue
            sel = pg.geoms[np.asarray(retry, np.int64)].copy()
            sel["rot"] |= 2
            sel["canvas_w"] = cfg.data.img_size[1]
            geoms2.append(sel)
            levels2.append(pg.levels[np.asarray(retry, np.int64)])
            w = sel["canvas_w"].tolist()
            for s0 in range(0, len(retry), bs):
                e0 = min(len(retry), s0 + bs)
                groups.append((w[s0:e0], w[s0:e0], base + np.arange(s0, e0, dtype=np.int64)))
                owner.append(pi)
            base += len(retry)
        if not groups:
            if _multi_rank():
                # the balancing round is a collective: a rank without retries still takes part in it
                self._run_groups_dev([], np.zeros(0, CROP_GEOM_DTYPE), pages_dev, stream, np.zeros(0, np.int64))
            return
        res = self._run_groups_dev(groups, np.concatenate(geoms2), pages_dev, stream, np.concatenate(levels2))
        S = cfg.max_label_length + 1
        second = self._gather_pages(res, owner, len(rec_out))
        for (ids, probs, _), (r_ids, r_probs), (retry, pos, scores) in zip(rec_out, second, retries):
            if not len(r_ids):
                continue
            _, r_scores = rec.tokenizer.decode_ids(r_ids, r_probs)
            for j, i in enumerate(retry):
                k = int(pos[i])
                if r_scores[j] > scores[k] and r_scores[j] >= thresh:
                    ids[k, :S] = r_ids[j]
                    probs[k, :S] = r_probs[j]

    def _assemble(self, host, rec_out):
        results = []
        _t = _span("collect.assemble")
        _t.__enter__()
        r = self.recognizer
        from .schemas import WordPrediction
        for (quads, scores, *_), (ids, probs, order) in zip(host, rec_out):
            p, s, d = r._decode_in_order(ids, probs, quads, order)
            # same pairing as ocr_aggregate (reference ocr.py:6-24); the values are produced by this module with
            # the right types, so the pydantic models are built without re-validating every coordinate
            words = [_fast_word(WordPrediction, q, c, dd, float(ds), float(rs))
                     for q, ds, c, rs, dd in zip(quads, scores, p, s, d)]
            results.append(OCRSchema.model_construct(words=words))
        _t.__exit__()
        return results

    def stream(self, batches, lookahead=2, prob_override=None, quads_override=None):
        """Pipelined iteration over many batches: `for results in ocr.stream(list_of_page_lists): ...` yields the
        per-batch result lists in order.  prob_override / quads_override, if given, are per-batch lists."""
        return _stream_impl(self, batches, lookahead, prob_override, quads_override)

    def __call__(self, pages, prob_override=None, quads_override=None):
        """pages: list of BGR uint8 arrays, of one size or of many, or pages already on the GPU (a list of CUDA (H, W, 3)
        uint8 tensors, an (n, H, W, 3) CUDA tensor or a DevicePages: no host staging and no upload, the detector and the
        crop kernels read the packed buffer).  prob_override / quads_override (benchmarks with random
        detector weights): the detector still runs, but post-processing sees the given probability maps / the
        recognizer the given quads."""
        return self.collect(self.submit(pages, prob_override, quads_override))


def _stream_impl(ocr, batches, lookahead, prob_override, quads_override):
    """Generator behind BatchedOCR.stream, four stages in order: a detector thread (own CUDA stream) runs up to
    `lookahead` batches ahead and feeds the host pool; a planner thread waits for each batch's host stage and builds the
    recognizer call (grouping, records, descriptors: host only); a recognizer thread does nothing but the device calls
    on its own stream, so the GPU goes from one batch's PARSeq straight into the next one's; the calling thread turns ids
    into strings / schemas and yields.  ctypes releases the GIL inside the C calls, so DBNet(i+2), host stage and
    planning(i+1), PARSeq(i) and assembly(i-1) overlap."""
    import queue
    import threading
    import torch
    det_stream = torch.cuda.Stream(priority=-1) if torch.cuda.is_available() else None
    rec_stream = torch.cuda.Stream() if torch.cuda.is_available() else None
    q = queue.Queue(maxsize=max(1, lookahead))
    err = []
    dev = torch.cuda.current_device() if torch.cuda.is_available() else None
    # CUDA tensor pages are packed on the caller's current stream (device_pages), which the producer thread does not
    # inherit
    caller_stream = torch.cuda.current_stream() if torch.cuda.is_available() else None

    def producer():
        try:
            if dev is not None:
                torch.cuda.set_device(dev)      # the current device is per host thread

            for k, pages in enumerate(batches):
                with _span("producer.next_batch"):
                    pass
                if caller_stream is not None:
                    with torch.cuda.stream(caller_stream):
                        dp = as_device_pages(pages)
                    pages = pages if dp is None else dp
                po = None if prob_override is None else prob_override[k]
                qo = None if quads_override is None else quads_override[k]
                q.put(ocr.submit(pages, po, qo, stream=det_stream, wait_recognized=True))
        except BaseException as e:  # surfaced in the consumer
            err.append(e)
        finally:
            q.put(None)

    q1 = queue.Queue(maxsize=2)
    q2 = queue.Queue(maxsize=2)

    def planner():
        """host stage results -> recognizer plan, one batch ahead of the GPU (pure host work)"""
        try:
            while True:
                h = q.get()
                if h is None:
                    break
                try:
                    q1.put((h, ocr._prepare_handle(h)))
                except BaseException:
                    h.done.set()
                    raise
        except BaseException as e:
            err.append(e)
            while True:
                h = q.get()
                if h is None:
                    break
                h.done.set()
        finally:
            q1.put(None)

    def recognizer():
        try:
            if dev is not None:
                torch.cuda.set_device(dev)
            while True:
                item = q1.get()
                if item is None:
                    break
                h, prepared = item
                try:
                    q2.put(ocr._run_handle(h, prepared, stream=rec_stream, defer=True))
                finally:
                    h.done.set()       # the staging slot of this batch may be reused
        except BaseException as e:
            err.append(e)
            while True:                     # keep draining (and releasing staging slots) so that the producer can finish
                item = q1.get()
                if item is None:
                    break
                item[0].done.set()
        finally:
            q2.put(None)

    threads = [threading.Thread(target=producer, daemon=True), threading.Thread(target=planner, daemon=True),
               threading.Thread(target=recognizer, daemon=True)]
    import sys
    # the device threads hold the GIL for microseconds between C calls; with the default 5 ms switch interval each of
    # those hand-overs can stall behind the assembly thread (tens of ms of pure Python per batch) and idle the GPU
    old_interval = sys.getswitchinterval()
    sys.setswitchinterval(min(old_interval, 0.0005))
    try:
        for t in threads:
            t.start()
        while True:
            item = q2.get()
            if item is None:
                break
            yield ocr._assemble(*ocr._finish_handle(item))
        for t in threads:
            t.join()
    finally:
        sys.setswitchinterval(old_interval)
    if err:
        raise err[0]


class _Handle:
    """What `submit` returns: the host-stage futures of a batch + the crop arena its workers write into."""

    def __init__(self, futures, arena, cap, pages_dev=None):
        import threading
        self.futures, self.arena, self.cap, self.pages_dev = futures, arena, cap, pages_dev
        self.done = threading.Event()       # set once the batch has been recognised (or abandoned)


_WORD_FIELDS = frozenset(("points", "content", "direction", "rec_score", "det_score"))


def _fast_word(cls, points, content, direction, det_score, rec_score):
    """WordPrediction.model_construct(...) without its per-call bookkeeping (no defaults, no aliases to resolve): the
    assembly thread builds thousands of these per batch while holding the GIL the device threads also need."""
    m = cls.__new__(cls)
    object.__setattr__(m, "__dict__", {"points": points, "content": content, "direction": direction,
                                       "rec_score": rec_score, "det_score": det_score})
    object.__setattr__(m, "__pydantic_fields_set__", set(_WORD_FIELDS))
    object.__setattr__(m, "__pydantic_extra__", None)
    object.__setattr__(m, "__pydantic_private__", None)
    return m


class _PendingResults:
    """Phase-2 output of the multi-rank recognizer call: `out[k]` = (ids, probs, group_len) of the groups recognised
    here (None for the ones sent away), `back` = results this rank owes to other ranks (None: nothing moved at all)."""

    def __init__(self, out, back, plan):
        self.out, self.back, self.plan = out, back, plan


class _Done:
    def __init__(self, value):
        self._v = value

    def result(self):
        return self._v
