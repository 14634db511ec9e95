"""Multi-GPU plumbing for the OCR path: one process per GPU, torch.distributed (NCCL over NVLink on the GPU box,
gloo in the CPU tests).  The reference has no distributed code at all (SURVEY.md section 2.2); this is new surface.

What crosses the fabric (SURVEY.md section 8e) - never inside a forward pass:
  * `broadcast_state_dict`   one-time weight broadcast from rank 0 (one flat buffer per dtype);
  * the crop scatter         whole reference mini-batches ("groups": the unit whose rows must stay together because
                             the AR loop stops per group) move between ranks so that every GPU gets a balanced number
                             of encoder tokens.  Control plane on host-side gloo groups (`meta_group`: costs,
                             assignment, descriptors - exchanged one batch ahead by the planner threads), data plane
                             `exchange_canvases_planned`: ONE all_to_all_single of device uint8 canvases over NCCL;
  * the result gather        (ids int32, probs fp32) per crop back to the owning rank over a second gloo group
                             (`exchange_results_planned`, `BatchedOCR._finish_results`, assembly thread).
Crops cut on the device leave from HBM as they are; crops cut by OpenCV on the host (`YTK_DEVICE_CROPS=0`) are
gathered and uploaded once, then take the same exchange.
Pages are sharded by rank for detection (page p -> rank p // pages_per_rank); that needs no communication.
"""
import numpy as np
import torch
import torch.distributed as dist


def _dev():
    return torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")


def broadcast_state_dict(sd, device=None):
    """Broadcast every floating tensor of rank 0's state_dict (one flat fp32 buffer), returns a CPU state_dict."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return sd
    device = _dev()
    keys = [k for k in sd if torch.is_floating_point(sd[k])]
    flat = torch.cat([sd[k].detach().reshape(-1).to(torch.float32) for k in keys]).to(device)
    dist.broadcast(flat, src=0)
    flat = flat.cpu()
    out, off = dict(sd), 0
    for k in keys:
        n = sd[k].numel()
        out[k] = flat[off:off + n].reshape(sd[k].shape).clone()
        off += n
    return out


def balance_groups(costs_by_rank, world, tolerance=0.03):
    """Deterministic group -> rank assignment.  costs_by_rank[r] = list of costs (encoder tokens) of the groups rank r
    owns.  Groups stay with their owner unless moving them lowers the maximum load by more than `tolerance`
    (longest-processing-time greedy over the groups of overloaded ranks).  Returns assign[r][g] = destination rank."""
    if len(costs_by_rank) != world:
        costs_by_rank = list(costs_by_rank) + [[] for _ in range(world - len(costs_by_rank))]
    load = [float(sum(c)) for c in costs_by_rank]
    assign = [[r] * len(c) for r, c in enumerate(costs_by_rank)]
    total = sum(load)
    if world == 1 or total == 0:
        return assign
    target = total / world
    # candidates: groups of ranks above target, largest first
    order = sorted(((c, r, g) for r, cs in enumerate(costs_by_rank) for g, c in enumerate(cs)), key=lambda t: (-t[0], t[1], t[2]))
    for c, r, g in order:
        if load[r] <= target * (1 + tolerance):
            continue
        dst = min(range(world), key=lambda k: (load[k], k))
        if dst != r and load[dst] + c < load[r] - 1e-9 and max(load[dst] + c, load[r] - c) < load[r]:
            assign[r][g] = dst
            load[r] -= c
            load[dst] += c
    return assign


STATS = {"exchange_calls": 0, "exchange_bytes_sent": 0, "exchange_bytes_received": 0, "exchange_ms": 0.0,
         "plan_ms": 0.0, "results_ms": 0.0}     # host time inside the control-plane collectives (includes waiting for peers)

_META = {}


def meta_group(which):
    """A host-side (gloo) process group for small control messages, one per purpose ("plan": group costs / descriptors
    exchanged by the planner threads one batch ahead of the GPU, "results": ids / probabilities of groups that were
    recognised on another rank, exchanged by the assembly threads).  They never touch the NCCL communicator the
    recognizer thread uses for the canvases, so the three kinds of traffic cannot block each other.  Created
    collectively on first use (every rank reaches that point in the same order); with a gloo default group the default
    group itself serves "plan" and one extra group "results"."""
    if which not in _META:
        _META[which] = dist.new_group(backend="gloo")
    return _META[which]


def all_gather_objects(obj, which):
    """all_gather of one picklable object per rank over the `which` meta group -> list indexed by rank."""
    import time
    t0 = time.perf_counter()
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, obj, group=meta_group(which))
    STATS[which + "_ms"] = STATS.get(which + "_ms", 0.0) + (time.perf_counter() - t0) * 1e3
    return out


def exchange_canvases_planned(canv, send_splits, recv_splits, out=None):
    """The crop scatter proper, with split sizes already agreed on by the planners: ONE all_to_all_single of device uint8
    canvases over NCCL / NVLink (CPU tensors under gloo).  Returns the flat receive buffer (ordered by source rank);
    `out` = where to receive (e.g. the tail of the recognizer's work buffer)."""
    import time
    t0 = time.perf_counter()
    recv = torch.empty(int(sum(recv_splits)), dtype=torch.uint8, device=canv.device) if out is None else out
    if recv.numel() != int(sum(recv_splits)):
        raise ValueError("exchange_canvases_planned: receive buffer has %d bytes, the plan says %d"
                         % (recv.numel(), int(sum(recv_splits))))
    dist.all_to_all_single(recv, canv[: int(sum(send_splits))], output_split_sizes=[int(v) for v in recv_splits],
                           input_split_sizes=[int(v) for v in send_splits])
    STATS["exchange_calls"] += 1
    STATS["exchange_bytes_sent"] += int(sum(send_splits))
    STATS["exchange_bytes_received"] += int(sum(recv_splits))
    STATS["exchange_ms"] += (time.perf_counter() - t0) * 1e3
    return recv


def exchange_results_planned(send, send_splits, recv_splits):
    """The way back of the crop scatter: ids / probabilities of the groups recognised for other ranks, as ONE
    all_to_all_single of host bytes over the "results" gloo group (the results are on the host already: the recognizer
    call ends with their D2H copy), byte counts agreed on by the planners.  send: flat uint8 numpy array ordered by
    destination rank.  Returns the flat uint8 numpy receive buffer ordered by source rank."""
    import time
    t0 = time.perf_counter()
    if send.size != int(sum(send_splits)):
        raise ValueError("exchange_results_planned: %d bytes to send, the plan says %d" % (send.size, int(sum(send_splits))))
    recv = torch.empty(int(sum(recv_splits)), dtype=torch.uint8)
    dist.all_to_all_single(recv, torch.from_numpy(np.ascontiguousarray(send)),
                           output_split_sizes=[int(v) for v in recv_splits],
                           input_split_sizes=[int(v) for v in send_splits], group=meta_group("results"))
    STATS["results_ms"] += (time.perf_counter() - t0) * 1e3
    STATS["results_bytes_sent"] = STATS.get("results_bytes_sent", 0) + int(send.size)
    return recv.numpy()
