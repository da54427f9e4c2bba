"""Batch sharding of independent utterances / clips over the GPUs of one box.

The hot path has no cross-sample operation (GroupNorm/LayerNorm/attention are per sample,
CFG pairs stay on one GPU), so the data path shards with NO collective (SURVEY.md 8e).
The only collectives are the two the north star names, both outside the kernels:

* one broadcast of the packed weights at start-up (``broadcast_state_dict``), and
* one all-gather of the finished fp32 waveforms per batch (``all_gather_rows``).

One process per GPU (``torch.distributed``; NCCL over NVLink on a multi-GPU machine, gloo in the
CPU tests).  The reference has no inference-time multi-GPU at all: its tool classes are
pinned to fixed devices by hand (audio-chatgpt.py:1051-1073).
"""
from __future__ import annotations

import os
from typing import Dict, List, Sequence, Tuple

import torch
import torch.distributed as dist


def init_distributed(backend: str = None) -> Tuple[int, int, int]:
    """(rank, world, local_rank) from the torchrun environment; no-op when WORLD_SIZE is unset/1."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend == "nccl":
            torch.cuda.set_device(local)
            dist.init_process_group(backend, rank=rank, world_size=world, device_id=torch.device("cuda", local))
        else:
            dist.init_process_group(backend, rank=rank, world_size=world)
    return rank, world, local


def shard_range(total: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous ceil(total/world) slices; trailing ranks may get fewer (or zero) items."""
    per = -(-total // world)
    lo = min(total, rank * per)
    return lo, min(total, lo + per)


def broadcast_state_dict(sd: Dict[str, torch.Tensor], src: int = 0, device=None) -> Dict[str, torch.Tensor]:
    """One flat blob per dtype, one broadcast each (a model's state dict is all-fp32 on this path: one broadcast).
    Every rank passes a dict with the same keys / shapes / dtypes (contents only matter on ``src``); the
    agreement is CHECKED with a hash of the (key, shape, dtype) list before any payload moves, and every entry
    comes back in its own dtype (no silent fp32 round trip for integer buffers or half checkpoints).
    The engines re-lay the weights out at ``create`` on every rank (deterministic host packing), so what
    travels is the reference-layout state dict, not the kernel-layout operand images."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return sd
    import hashlib
    keys = list(sd.keys())
    dev = device if device is not None else (torch.device("cuda", torch.cuda.current_device())
                                             if dist.get_backend() == "nccl" else torch.device("cpu"))
    sig = hashlib.sha256(repr([(k, tuple(sd[k].shape), str(sd[k].dtype)) for k in keys]).encode()).digest()[:8]
    mine = torch.tensor(list(sig), dtype=torch.int64, device=dev)
    ref = mine.clone()
    dist.broadcast(ref, src=src)
    agree = torch.tensor([1 if torch.equal(ref, mine) else 0], dtype=torch.int64, device=dev)
    dist.all_reduce(agree, op=dist.ReduceOp.MIN)
    if int(agree.item()) != 1:
        raise RuntimeError("broadcast_state_dict: ranks disagree on the (key, shape, dtype) list of the state dict")
    out: Dict[str, torch.Tensor] = {}
    by_dtype: Dict[torch.dtype, List[str]] = {}
    for k in keys:
        by_dtype.setdefault(sd[k].dtype, []).append(k)
    for dt, ks in by_dtype.items():
        sizes = [sd[k].numel() for k in ks]
        flat = torch.empty(sum(sizes), dtype=dt, device=dev)
        if dist.get_rank() == src:
            off = 0
            for k, n in zip(ks, sizes):
                flat[off:off + n].copy_(sd[k].reshape(-1))
                off += n
        dist.broadcast(flat, src=src)
        flat_cpu = flat.cpu()
        off = 0
        for k, n in zip(ks, sizes):
            out[k] = flat_cpu[off:off + n].reshape(sd[k].shape).clone()
            off += n
    return {k: out[k] for k in keys}


class AsyncGather:
    """All-gather of finished per-rank row blocks that stays OFF the compute stream's critical path: ``submit(x)``
    enqueues ``all_gather_into_tensor`` asynchronously (NCCL's own stream, ordered after the work that produced
    ``x``), so the gather of batch i overlaps the computation of batch i+1; ``drain()`` makes the current stream
    wait for everything outstanding and returns the gathered tensors in submission order."""

    def __init__(self):
        self._pending = []

    def submit(self, x: torch.Tensor):
        if not dist.is_initialized() or dist.get_world_size() == 1:
            self._pending.append((None, x))
            return
        world = dist.get_world_size()
        x = x.contiguous()
        out = torch.empty((world * x.shape[0],) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        work = dist.all_gather_into_tensor(out, x, async_op=True)
        self._pending.append((work, out, x))

    def drain(self):
        outs = []
        for item in self._pending:
            if item[0] is not None:
                item[0].wait()          # stream-level wait: the current stream is ordered after the collective
            outs.append(item[1])
        self._pending = []
        return outs


def all_gather_rows(x: torch.Tensor, counts: Sequence[int] = None) -> torch.Tensor:
    """Concatenate per-rank row blocks [b_r, ...] along dim 0 on every rank.  ``counts`` (rows
    per rank) enables ragged shards; blocks are padded to max(counts) for the collective."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return x
    world = dist.get_world_size()
    if counts is None:
        out = torch.empty((world * x.shape[0],) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        dist.all_gather_into_tensor(out, x.contiguous())
        return out
    m = max(counts)
    pad = torch.zeros((m,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    pad[: x.shape[0]] = x
    out = torch.empty((world * m,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    dist.all_gather_into_tensor(out, pad)
    return torch.cat([out[r * m: r * m + counts[r]] for r in range(world)], dim=0)


class P2PGather:
    """All-gather of finished per-rank row blocks over NVLink by the COPY ENGINES, not by SM kernels: every rank owns
    a gather buffer [world, *block]; the buffers are exchanged once as CUDA IPC handles (the mechanism
    ``torch.multiprocessing`` uses to share CUDA tensors), and ``submit(x)`` issues one peer ``cudaMemcpyAsync`` per
    destination (``tensor.copy_`` between devices) on a side stream that waits on the producing stream through an
    event.  Nothing of it runs on the SMs, so a persistent 148-CTA compute grid is not disturbed (an NCCL all-gather
    kernel launched under such a grid delays whichever CTAs it displaces: round 1 lost 3.7 points of weak-scaling
    efficiency there).  ``drain()`` waits for this rank's copies and meets the other ranks at a barrier; after it,
    ``gathered(slot)`` holds every rank's block.  Double-buffered: consecutive submits alternate between two slots.
    Measured (bench.py, HiFi-GAN 8 x 800 frames per rank): 0.6 % ahead of the asynchronous NCCL gather at N = 2, 4 %
    behind it at N = 4 (N - 1 serial peer copies per rank) -- bench.py therefore defaults to AsyncGather."""

    def __init__(self, block_shape, dtype=torch.float32, device=None, slots: int = 2):
        from torch.multiprocessing.reductions import reduce_tensor
        assert dist.is_initialized() and dist.get_world_size() > 1
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        self.dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.slots = slots
        self.buf = torch.zeros((slots, self.world) + tuple(block_shape), dtype=dtype, device=self.dev)
        fn, args = reduce_tensor(self.buf)
        handles = [None] * self.world
        dist.all_gather_object(handles, args)
        self.peers, err = [], None
        try:
            for r in range(self.world):
                self.peers.append(self.buf if r == self.rank else fn(*handles[r]))
            probe = torch.zeros(1, dtype=dtype, device=self.dev)
            for r in range(self.world):                # one element to every peer: mapping and peer access really work
                self.peers[r][0, self.rank].reshape(-1)[:1].copy_(probe)
            torch.cuda.synchronize(self.dev)
        except Exception as e:                         # noqa: BLE001 -- reported below, on every rank together
            err = e
        # every rank learns whether ALL mappings succeeded (instead of a barrier a failed rank would never reach)
        flag = torch.tensor([0 if err is not None else 1], dtype=torch.int32, device=self.dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        if int(flag.item()) == 0:
            raise RuntimeError(f"P2PGather: mapping the peers' buffers failed on at least one rank (this rank: {err!r})")
        self.stream = torch.cuda.Stream(device=self.dev)
        self.n = 0

    def submit(self, x: torch.Tensor):
        slot = self.n % self.slots
        self.n += 1
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.dev))
        x.record_stream(self.stream)                    # the block must outlive the asynchronous copies
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(ev)
            for r in range(self.world):
                self.peers[r][slot, self.rank].copy_(x, non_blocking=True)
        return slot

    def drain(self):
        torch.cuda.current_stream(self.dev).wait_stream(self.stream)
        self.stream.synchronize()
        dist.barrier()

    def gathered(self, slot: int) -> torch.Tensor:
        return self.buf[slot].reshape((-1,) + tuple(self.buf.shape[3:]))


# ---- mixed dispatch (BASELINE configs[4]): greedy longest-processing-time assignment ----
HIFIGAN_GFLOP_PER_FRAME = 0.614          # V1, SURVEY.md 8d
DDIM100_TFLOP_PER_CLIP = 18.66 + 0.39    # UNet x200 forwards + VAE decode


def job_cost_tflop(kind: str, frames: int = 0) -> float:
    if kind == "tts":
        return HIFIGAN_GFLOP_PER_FRAME * frames * 1e-3
    if kind == "t2a":
        return DDIM100_TFLOP_PER_CLIP + HIFIGAN_GFLOP_PER_FRAME * 624 * 1e-3
    raise ValueError(kind)


def lpt_assign(costs: Sequence[float], workers: int) -> List[List[int]]:
    """Greedy LPT: jobs sorted by decreasing cost, each to the currently least-loaded worker.
    Returns per-worker job-index lists (deterministic: ties broken by lower worker id)."""
    order = sorted(range(len(costs)), key=lambda i: (-costs[i], i))
    load = [0.0] * workers
    out: List[List[int]] = [[] for _ in range(workers)]
    for i in order:
        w = min(range(workers), key=lambda j: (load[j], j))
        out[w].append(i)
        load[w] += costs[i]
    return out


def run_mixed(jobs: Sequence[Tuple[str, int]], run_job, *, sync=None, run_group=None, group_size: Dict[str, int] = None) -> Dict[str, object]:
    """BASELINE configs[4] (mixed dispatch): ``jobs`` = [(kind, frames), ...] known to every rank in the same
    order; greedy-LPT assignment by the FLOP cost model (SURVEY.md 8e), every rank runs its own jobs with
    ``run_job(index, kind, frames)`` (no data-path collective), then ONE all_gather of the per-rank timings.

    Returns, on every rank: ``assignment`` (per-rank job indices), ``busy_s`` (per-rank busy seconds),
    ``makespan_s`` (max over ranks), ``jobs_per_s`` and ``busy_fraction`` (busy / makespan per rank).
    ``sync`` is called before each clock read (pass ``torch.cuda.synchronize`` on a GPU).
    ``run_group(kind, indices)`` (optional) lets a rank serve its OWN jobs of one kind in micro-batches of at most
    ``group_size[kind]`` (default 1) -- e.g. four text-to-audio clips as one CFG batch of 8; the assignment itself
    is unchanged."""
    import time
    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    costs = [job_cost_tflop(k, f) for k, f in jobs]
    assignment = lpt_assign(costs, world)
    if sync:
        sync()
    t0 = time.perf_counter()
    if run_group is None:
        for i in assignment[rank]:
            run_job(i, jobs[i][0], jobs[i][1])
    else:
        gs = group_size or {}
        by_kind: Dict[str, List[int]] = {}
        for i in assignment[rank]:
            by_kind.setdefault(jobs[i][0], []).append(i)
        for kind, idxs in by_kind.items():
            n = max(1, int(gs.get(kind, 1)))
            for a in range(0, len(idxs), n):
                run_group(kind, idxs[a:a + n])
    if sync:
        sync()
    busy = time.perf_counter() - t0
    if world > 1:
        dev = (torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu"))
        mine = torch.tensor([busy], dtype=torch.float64, device=dev)
        allb = torch.empty(world, dtype=torch.float64, device=dev)
        dist.all_gather_into_tensor(allb, mine)
        busy_s = [float(v) for v in allb.cpu()]
    else:
        busy_s = [busy]
    mk = max(busy_s)
    return {"assignment": assignment, "busy_s": busy_s, "makespan_s": mk,
            "jobs_per_s": len(jobs) / mk if mk > 0 else float("inf"),
            "busy_fraction": [b / mk if mk > 0 else 1.0 for b in busy_s],
            "model_load_tflop": [sum(costs[i] for i in w) for w in assignment]}
