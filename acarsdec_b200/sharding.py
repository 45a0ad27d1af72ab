"""Multi-GPU plumbing: one process per GPU, torch.distributed for rendezvous only.

The path shards without any data-path collective (SURVEY.md §8e): channels share nothing but the
read-only matched filter, streams share nothing at all.

  * many streams (BASELINE config 4): stream index ranges per rank, zero communication;
  * one wide stream (configs 3, 5): channel index ranges per rank; every rank needs the same raw
    u8 IQ block, which is the single broadcast the north star allows (NCCL over NVLink on GPUs,
    gloo in the CPU tests) — each rank then channelizes/demodulates only its own channels.

Decoded messages come back per rank and are merged in the reference's emission order
(block-major, then stream, then channel, then time; rtl.c:357-360); for the streaming front-ends (real input,
CS16) the emission group of acb_set_emission_groups takes the block's place.
"""
from __future__ import annotations

import bisect
import os
from typing import Iterable, Sequence


def env_rank_world():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))


def split_range(n: int, world: int, rank: int) -> range:
    """Contiguous, balanced (sizes differ by at most 1), order-preserving split of range(n)."""
    if not (0 <= rank < world):
        raise ValueError("rank outside world")
    base, extra = divmod(n, world)
    lo = rank * base + min(rank, extra)
    return range(lo, lo + base + (1 if rank < extra else 0))


def stream_range(total_streams: int, world: int, rank: int) -> range:
    return split_range(total_streams, world, rank)


def rank_counts(counts, total_streams: int, world: int, rank: int):
    """The per-stream counts of a ragged submit that this rank's streams (stream_range) take."""
    r = stream_range(total_streams, world, rank)
    return counts[r.start:r.stop]


def channel_range(nch: int, world: int, rank: int) -> range:
    return split_range(nch, world, rank)


def init_process_group(backend: str | None = None):
    """torch.distributed rendezvous from the torchrun environment (MASTER_ADDR must be 127.0.0.1
    style resolvable).  Returns (dist module or None, rank, world, local_rank)."""
    rank, world, local = env_rank_world()
    if world == 1:
        return None, rank, world, local
    import torch
    import torch.distributed as dist
    if backend is None:
        backend = "nccl" if torch.cuda.is_available() else "gloo"
    kw = {}
    if backend == "nccl":
        torch.cuda.set_device(local)
        kw["device_id"] = torch.device("cuda", local)
    dist.init_process_group(backend, **kw)
    return dist, rank, world, local


def broadcast_iq(dist, tensor, src: int = 0):
    """The one collective of the wide-stream case: the ingest rank's raw uint8 IQ block to all."""
    if dist is not None:
        dist.broadcast(tensor, src=src)
    return tensor


def reduce_scalar(dist, x: float, op: str, device=None) -> float:
    """max / sum of a python float over ranks (timing and sample counts)."""
    if dist is None:
        return x
    import torch
    t = torch.tensor([x], dtype=torch.float64, device=device)
    dist.all_reduce(t, op={"max": dist.ReduceOp.MAX, "sum": dist.ReduceOp.SUM}[op])
    return float(t.item())


def whole_job_throughput(dist, samples_local: float, seconds_local: float, device=None) -> float:
    """Aggregate samples/s: all ranks' samples over the slowest rank's time."""
    total = reduce_scalar(dist, samples_local, "sum", device)
    slowest = reduce_scalar(dist, seconds_local, "max", device)
    return total / slowest


GROUP_SUBMIT, GROUP_OUTPUTS, GROUP_INPUT = 0, 1, 2      # acb_set_emission_groups's units


def stream_groups(unit: int, period: int, K: int, pos: int, nout: int) -> list:
    """Emission-group starts of a streaming submit that produced envelope samples [pos, pos + nout), as a context cuts
    them (acb_set_emission_groups): the first is pos, then one every `period` outputs counted from the stream start
    (GROUP_OUTPUTS), or one per transfer of `period` input samples (GROUP_INPUT: output m completes with input sample
    (m+1)K - 1, so transfer t starts a group at output t*period // K).  A submit that produced no row has no group."""
    if nout <= 0:
        return []
    g, hi = [pos], pos + nout
    if unit == GROUP_OUTPUTS:
        b = (pos // period + 1) * period
        while b < hi:
            g.append(b)
            b += period
    elif unit == GROUP_INPUT:
        t = pos * K // period + 1                          # transfers that start after output `pos` began
        while True:
            b = t * period // K                            # first output completed inside transfer t
            if b >= hi:
                break
            if b > g[-1]:
                g.append(b)
            t += 1
    return g


def group_number(unit: int | None, period: int, K: int, pos: int) -> int:
    """The number, counted from the stream's start, of the emission group holding envelope sample `pos` (the context's
    rule for streams at different positions, acb_set_emission_groups): unit None is u8 IQ, a group per 1024-row block;
    GROUP_OUTPUTS one per `period` outputs; GROUP_INPUT the transfers' first outputs t*period // K (t >= 1) in (0, pos];
    GROUP_SUBMIT numbers none (the submit is the group).  Within a submit frames leave in (group_number, stream, channel,
    time) order."""
    if unit is None:
        return pos // 1024
    if unit == GROUP_OUTPUTS:
        return pos // period
    if unit == GROUP_INPUT:
        return ((pos + 1) * K - 1) // period if period >= K else pos
    return 0


def group_of(starts: Sequence[int], pos: int) -> int:
    """Index of a message's emission group: the last start at or before its pos (`starts` ascending)."""
    return bisect.bisect_right(starts, pos)


def merge_messages(per_rank: Sequence[Iterable], key=lambda m: (m.block, m.stream, m.chn, m.pos)):
    """Per-rank message lists (each already in emission order, with GLOBAL stream/channel
    indices) -> one list in the reference's emission order."""
    out = [m for lst in per_rank for m in lst]
    out.sort(key=key)
    return out
