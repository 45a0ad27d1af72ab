"""One wide IQ stream served by several GPUs, one process per GPU (SURVEY.md §8e; BASELINE configs 3 and 5).

Every rank owns a contiguous range of the stream's channels.  The ingest rank (0) copies each raw u8 IQ block
host -> device once; ONE broadcast (NCCL over NVLink/NVSwitch; gloo in CPU tests of the plumbing) hands it to
the other ranks; each rank channelizes and demodulates only its own channels straight from the broadcast
buffer (acb_submit_device, ordered behind the broadcast by a CUDA event — no host sync).  No collective inside
the channelizer or the demodulator.  Decoded messages go back to rank 0 and are merged into the reference's
emission order (block, then channel, then time; rtl.c:357-360).

The streaming front-ends' input (kind "real": air.c's float32 samples; kind "cs16": soapy.c / sdrplay.c's int16 I,Q)
takes the same path with any number of samples per submit: rank 0 broadcasts them, every rank appends them behind its
context's carried remainder with acb_submit_real_device / acb_submit_cs16_device, and the merge follows the emission
groups of acb_set_emission_groups (group, then channel, then time), which every rank cuts alike.

The reference has no counterpart: one thread serves every channel (rtl.c:344-360).
"""
from __future__ import annotations

import numpy as np

from . import api, sharding


FLAG_REAL_INPUT, FLAG_CS16_INPUT = 2, 4


class WideStream:
    def __init__(self, dist, rank: int, world: int, local: int, K: int, freqs_hz, fc_hz: int | None, max_blocks: int,
                 taps: int = 0, wf_all: np.ndarray | None = None, flags: int = 0, kind: str = "u8", variant: int = 0,
                 group: tuple = (sharding.GROUP_SUBMIT, 0)):
        """kind "u8": raw u8 IQ blocks (rtl.c), `fc_hz` the centre acb_choose_fc gave.  kind "real" (air.c) or "cs16"
        (soapy.c / sdrplay.c by `variant`, interleaved I,Q): any number of samples per submit, the remainder carried by
        every rank; `fc_hz` None or 0 chooses the centre once over all channels (acb_air_choose_fc, acb_choose_fc), and
        `group` = (unit, period) are the emission groups of acb_set_emission_groups, which the merge follows."""
        import torch
        self.torch, self.dist, self.rank, self.world, self.local = torch, dist, rank, world, local
        self.K, self.max_blocks = K, max_blocks
        self.nch_total = len(freqs_hz)
        self.mine = sharding.channel_range(self.nch_total, world, rank)
        self.kind = kind
        if kind != "u8":
            self._init_streaming(freqs_hz, fc_hz, taps, wf_all, flags, variant, group)
            return
        self.blk_bytes = 2048 * K
        self.dev = torch.device("cuda", local)
        torch.cuda.set_device(local)
        # two broadcast buffers: submit i+1 is filled while submit i is still being channelized
        self.bufs = [torch.empty(max_blocks * self.blk_bytes, dtype=torch.uint8, device=self.dev) for _ in range(2)]
        self.ev = [torch.cuda.Event() for _ in range(2)]
        self.t0 = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        self.t1 = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        self.nsub = 0
        self.inflight = 0
        self.bcast_ms = 0.0
        self.ctx = None
        if len(self.mine):
            self.ctx = api.Context(K, 1, len(self.mine), max_blocks, device=local, flags=flags | 1, taps=taps)
            if wf_all is not None:
                self.ctx.set_wf(0, wf_all[self.mine.start:self.mine.stop])
            else:
                self.ctx.set_plan_at(0, list(freqs_hz)[self.mine.start:self.mine.stop], fc_hz)

    def _init_streaming(self, freqs_hz, fc_hz, taps, wf_all, flags, variant, group):
        torch, K, lib = self.torch, self.K, api.load()
        if self.kind not in ("real", "cs16"):
            raise ValueError(f"kind {self.kind!r}: u8, real or cs16")
        f = np.asarray(list(freqs_hz), dtype=np.uint32)
        if not fc_hz:                                    # one centre for every rank, chosen over all channels
            fc_hz = lib.acb_air_choose_fc(int(f.min()), int(f.max())) if self.kind == "real" else lib.acb_choose_fc(f.ctypes.data, len(f), K)
            if not fc_hz:
                raise api.AcbError("Frequencies too far apart")
        self.fc_hz = int(fc_hz)
        self.group = group
        self.dev = torch.device("cuda", self.local)
        torch.cuda.set_device(self.local)
        # room for a submit of max_blocks*1024*K samples plus the carried remainder (< K)
        self.cap = (self.max_blocks * 1024 + 1) * K
        per = 1 if self.kind == "real" else 2            # tensor elements per sample
        dtype = torch.float32 if self.kind == "real" else torch.int16
        self.bufs = [torch.empty(self.cap * per, dtype=dtype, device=self.dev) for _ in range(2)]
        self.ev = [torch.cuda.Event() for _ in range(2)]
        self.t0 = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        self.t1 = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        self.nsub = 0
        self.uncovered = []                              # (buffer, rows) of the submits no collect / sync has covered yet
        self.carry = 0                                   # samples short of a row, as every rank's context carries them
        self.pos = 0                                     # envelope samples produced so far
        self.starts = []                                 # emission-group starts of the submits not yet merged
        self.bcast_ms = 0.0
        self.ctx = None
        if len(self.mine):
            kflag = FLAG_REAL_INPUT if self.kind == "real" else FLAG_CS16_INPUT
            self.ctx = api.Context(K, 1, len(self.mine), self.max_blocks, device=self.local, flags=flags | kflag, taps=taps)
            mine = f[self.mine.start:self.mine.stop]
            if wf_all is not None:
                self.ctx.set_wf(0, wf_all[self.mine.start:self.mine.stop])
            elif self.kind == "real":
                self.ctx.set_plan_air_at(0, mine, self.fc_hz)
            else:
                self.ctx.set_plan_cs16(0, mine, variant, self.fc_hz)
            self.ctx.set_emission_groups(*group)

    def _free_buffer(self, b: int) -> None:
        """Wait until no submit that read buffer b is still uncovered: a submit that produced rows is covered by the
        collect that reaches it (oldest first), one that produced none only by a sync."""
        readers = [u for u in self.uncovered if u[0] == b]
        if not readers:
            return
        if self.ctx is None or any(rows == 0 for _, rows in readers):
            if self.ctx is not None:
                self.ctx.sync()
            self.uncovered.clear()
            return
        while any(u[0] == b for u in self.uncovered):
            self.ctx.collect()
            oldest = next(i for i, u in enumerate(self.uncovered) if u[1] > 0)
            del self.uncovered[oldest]

    def _submit_stream(self, x_host, nsamples: int) -> int:
        torch = self.torch
        if not 0 < nsamples <= self.cap - self.carry:
            raise ValueError(f"nsamples={nsamples} outside 1..{self.cap - self.carry}")
        b = self.nsub & 1
        self._free_buffer(b)
        per = 1 if self.kind == "real" else 2
        buf = self.bufs[b][:nsamples * per]
        self.t0[b].record()
        if self.rank == 0:
            src = x_host if isinstance(x_host, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x_host))
            buf.copy_(src.reshape(-1)[:nsamples * per], non_blocking=True)
        if self.dist is not None:
            self.dist.broadcast(buf, src=0)              # the single collective of the data path
        self.t1[b].record()
        self.ev[b].record()
        nout = (self.carry + nsamples) // self.K
        if self.ctx is not None:
            self.ctx.wait_event(self.ev[b].cuda_event)
            fn = self.ctx.submit_real_device if self.kind == "real" else self.ctx.submit_cs16_device
            got = fn(buf.data_ptr(), nsamples, nsamples)
            if got != nout:
                raise api.AcbError(f"rank {self.rank} produced {got} envelope samples, the stream {nout}")
        self.carry = (self.carry + nsamples) % self.K
        self.starts += sharding.stream_groups(self.group[0], self.group[1], self.K, self.pos, nout)
        self.pos += nout
        self.uncovered.append((b, nout))
        self.nsub += 1
        return nout

    def submit(self, iq_host, nblk: int) -> None:
        """u8: iq_host is rank 0's block(s) as a uint8 torch tensor (pinned) or numpy array, ignored elsewhere, and nblk
        the number of blocks.  real / cs16: rank 0's samples (float32 (n,), or int16 (n, 2) I,Q; numpy or a torch tensor)
        and their count n, which every rank passes; returns the envelope samples produced."""
        if self.kind != "u8":
            return self._submit_stream(iq_host, nblk)
        torch = self.torch
        b = self.nsub & 1
        if self.inflight == 2:                       # buffer b still feeds the submit two back
            if self.ctx is not None:
                self.ctx.collect()
            self.inflight -= 1
        n = nblk * self.blk_bytes
        buf = self.bufs[b][:n]
        self.t0[b].record()
        if self.rank == 0:
            src = iq_host if isinstance(iq_host, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(iq_host).reshape(-1))
            buf.copy_(src[:n], non_blocking=True)
        if self.dist is not None:
            self.dist.broadcast(buf, src=0)          # the single collective of the data path
        self.t1[b].record()
        self.ev[b].record()
        if self.ctx is not None:
            self.ctx.wait_event(self.ev[b].cuda_event)
            self.ctx.submit_device(buf.data_ptr(), nblk, n)
        self.nsub += 1
        self.inflight += 1

    def sync(self) -> None:
        if self.ctx is not None:
            self.ctx.sync()
        self.torch.cuda.synchronize()
        self.inflight = 0
        if self.kind != "u8":
            self.uncovered.clear()

    def ingest_ms(self) -> float:
        """H2D (rank 0) + broadcast device time of the last two submits' average (CUDA events, torch stream)."""
        ms = [self.t0[i].elapsed_time(self.t1[i]) for i in range(min(2, self.nsub))]
        return sum(ms) / max(1, len(ms))

    def drain_local(self):
        """This rank's messages as tuples with the GLOBAL channel index:
        (block, stream, chn, pos, len, err, txt, crc, lvl_bits)."""
        out = []
        if self.ctx is not None:
            for m in self.ctx.drain():
                out.append((int(m.block), 0, m.chn + self.mine.start, int(m.pos), m.len, m.err, bytes(m.txt[:m.len]),
                            bytes(m.crc), int(np.float32(m.lvl).view(np.uint32))))
        return out

    def gather(self):
        """All ranks' messages merged in emission order on every rank (object all-gather: a few KB)."""
        mine = self.drain_local()
        parts = [mine]
        if self.dist is not None:
            parts = [None] * self.world
            self.dist.all_gather_object(parts, mine)
        if self.kind == "u8":
            return sharding.merge_messages(parts, key=lambda m: m[:4])
        # streaming kinds: (emission group, stream, channel, time), as one context orders them
        starts = self.starts
        merged = sharding.merge_messages(parts, key=lambda m: (sharding.group_of(starts, m[3]),) + m[1:4])
        if not self.uncovered:                           # everything submitted has been merged
            self.starts = []
        return merged

    def close(self) -> None:
        if self.ctx is not None:
            self.ctx.close()
            self.ctx = None
