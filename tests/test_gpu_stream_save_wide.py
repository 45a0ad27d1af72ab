"""Moving streams (acb_save_streams / acb_load_streams) at wide shapes: records of hundreds of channels, whose device
regions span many SP_CHUNKs of k_stream_pack / k_stream_unpack; a thousand records in one call; and channel splits whose
part boundaries fall inside an 8-channel group (CH_GROUP) and between wideband channel tiles (WB_CTILE).

The promise is tests/test_gpu_stream_save.py's: a moved stream continues bit for bit (messages with every field, the last
envelope rows, chain states, decode and level statistics), and the target's other streams do not change.  Frames are in
flight at the save on the channels on both sides of every boundary: 7/8 (a channel group), 99/100 and 199/200 (three
parts of 300, slot 4 of a group), 149/150 (two parts of 300), 255/256 (a wideband tile) and the last channel."""
import functools

import numpy as np
import pytest

from acarsdec_b200 import api, synth
from test_gpu_level_stats_wide import Dev, submit
from test_gpu_stream_save import _full, _same_levels
from test_wideband_real_oracle import air_freqs

pytestmark = pytest.mark.gpu

DECODE, LEVEL = api.FLAG_DECODE_STATS, api.FLAG_LEVEL_STATS
FLAG_REAL, FLAG_CS16 = 2, 4
FC, FF, FFR, FW, FWR = 8, 16, 32, 64, 128
OUTBLK = 1024
OPEN = (3, 4, 5)                               # F_TXT, F_CRC1, F_CRC2: a frame is being assembled
SRC = 1                                        # the moved stream

# restated from acb_internal.h / context.cu (mv_layout)
SP_CHUNK = 256 * 16 * 4                        # bytes of one k_stream_pack CTA
CHAIN_STATE_BYTES, CH_GROUP, WB_CTILE = 432, 8, 256


def bounds(nch):
    """the channels next to every boundary the conversions have (those that exist at nch)"""
    b = [6, 7, 8, 13, 14, 15, 19] if nch <= 20 else [7, 8, 99, 100, 149, 150, 199, 200, 255, 256]
    return sorted({c for c in b if c < nch} | {nch - 1})


def freqs(kind, K, nch):
    if kind == "real":
        return air_freqs(K, nch)
    return [120_000_000 + 25_000 * i for i in range(nch)]


def kflag(kind):
    return FLAG_REAL if kind == "real" else FLAG_CS16 if kind == "cs16" else 0


def plan(ctx, kind, s, fd):
    """plans stream s; returns its centre frequency"""
    if kind == "u8":
        return ctx.set_plan(s, fd)
    if kind == "real":
        return ctx.set_plan_air(s, fd)
    return ctx.set_plan_cs16(s, fd, 0)


def make(kind, K, nch, S, flags, taps, parts=None, mode=1):
    """a context, or (parts: a number of parts on device 0) a channel split (mode 1) or stream split (mode 0)"""
    fl = flags | kflag(kind) | DECODE | LEVEL
    ctx = api.Context(K, S, nch, 2, flags=fl, taps=taps) if parts is None else \
        api.MultiContext(K, S, nch, 2, [0] * parts, mode=mode, flags=fl, taps=taps)
    fd = freqs(kind, K, nch)
    fc = [plan(ctx, kind, s, fd) for s in range(S)]
    return ctx, fc[0]


def schedule(kind, K):
    """per submit, the samples (u8: blocks) of the moved stream; the save follows submit SAVE_AT.  The streaming kinds
    carry a partial row across the save, and the open level window is partly filled."""
    if kind == "u8":
        return [2, 1, 2, 2, 2, 1]
    return [r * K + e for r, e in zip([2047, 1024, 2000, 2040, 2047, 1024], [5, 7, 11, 3, 2, 1])]


SAVE_AT = 3


@functools.lru_cache(maxsize=4)
def signal(kind, K, nch, fc, n, seed):
    """the moved stream: a frame starting 0.15 s before the save on every boundary channel (in its text at the save), and
    frames complete before it on a few channels"""
    sched = schedule(kind, K)
    rows_at_save = sum(sched[:SAVE_AT]) * OUTBLK if kind == "u8" else sum(sched[:SAVE_AT]) // K
    t_save = rows_at_save / synth.INTRATE
    rng = np.random.default_rng(seed)
    p = synth.StreamPlan(K=K, freqs_hz=tuple(freqs(kind, K, nch)), fc_hz=int(fc), seed=seed)
    for c in bounds(nch):
        txt = synth.random_text(rng, 60)
        p.bursts.append(synth.Burst(chan=c, t0=t_save - 0.15, frame=synth.frame_bytes(txt), amp=float(rng.uniform(9, 13)),
                                    phase=float(rng.uniform(0, 6.28))))
    for c in bounds(nch)[::3]:
        p.bursts.append(synth.Burst(chan=c, t0=0.02, frame=synth.frame_bytes(synth.random_text(rng, 12)), amp=11.0))
    if kind == "u8":
        return synth.render_blocks(p, 0, n // (OUTBLK * K)).reshape(-1)
    if kind == "real":
        return synth.render_real(p, 0, n)
    return synth.render_cs16(p, 0, n)


def unit(kind, K):
    return OUTBLK * K * 2 if kind == "u8" else 1


class Feed:
    """a context's streams, each reading its own signal from its own offset; ragged submits"""

    def __init__(self, ctx, kind, K, sigs, dev=False):
        self.ctx, self.kind, self.K, self.sigs = ctx, kind, K, sigs
        self.off = [0] * len(sigs)
        self.store = Dev() if dev else None
        self.i = 0
        self.rows = None

    def submit(self, counts):
        u = unit(self.kind, self.K)
        parts = [self.sigs[k][self.off[k] * u:(self.off[k] + c) * u] if c else self.sigs[k][:0] for k, c in enumerate(counts)]
        dev = self.store is not None and self.i % 2 == 1
        self.rows = submit(self.ctx, self.kind, self.K, parts, counts, dev, self.store)
        self.off = [o + c for o, c in zip(self.off, counts)]
        self.i += 1


def states(ctx, s, nch):
    return [bytes(ctx.get_state(s, c)) for c in range(nch)]


def stats(ctx, s):
    inp, ch = ctx.level_stats()
    return [ctx.decode_stats()[s].tobytes(), inp[s].tobytes(), ch[s].tobytes()]


def without_level_sums(blob, nch):
    """a DECODE | LEVEL blob with its CRC, every record's open-window carries and channel level table zeroed: what a
    channel split must give byte for byte (its parts tile the envelope level sums by their own channel counts).  The
    record's tail is [LevelCarry x nch][decode stats x nch][input levels][channel levels x nch], with no padding."""
    info = api.blob_info(blob)
    rec, b = info.record_bytes, bytearray(blob)
    assert len(b) == 64 + info.count * rec and (nch * (16 + 120 + 40) + 32) % 16 == 0
    b[12:16] = bytes(4)
    for i in range(info.count):
        end = 64 + (i + 1) * rec
        lch = end - nch * 40
        lcarry = lch - 32 - nch * 120 - nch * 16
        b[lcarry:lcarry + nch * 16] = bytes(nch * 16)
        b[lch:end] = bytes(nch * 40)
    return bytes(b)


class Case:
    """the moved stream's signal, the other stream's, the reference run and the saves"""

    def __init__(self, kind, K, nch, flags, taps):
        self.kind, self.K, self.nch, self.flags, self.taps = kind, K, nch, flags, taps
        self.sched = schedule(kind, K)
        n = sum(self.sched) * (OUTBLK * K if kind == "u8" else 1)
        _, fc = make_probe(kind, K, nch, flags, taps)
        # both streams of the source carry the same signal (rendering hundreds of channels is the slow part), so a
        # record that lands in the other slot is caught only by the positions; the targets' other streams differ
        self.sig = [signal(kind, K, nch, fc, n, K + nch)] * 2
        ref, _ = make(kind, K, nch, 2, flags, taps)
        f = Feed(ref, kind, K, self.sig, dev=True)
        for c in self.sched:
            f.submit([c, c])
        self.last = ref.read_dm(int(max(f.rows)))[SRC, :int(f.rows[SRC])]
        ref.sync()
        self.msgs = [_full(m) for m in ref.drain() if m.stream == SRC]
        self.state, self.stats = states(ref, SRC, nch), stats(ref, SRC)
        ref.close()
        assert len(self.msgs) > 0

    def save(self, parts=None):
        """the source (a single context, or a channel split of `parts`) fed up to the save: the blob, the moved
        stream's messages drained after it, and which boundary channels had a frame open"""
        src, _ = make(self.kind, self.K, self.nch, 2, self.flags, self.taps, parts)
        f = Feed(src, self.kind, self.K, self.sig, dev=parts is None)
        for c in self.sched[:SAVE_AT]:
            f.submit([c, c])
        blob = src.save_streams([SRC])
        open_ = [c for c in bounds(self.nch) if src.get_state(SRC, c).Acarsstate in OPEN]
        src.sync()
        pre = [_full(m) for m in src.drain() if m.stream == SRC]
        src.close()
        return blob, pre, open_

    def cont(self, ctx, T, dst, blob, pre, load=True, others=None):
        """the target: streams other than dst fed `others` (their own signals) before and after the load; dst loads the
        blob and continues the moved stream.  Returns (messages, last rows, states, stats, others' output)."""
        kind, K = self.kind, self.K
        sigs = [others[k] if k != dst and others else self.sig[SRC] for k in range(T)]
        f = Feed(ctx, kind, K, sigs, dev=isinstance(ctx, api.Context))
        busy = others is not None
        if busy:
            f.submit([self.sched[0] if k != dst else 0 for k in range(T)])
        if load:
            ctx.load_streams([dst], blob)
        f.off[dst] = sum(self.sched[:SAVE_AT])
        for c in self.sched[SAVE_AT:]:
            f.submit([(c if busy else 0) if k != dst else (c if load else 0) for k in range(T)])
        last = ctx.read_dm(int(max(f.rows)))[dst, :int(f.rows[dst])] if isinstance(ctx, api.Context) else None
        ctx.sync()
        msgs = ctx.drain()
        mine = [(SRC,) + _full(m)[1:] for m in msgs if m.stream == dst]
        out = dict(msgs=pre + mine, last=last, state=states(ctx, dst, self.nch), stats=stats(ctx, dst),
                   others=([_full(m) for m in msgs if m.stream != dst], [states(ctx, k, self.nch) for k in range(T) if k != dst]))
        ctx.close()
        return out

    def check(self, got, chan_split=False):
        assert got["msgs"] == self.msgs, "messages"
        if got["last"] is not None:
            assert got["last"].shape == self.last.shape and np.array_equal(got["last"].view(np.uint32), self.last.view(np.uint32)), \
                "envelope"
        assert got["state"] == self.state, "chain states"
        if chan_split:
            assert got["stats"][:2] == self.stats[:2] and _same_levels(got["stats"][2], self.stats[2]), "statistics"
        else:
            assert got["stats"] == self.stats, "statistics"


def make_probe(kind, K, nch, flags, taps):
    """the centre frequency the plan chooses (the signal is rendered around it)"""
    ctx, fc = make(kind, K, nch, 1, flags, taps)
    ctx.close()
    return None, fc


def assert_in_flight(open_, nch, parts_at):
    """a frame open at the save next to every part boundary (on one side or the other) and on most boundary channels"""
    for b in parts_at:
        assert b - 1 in open_ or b in open_, (b, open_)
    assert len(open_) * 2 >= len(bounds(nch)), open_


# ------------------------------------------------------------------ records of hundreds of channels

LARGE = [("u8", 1600, 0, 0), ("u8", 1600, 0, 4 * 1600 + 3), ("u8", 1600, FW, 0), ("cs16", 1600, FW, 2 * 1600 + 3),
         ("real", 1608, FWR, 0)]


@pytest.mark.parametrize("kind,K,flags,taps", LARGE)
def test_large_regions(kind, K, flags, taps):
    """one stream of 300 channels moved to another slot of a busier context: the chain states span more than 7 SP_CHUNKs
    and the exact tables over 100"""
    nch, T, dst = 300, 3, 2
    assert nch * CHAIN_STATE_BYTES > 7 * SP_CHUNK
    assert -(-nch // CH_GROUP) * K * CH_GROUP * 2 * 4 > 100 * SP_CHUNK       # R_WF: at least taps_pad >= K taps per group
    case = Case(kind, K, nch, flags, taps)
    blob, pre, open_ = case.save()
    assert api.blob_info(blob).record_bytes > 100 * SP_CHUNK
    assert_in_flight(open_, nch, [8, 100, 150, 200, 256])
    rng = np.random.default_rng(3)
    others = [(rng.integers(0, 256, size=len(case.sig[0]), dtype=np.uint8) if kind == "u8" else
               rng.integers(-900, 900, size=case.sig[0].shape, dtype=np.int16) if kind == "cs16" else
               (rng.standard_normal(len(case.sig[0])) * 0.01).astype(np.float32)) for _ in range(2)]
    others = [others[0], others[1], None]
    got = case.cont(make(kind, K, nch, T, flags, taps)[0], T, dst, blob, pre, others=others)
    case.check(got)
    twin = case.cont(make(kind, K, nch, T, flags, taps)[0], T, dst, blob, pre, load=False, others=others)
    assert got["others"] == twin["others"], "the target's other streams changed"


# ------------------------------------------------------------------ a thousand records in one call

def test_many_records():
    """1000 streams x 8 channels saved in a permuted order and loaded, by the same list, into a second context: every
    stream continues as the unmoved reference"""
    kind, K, nch, S = "cs16", 160, 8, 1000
    fd = freqs(kind, K, nch)
    rng = np.random.default_rng(1000)
    pool = rng.integers(-2000, 2000, size=(S * 613 + 40000, 2), dtype=np.int16)
    sig = [pool[s * 613:s * 613 + 40000] for s in range(S)]
    sched = [[int(x) for x in rng.integers(0, 10000, size=S)] for _ in range(4)]
    perm = [int(x) for x in rng.permutation(S)]

    def ctx():
        c = api.Context(K, S, nch, 1, flags=FLAG_CS16 | DECODE | LEVEL)
        for s in range(S):
            c.set_plan_cs16(s, fd, 0)
        return c

    def run(c, subs, off=None):
        """each stream's own new rows of every submit"""
        f = Feed(c, kind, K, sig)
        if off:
            f.off = off
        env = []
        for cnt in subs:
            f.submit(cnt)
            dm = c.read_dm(int(max(f.rows)))
            env.append([dm[s, :int(f.rows[s])].copy() for s in range(S)])
        return f, env

    ref = ctx()
    _, env_ref = run(ref, sched)
    ref.sync()
    src = ctx()
    f, _ = run(src, sched[:2])
    blob = src.save_streams(perm)
    assert api.blob_info(blob).count == S
    src.close()
    tgt = ctx()
    tgt.load_streams(perm, blob)
    _, env = run(tgt, sched[2:], off=f.off)
    tgt.sync()
    for i, (a, b) in enumerate(zip(env, env_ref[2:])):
        bad = [s for s in range(S) if not np.array_equal(a[s].view(np.uint32), b[s].view(np.uint32))]
        assert not bad, (i, bad[:10])
    assert [states(tgt, s, nch) for s in range(S)] == [states(ref, s, nch) for s in range(S)]
    assert np.array_equal(tgt.decode_stats(), ref.decode_stats())
    (ti, tc), (ri, rc) = tgt.level_stats(), ref.level_stats()
    assert ti.tobytes() == ri.tobytes() and tc.tobytes() == rc.tobytes()
    tgt.close()
    ref.close()


# ------------------------------------------------------------------ channel splits that cut groups and tiles

# (kind, K, flags, taps): every form, its table kind
FORMS20 = [("u8", 160, 0, 2 * 160 + 48), ("u8", 160, FC, 0), ("u8", 160, FF, 2 * 160 + 48), ("u8", 160, FW, 0),
           ("cs16", 160, FW, 2 * 160 + 48), ("real", 200, 0, 0), ("real", 200, FC, 0), ("real", 200, FWR, 0)]
FORMS300 = [("u8", 1600, 0, 2 * 1600 + 3), ("u8", 1600, FW, 0), ("real", 800, FC, 0)]
# and one part of all 300 channels: a part whose own wideband plan has two tiles
SPLITS = [(k, K, f, t, 20, 3) for k, K, f, t in FORMS20] + [(k, K, f, t, 300, p) for k, K, f, t in FORMS300 for p in (2, 3)] + \
    [("u8", 1600, FW, 0, 300, 1)]


def part_starts(nch, parts):
    """acb_multi_create's split: the first channel of every part but the first"""
    base, extra = divmod(nch, parts)
    out, c = [], 0
    for i in range(parts - 1):
        c += base + (i < extra)
        out.append(c)
    return out


def test_split_shapes():
    assert part_starts(20, 3) == [7, 14] and part_starts(300, 2) == [150] and part_starts(300, 3) == [100, 200]
    assert [b % CH_GROUP for b in part_starts(20, 3)] == [7, 6]            # inside group 0 and group 1
    assert [b % CH_GROUP for b in part_starts(300, 3)] == [4, 0] and 100 // CH_GROUP != 99 // CH_GROUP + 1
    assert -(-300 // WB_CTILE) == 2 and -(-150 // WB_CTILE) == 1            # the full blob's two tiles, one per part
    assert part_starts(300, 1) == []                                        # a single part of two tiles


@pytest.mark.parametrize("kind,K,flags,taps,nch,parts", SPLITS)
def test_channel_split_moves(kind, K, flags, taps, nch, parts):
    """A channel split's blob is the single context's but for the envelope level sums; the moved stream continues bit
    for bit single -> split, split -> single, split -> a split of another part count, and split -> stream split"""
    case = Case(kind, K, nch, flags, taps)
    blob1, pre, open_ = case.save()
    assert_in_flight(open_, nch, part_starts(nch, parts))
    blobp, pre_p, _ = case.save(parts)
    assert pre_p == pre
    assert without_level_sums(blobp, nch) == without_level_sums(blob1, nch)
    other = 2 if parts != 2 else 3
    for tgt, src_blob, split in ((make(kind, K, nch, 2, flags, taps, parts)[0], blob1, True),
                                 (make(kind, K, nch, 2, flags, taps)[0], blobp, True),
                                 (make(kind, K, nch, 2, flags, taps, other)[0], blobp, True),
                                 (make(kind, K, nch, 2, flags, taps, 2, mode=0)[0], blobp, True)):
        case.check(case.cont(tgt, 2, SRC, src_blob, pre), chan_split=split)


@pytest.mark.parametrize("kind", ["u8", "cs16"])
def test_channel_split_moves_across_devices(kind):
    """300 channels over parts on devices 0 and 1"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: the move across devices needs two")
    K, nch = 1600, 300
    flags, taps = (FW, 0) if kind == "u8" else (FW, 2 * 1600 + 3)
    case = Case(kind, K, nch, flags, taps)
    blob1, pre, _ = case.save()
    fl = flags | kflag(kind) | DECODE | LEVEL
    for mode in (1, 0):
        m = api.MultiContext(K, 2, nch, 2, [0, 1], mode=mode, flags=fl, taps=taps)
        for s in range(2):
            plan(m, kind, s, freqs(kind, K, nch))
        case.check(case.cont(m, 2, SRC, blob1, pre), chan_split=True)
