"""Independent receivers: the ragged submits (a count per stream) and acb_reset_stream.

The rule: stream s of a context fed ragged submits gives exactly what a one-stream context of the same configuration
gives when it is fed only stream s's samples with the same cuts (a zero count being no call at all).  That is every
envelope row the stream produced, every message field in order, every chain state and, with ACB_FLAG_DECODE_STATS, every
decode count.  The inputs carry frames that straddle the cuts, and one stream stalls (zero counts for several submits)
in the middle of its traffic."""
import numpy as np
import pytest

from acarsdec_b200 import api, sharding, synth
from common import msg_tuple

pytestmark = pytest.mark.gpu

FLAG_REAL, FLAG_CS16, DECODE_STATS = 2, 4, 256
FAST_CHANNELIZER, FAST_FILTER, FAST_FILTER_REAL, FAST_WIDEBAND, FAST_WIDEBAND_REAL = 8, 16, 32, 64, 128
NCH, MAXBLK = 4, 3
U8_FM = (131.525, 131.550, 131.725, 131.825)
REAL_FM = (131.400, 131.425, 131.450, 131.500)
CS16_FM = (130.000, 130.025, 130.050, 130.100)


U8 = ("u8", "u8g")              # u8g: u8 IQ at K % 8 != 0, the GENERIC form


def _K(kind):
    return 200 if kind == "real" else 164 if kind == "u8g" else 160


def _freqs(kind):
    K = _K(kind)
    if kind == "real":
        fd, fc, _ = api.air_plan(K * 12500, REAL_FM)
        return REAL_FM, fd, fc
    fm = U8_FM if kind in U8 else CS16_FM
    fd, _, fc = api.plan(K, fm)
    return fm, fd, fc


def _signal(kind, nstreams, n, seed):
    """Per stream: u8 (n*2,) bytes of whole blocks, float32 (n,), or int16 (n, 2)."""
    K = _K(kind)
    fm, fd, fc = _freqs(kind)
    out = []
    for s in range(nstreams):
        p = synth.make_plan(K, fm, fc, seconds=n / (K * 12500), seed=seed + 13 * s, msgs_per_chan_per_sec=14.0, text_len=(5, 20),
                            amp=(8.0, 14.0))
        if kind in U8:
            out.append(synth.render_blocks(p, 0, n // (1024 * K)).reshape(-1))
        elif kind == "real":
            out.append(synth.render_real(synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, bursts=p.bursts, seed=p.seed), 0, n))
        else:
            out.append(synth.render_cs16(p, 0, n))
    return out


def _make(kind, nstreams, flags, taps, wf_streams=()):
    K = _K(kind)
    _, fd, fc = _freqs(kind)
    kf = FLAG_REAL if kind == "real" else FLAG_CS16 if kind in ("cs16", "planar") else 0
    ctx = api.Context(K, nstreams, NCH, MAXBLK, flags=flags | kf, taps=taps)
    for s in range(nstreams):
        if kind in U8:
            ctx.set_plan_at(s, fd, fc)
        elif kind == "real":
            ctx.set_plan_air_at(s, fd, fc)
        else:
            ctx.set_plan_cs16(s, fd, 1 if kind == "planar" else 0, fc)
    for s in wf_streams:                               # a caller's table: that stream (and so the submit) runs EXACT
        t = taps or K
        if kind in U8:
            wf = api.build_wf_lp(K, t, U8_FM) if t > K else api.build_wf(K, U8_FM)
        elif kind == "real":
            wf = api.build_wf_air_lp(K * 12500, t, REAL_FM) if t > K else api.build_wf_air(K * 12500, REAL_FM)
        else:
            wf = api.build_wf_cs16_lp(0, K, t, fd, fc) if t > K else api.build_wf_cs16(0, K, fd, fc)
        ctx.set_wf(s % nstreams, wf)
    return ctx


class Dev:
    """Device copies of submits' inputs, kept until the end of the test (the input lifetime rule)."""

    def __init__(self):
        self.keep = []

    def put(self, a):
        import torch
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self.keep.append(t)
        return t


def _submit(ctx, kind, parts, counts, dev, store, stride_pad=0):
    """One ragged submit: parts[s] is stream s's slice (length counts[s]).  Returns per-stream rows (u8: blocks*1024)."""
    S = len(parts)
    K = _K(kind)
    if kind in U8:
        bb = 1024 * K * 2
        w = max(counts) * bb + stride_pad * 16
        buf = np.zeros((S, w), dtype=np.uint8)
        for s, p in enumerate(parts):
            buf[s, :len(p)] = p
        nblk = np.array(counts, dtype=np.int32)
        if dev:
            t = store.put(buf)
            ctx.submit_device(t.data_ptr(), 0, w, counts=nblk)
        else:
            ctx.submit_host(buf, counts=nblk)
        return nblk.astype(np.int64) * 1024
    w = max(counts) + stride_pad
    if kind == "real":
        buf = np.zeros((S, w), dtype=np.float32)
    else:
        buf = np.zeros((S, w, 2), dtype=np.int16)
    for s, p in enumerate(parts):
        buf[s, :len(p)] = p
    if dev:
        if kind == "planar":
            xi, xq = store.put(buf[..., 0]), store.put(buf[..., 1])
            return ctx.submit_tensor(xi, xq, counts=counts)
        return ctx.submit_tensor(store.put(buf), counts=counts)
    if kind == "real":
        return ctx.submit_real(buf, counts=counts)
    if kind == "cs16":
        return ctx.submit_cs16(buf, counts=counts)
    return ctx.submit_cs16_planar(np.ascontiguousarray(buf[..., 0]), np.ascontiguousarray(buf[..., 1]), counts=counts)


def _submit_one(ctx, kind, part, dev, store):
    """A lockstep submit of a one-stream context; returns its rows."""
    if kind in U8:
        nblk = len(part) // (1024 * _K(kind) * 2)
        if dev:
            t = store.put(part[None])
            ctx.submit_device(t.data_ptr(), nblk, len(part))
        else:
            ctx.submit_host(np.ascontiguousarray(part[None]), nblk)
        return nblk * 1024
    if dev:
        if kind == "planar":
            return ctx.submit_tensor(store.put(part[None, :, 0]), store.put(part[None, :, 1]))
        return ctx.submit_tensor(store.put(part[None]))
    if kind == "real":
        return ctx.submit_real(np.ascontiguousarray(part[None]))
    if kind == "cs16":
        return ctx.submit_cs16(np.ascontiguousarray(part[None]))
    return ctx.submit_cs16_planar(np.ascontiguousarray(part[None, :, 0]), np.ascontiguousarray(part[None, :, 1]))


def _schedule(kind, nstreams, nsub, rng, stall=1):
    """Per submit, per stream counts (u8: blocks; else samples); stream `stall` stalls for three submits mid-run."""
    K = _K(kind)
    sched = []
    for i in range(nsub):
        if kind in U8:
            c = [int(rng.integers(0, MAXBLK + 1)) for _ in range(nstreams)]
        else:
            c = [int(rng.choice([0, rng.integers(1, K), rng.integers(K, 3000), rng.integers(3000, MAXBLK * 1024 * K - K)],
                                p=[0.15, 0.1, 0.1, 0.65])) for _ in range(nstreams)]
        if 2 <= i < 5:
            c[stall] = 0
        if max(c) == 0:
            c[0] = 1
        sched.append(c)
    return sched


def _unit(kind):
    return 1024 * _K(kind) * 2 if kind in U8 else 1


def _run_multi(kind, ctx, sig, sched, devmode, store, read_env=True):
    """Feed the schedule; returns per-stream envelope rows (concatenated), messages, nout per submit."""
    S = len(sig)
    u = _unit(kind)
    off = [0] * S
    env = [[] for _ in range(S)]
    for i, counts in enumerate(sched):
        parts = [sig[s][off[s] * (u if kind in U8 else 1):(off[s] + counts[s]) * (u if kind in U8 else 1)] for s in range(S)]
        dev = devmode == "dev" or (devmode == "mix" and i % 2 == 1)
        rows = _submit(ctx, kind, parts, counts, dev, store, stride_pad=3)
        if read_env:
            dm = ctx.read_dm(int(max(rows)))
            for s in range(S):
                env[s].append(dm[s, :int(rows[s])])
        for s in range(S):
            off[s] += counts[s]
    ctx.sync()
    return [np.concatenate(e) if e else np.zeros((0, NCH), np.float32) for e in env], ctx.drain()


def _run_single(kind, flags, taps, sig_s, counts_s, devmode, store, wf=False, read_env=True):
    ctx = _make(kind, 1, flags, taps, wf_streams=(0,) if wf else ())
    u = _unit(kind) if kind in U8 else 1
    off, env = 0, []
    for i, c in enumerate(counts_s):
        if c == 0:
            continue
        dev = devmode == "dev" or (devmode == "mix" and i % 2 == 1)
        rows = _submit_one(ctx, kind, sig_s[off * u:(off + c) * u], dev, store)
        if read_env:
            env.append(ctx.read_dm(int(rows))[0])
        off += c
    ctx.sync()
    msgs = ctx.drain()
    states = [bytes(ctx.get_state(0, ch)) for ch in range(NCH)]
    stats = ctx.decode_stats() if flags & DECODE_STATS else None
    ctx.close()
    return (np.concatenate(env) if env else np.zeros((0, NCH), np.float32)), msgs, states, stats


def _full(m):
    return msg_tuple(m) + (m.pos, m.block, m.soh_pos)


def _check_against_single(kind, flags, taps, S, sig, sched, ctx, env, msgs, devmode, store, wf_streams=()):
    stats = ctx.decode_stats() if flags & DECODE_STATS else None
    for s in range(S):
        e1, m1, st1, ds1 = _run_single(kind, flags, taps, sig[s], [c[s] for c in sched], devmode, store, wf=s in wf_streams)
        assert env[s].shape == e1.shape and np.array_equal(env[s].view(np.uint32), e1.view(np.uint32)), f"stream {s}: envelope"
        mine = [_full(m) for m in msgs if m.stream == s]
        assert mine == [_full(m) for m in m1], f"stream {s}: messages"
        assert [bytes(ctx.get_state(s, ch)) for ch in range(NCH)] == st1, f"stream {s}: chain states"
        if stats is not None:
            assert np.array_equal(stats[s], ds1[0]), f"stream {s}: decode statistics"


# (kind, flags, taps, streams given their own table): every channelizer form of the kind
FORMS = {
    "u8": [(0, 0, ()), (FAST_CHANNELIZER, 0, ()), (FAST_FILTER, 2 * 160 + 48, ()), (FAST_WIDEBAND, 0, ()),
           (FAST_WIDEBAND, 2 * 160 + 48, ()), (0, 2 * 160 + 48, ()), (FAST_CHANNELIZER, 0, (2,)), (DECODE_STATS, 0, ())],
    "u8g": [(0, 2 * 164 + 40, ()), (DECODE_STATS, 2 * 164 + 40, ())],
    "real": [(0, 0, ()), (FAST_CHANNELIZER, 0, ()), (FAST_FILTER_REAL, 2 * 200 + 40, ()), (FAST_WIDEBAND_REAL, 0, ()),
             (FAST_WIDEBAND_REAL, 2 * 200 + 40, ()), (0, 2 * 200 + 40, ()), (DECODE_STATS | FAST_CHANNELIZER, 0, ())],
    "cs16": [(0, 0, ()), (FAST_CHANNELIZER, 0, ()), (FAST_FILTER, 2 * 160 + 48, ()), (FAST_WIDEBAND, 2 * 160 + 48, ()),
             (0, 2 * 160 + 48, ()), (FAST_CHANNELIZER, 0, (1,)), (DECODE_STATS | FAST_FILTER, 2 * 160 + 48, ())],
    "planar": [(0, 0, ()), (FAST_WIDEBAND, 0, ()), (FAST_FILTER | DECODE_STATS, 2 * 160 + 48, ())],
}
CASES = [(k, *f, d) for k, fs in FORMS.items() for f in fs for d in ("host", "dev", "mix")]


@pytest.mark.parametrize("kind,flags,taps,wf_streams,devmode", CASES)
def test_ragged_matches_one_stream_contexts(kind, flags, taps, wf_streams, devmode):
    rng = np.random.default_rng(abs(hash((kind, flags, taps, devmode))) % 2**32)
    S = int(rng.integers(5, 8))
    nsub = 10
    sched = _schedule(kind, S, nsub, rng)
    n = [sum(c[s] for c in sched) for s in range(S)]
    length = max(n) * (1024 * _K(kind) if kind in U8 else 1)
    sig = _signal(kind, S, max(length, 1024 * _K(kind)), seed=int(rng.integers(1 << 20)))
    store = Dev()
    # a caller's table runs the context's submits on EXACT: every stream gets one, as its one-stream context does
    wf_streams = tuple(range(S)) if wf_streams else ()
    ctx = _make(kind, S, flags, taps, wf_streams)
    env, msgs = _run_multi(kind, ctx, sig, sched, devmode, store)
    assert sum(len(e) for e in env) > 0 and len(msgs) > 0
    _check_against_single(kind, flags, taps, S, sig, sched, ctx, env, msgs, devmode, store, wf_streams)
    ctx.close()


@pytest.mark.parametrize("kind", ["u8", "real", "cs16", "planar"])
def test_equal_counts_are_the_lockstep_call(kind):
    rng = np.random.default_rng(5)
    S = 6
    K = _K(kind)
    sig = _signal(kind, S, 6 * 1024 * K, seed=99)
    cuts = [1, 2, 1, 2] if kind in U8 else [5000, 1024 * K + 17, 333, 2 * 1024 * K - 2 * K]
    out = []
    for ragged in (False, True):
        ctx = _make(kind, S, 0, 0)
        off, envs = 0, []
        for c in cuts:
            u = _unit(kind)
            part = np.stack([x[off * u:(off + c) * u] for x in sig])
            if ragged:
                rows = _submit(ctx, kind, list(part), [c] * S, False, None)
                nsamp = int(rows[0])
            elif kind in U8:
                ctx.submit_host(part, c)
                nsamp = c * 1024
            elif kind == "real":
                nsamp = ctx.submit_real(part)
            elif kind == "cs16":
                nsamp = ctx.submit_cs16(part)
            else:
                nsamp = ctx.submit_cs16_planar(np.ascontiguousarray(part[..., 0]), np.ascontiguousarray(part[..., 1]))
            envs.append(ctx.read_dm(nsamp))
            off += c
        ctx.sync()
        out.append((envs, [(m.stream,) + _full(m) for m in ctx.drain()], ctx.stats().kernel_launches))
        ctx.close()
    (e0, m0, k0), (e1, m1, k1) = out
    assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(e0, e1))
    assert m0 == m1 and len(m0) > 0
    assert k0 == k1                                     # the same kernels: equal counts take the lockstep path


@pytest.mark.parametrize("kind,unit,period", [("u8", None, 0), ("cs16", 0, 0), ("cs16", 1, 1024), ("real", 2, 65536),
                                              ("real", 2, 150)])
def test_drained_order_follows_the_emission_key(kind, unit, period):
    """Across streams at different positions the drained sequence of each submit is sorted by (group number counted
    from the stream's own start, stream, channel, time)."""
    rng = np.random.default_rng(17)
    S = 6
    K = _K(kind)
    sched = _schedule(kind, S, 8, rng)
    length = max(sum(c[s] for c in sched) for s in range(S)) * (1024 * K if kind in U8 else 1)
    sig = _signal(kind, S, max(length, 1024 * K), seed=123)
    ctx = _make(kind, S, 0, 0)
    if unit is not None:
        ctx.set_emission_groups(unit, period)
    store = Dev()
    u = _unit(kind)
    off = [0] * S
    nmsg = 0
    for i, counts in enumerate(sched):
        if i == 4:
            ctx.reset_stream(2)                          # one stream starts again at position 0
        parts = [sig[s][off[s] * u:(off[s] + counts[s]) * u] for s in range(S)]
        _submit(ctx, kind, parts, counts, False, store)
        off = [o + c for o, c in zip(off, counts)]
        ctx.sync()
        got = ctx.drain()
        nmsg += len(got)
        key = [(sharding.group_number(unit if kind not in U8 else None, period, K, m.pos), m.stream, m.chn, m.pos) for m in got]
        assert key == sorted(key), f"submit {i}"
    assert nmsg > 0
    ctx.close()


@pytest.mark.parametrize("kind,flags,taps", [("u8", 0, 2 * 160 + 48), ("u8", FAST_FILTER, 2 * 160 + 48), ("u8g", 0, 2 * 164 + 40),
                                             ("u8g", DECODE_STATS, 2 * 164 + 40), ("u8", FAST_WIDEBAND | DECODE_STATS, 2 * 160 + 48),
                                             ("cs16", 0, 0),
                                             ("cs16", FAST_WIDEBAND | DECODE_STATS, 2 * 160 + 48), ("real", FAST_FILTER_REAL, 440)])
def test_reset_stream(kind, flags, taps):
    """Stream 1 is retuned and reset mid-run: the other streams match the run without the reset, and stream 1 matches a
    fresh one-stream context (planned the new way) fed from that point."""
    rng = np.random.default_rng(23)
    S, nsub, at = 5, 7, 3
    K = _K(kind)
    sched = _schedule(kind, S, nsub, rng, stall=3)
    length = max(sum(c[s] for c in sched) for s in range(S)) * (1024 * K if kind in U8 else 1)
    sig = _signal(kind, S, max(length, 1024 * K), seed=77)
    u = _unit(kind)
    fm, fd, fc = _freqs(kind)
    fd2 = list(fd[::-1])                                 # the retune: the same channels in the other order

    def plan2(ctx, s):
        if kind in U8:
            ctx.set_plan_at(s, fd2, fc)
        elif kind == "real":
            ctx.set_plan_air_at(s, fd2, fc)
        else:
            ctx.set_plan_cs16(s, fd2, 0, fc)

    results = []
    for do_reset in (False, True):
        ctx = _make(kind, S, flags, taps)
        off = [0] * S
        env = [[] for _ in range(S)]
        for i, counts in enumerate(sched):
            if do_reset and i == at:
                plan2(ctx, 1)
                ctx.reset_stream(1)
            parts = [sig[s][off[s] * u:(off[s] + counts[s]) * u] for s in range(S)]
            rows = _submit(ctx, kind, parts, counts, False, None)
            dm = ctx.read_dm(int(max(rows)))
            for s in range(S):
                if i >= at:
                    env[s].append(dm[s, :int(rows[s])])
            off = [o + c for o, c in zip(off, counts)]
        ctx.sync()
        msgs = ctx.drain()
        states = {s: [bytes(ctx.get_state(s, ch)) for ch in range(NCH)] for s in range(S)}
        stats = ctx.decode_stats() if flags & DECODE_STATS else None
        results.append((env, msgs, states, stats))
        ctx.close()
    (e0, m0, st0, ds0), (e1, m1, st1, ds1) = results
    for s in (0, 2, 3, 4):
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(e0[s], e1[s])), f"stream {s}"
        assert [_full(m) for m in m0 if m.stream == s] == [_full(m) for m in m1 if m.stream == s]
        assert st0[s] == st1[s]
        if ds0 is not None:
            assert np.array_equal(ds0[s], ds1[s])
    # stream 1 after the reset: a fresh context with the new plan, fed from submit `at` on
    ctx1 = api.Context(K, 1, NCH, MAXBLK, flags=flags | (FLAG_REAL if kind == "real" else FLAG_CS16 if kind not in U8 else 0), taps=taps)
    plan2(ctx1, 0)
    start = sum(c[1] for c in sched[:at])
    off, env = start, []
    for counts in sched[at:]:
        c = counts[1]
        if c == 0:
            continue
        rows = _submit_one(ctx1, kind, sig[1][off * u:(off + c) * u], False, None)
        env.append(ctx1.read_dm(int(rows))[0])
        off += c
    ctx1.sync()
    want = ctx1.drain()
    e_reset = np.concatenate(e1[1])
    assert np.array_equal(e_reset.view(np.uint32), np.concatenate(env).view(np.uint32))
    # messages of stream 1 completed after the reset (frames in flight at the reset were still delivered, from before)
    got = [_full(m) for m in m1 if m.stream == 1]
    assert got[len(got) - len(want):] == [_full(m) for m in want]
    assert st1[1] == [bytes(ctx1.get_state(0, ch)) for ch in range(NCH)]
    if ds1 is not None:
        assert np.array_equal(ds1[1], ctx1.decode_stats()[0])
    ctx1.close()


@pytest.mark.parametrize("kind", ["u8", "real", "cs16", "planar"])
def test_refusals_read_nothing_and_keep_the_carry(kind):
    """Every refusal, then the next submit: the run matches the run without the refused calls."""
    rng = np.random.default_rng(31)
    S = 5
    K = _K(kind)
    sched = _schedule(kind, S, 6, rng)
    length = max(sum(c[s] for c in sched) for s in range(S)) * (1024 * K if kind in U8 else 1)
    sig = _signal(kind, S, max(length, 1024 * K), seed=5)
    u = _unit(kind)
    runs = []
    for refuse in (False, True):
        ctx = _make(kind, S, 0, 0)
        lib, h = ctx.lib, ctx.h
        off = [0] * S
        for i, counts in enumerate(sched):
            if refuse and i == 2:
                z = np.zeros(S, dtype=np.int32 if kind in U8 else np.uint64)
                big = z.copy()
                big[1] = MAXBLK + 1 if kind in U8 else MAXBLK * 1024 * K + K
                neg = np.zeros(S, dtype=np.int32)
                neg[0] = -1
                buf = np.zeros(1 << 24, dtype=np.uint8)
                p = buf.ctypes.data
                if kind in U8:
                    bb = 1024 * K * 2
                    two = np.full(S, 2, dtype=np.int32)
                    assert lib.acb_submit_host_ragged(h, p, bb, z.ctypes.data) == -1                  # every count 0
                    assert lib.acb_submit_host_ragged(h, p, bb, big.ctypes.data) == -1                # above the cap
                    assert lib.acb_submit_host_ragged(h, p, bb, neg.ctypes.data) == -1                # negative
                    assert lib.acb_submit_host_ragged(h, p, bb, two.ctypes.data) == -1                # stride < largest
                    assert lib.acb_submit_host_ragged(h, p, bb + 8, np.ones(S, np.int32).ctypes.data) == -1   # stride % 16
                    assert lib.acb_submit_real_host_ragged(h, p, 100, z.ctypes.data, None) == -1     # wrong kind
                else:
                    fn = lib.acb_submit_real_host_ragged if kind == "real" else lib.acb_submit_cs16_host_ragged
                    other = lib.acb_submit_cs16_host_ragged if kind == "real" else lib.acb_submit_real_host_ragged
                    ok = np.full(S, 100, dtype=np.uint64)
                    assert fn(h, p, 1000, z.ctypes.data, None) == -1                                  # every count 0
                    assert fn(h, p, MAXBLK * 1024 * K + K, big.ctypes.data, None) == -1              # above the cap
                    assert fn(h, p, 50, ok.ctypes.data, None) == -1                                   # stride < largest
                    assert other(h, p, 1000, ok.ctypes.data, None) == -1                              # wrong kind
                    assert lib.acb_submit_host_ragged(h, p, 1 << 20, np.ones(S, np.int32).ctypes.data) == -1
                    assert lib.acb_submit_cs16_device_ragged(h, p, 1000, ok.ctypes.data, None) == -1  # host memory
            parts = [sig[s][off[s] * u:(off[s] + counts[s]) * u] for s in range(S)]
            _submit(ctx, kind, parts, counts, False, None)
            off = [o + c for o, c in zip(off, counts)]
        ctx.sync()
        runs.append(([_full(m) + (m.stream,) for m in ctx.drain()],
                     [bytes(ctx.get_state(s, ch)) for s in range(S) for ch in range(NCH)]))
        ctx.close()
    assert runs[0] == runs[1] and len(runs[0][0]) > 0


def test_input_lifetime_under_ragged_submits():
    """Device and pinned inputs rotated through three buffers, each overwritten as soon as the rule frees it (when
    submit N+2 has returned, or a collect covered it): the result is the one fresh buffers give."""
    kind, S = "cs16", 5
    K = _K(kind)
    rng = np.random.default_rng(41)
    sched = _schedule(kind, S, 9, rng)
    for c in sched:
        c[0] = max(c[0], 2 * K)                         # every submit produces rows: one collect covers one submit
    length = max(sum(c[s] for c in sched) for s in range(S))
    sig = _signal(kind, S, max(length, 1024 * K), seed=8)
    import torch
    results = []
    for reuse in (False, True):
        ctx = _make(kind, S, 0, 0)
        w = MAXBLK * 1024 * K
        bufs = [torch.zeros((S, w, 2), dtype=torch.int16, device="cuda") for _ in range(3)]
        off = [0] * S
        for i, counts in enumerate(sched):
            b = bufs[i % 3] if reuse else torch.zeros((S, w, 2), dtype=torch.int16, device="cuda")
            if not reuse:
                bufs.append(b)
            for s in range(S):
                b[s, :counts[s]] = torch.from_numpy(np.ascontiguousarray(sig[s][off[s]:off[s] + counts[s]])).cuda()
            torch.cuda.synchronize()
            ctx.submit_tensor(b, counts=counts)
            if reuse and i >= 1:
                ctx.collect()                            # covers submit i-1: its buffer may be refilled next time round
            off = [o + c for o, c in zip(off, counts)]
        ctx.sync()
        results.append([_full(m) + (m.stream,) for m in ctx.drain()])
        ctx.close()
    assert results[0] == results[1] and len(results[0]) > 0


def test_thousands_of_streams():
    """2112 streams x 8 channels of CS16 with ragged counts (a tenth of them stalled): a sample of streams matches
    one-stream contexts."""
    S, nch, K, nsub, cmax = 2112, 8, 160, 5, 120000
    fm = (130.000, 130.025, 130.050, 130.100, 130.125, 130.150, 130.200, 130.250)
    fd, _, fc = api.plan(K, fm)
    base = []
    for j in range(4):
        p = synth.make_plan(K, fm, fc, seconds=nsub * cmax / (K * 12500), seed=300 + j, msgs_per_chan_per_sec=20.0,
                            text_len=(5, 20), amp=(8.0, 14.0))
        base.append(synth.render_cs16(p, 0, nsub * cmax))
    rng = np.random.default_rng(3)
    ctx = api.Context(K, S, nch, 1, flags=FLAG_CS16 | FAST_CHANNELIZER)
    for s in range(S):
        ctx.set_plan_cs16(s, fd, 0, fc)
    sched = []
    for i in range(nsub):
        c = rng.integers(cmax // 2, cmax, size=S)
        c[rng.random(S) < 0.1] = 0
        sched.append(c)
    off = np.zeros(S, dtype=np.int64)
    sample = [0, 1, 7, 500, 1501, S - 1]
    env = {s: [] for s in sample}
    buf = np.zeros((S, cmax, 2), dtype=np.int16)
    for counts in sched:
        for s in range(S):
            buf[s, :counts[s]] = base[s % 4][off[s]:off[s] + counts[s]]
        rows = ctx.submit_cs16(buf, counts=counts)
        dm = ctx.read_dm(int(rows.max()))
        for s in sample:
            env[s].append(dm[s, :rows[s]])
        off += counts
    ctx.sync()
    msgs = ctx.drain()
    assert len(msgs) > 0
    for s in sample:
        c1 = api.Context(K, 1, nch, 1, flags=FLAG_CS16 | FAST_CHANNELIZER)
        c1.set_plan_cs16(0, fd, 0, fc)
        o, e1 = 0, []
        for counts in sched:
            if counts[s]:
                r = c1.submit_cs16(np.ascontiguousarray(base[s % 4][None, o:o + counts[s]]))
                e1.append(c1.read_dm(r)[0])
                o += counts[s]
        c1.sync()
        assert np.array_equal(np.concatenate(env[s]).view(np.uint32), np.concatenate(e1).view(np.uint32)), f"stream {s}"
        assert [_full(m) for m in msgs if m.stream == s] == [_full(m) for m in c1.drain()], f"stream {s}"
        c1.close()
    ctx.close()


def test_generic_stream_that_starts_late():
    """GENERIC u8 at taps > K: streams 0 and 3 bring no block in the first submits, so the others are ahead of them when
    their first rows (whose window reaches before their start) are computed."""
    kind, S, taps = "u8g", 5, 2 * 164 + 40
    sched = [[0, 2, 1, 0, 3], [0, 1, 2, 0, 1], [1, 3, 0, 2, 2], [2, 0, 3, 1, 1], [3, 1, 1, 3, 0]]
    length = max(sum(c[s] for c in sched) for s in range(S)) * 1024 * _K(kind)
    sig = _signal(kind, S, length, seed=61)
    store = Dev()
    ctx = _make(kind, S, DECODE_STATS, taps)
    env, msgs = _run_multi(kind, ctx, sig, sched, "host", store)
    _check_against_single(kind, DECODE_STATS, taps, S, sig, sched, ctx, env, msgs, "host", store)
    ctx.close()


@pytest.mark.parametrize("kind", ["u8", "real", "cs16", "planar"])
@pytest.mark.parametrize("mode", [0, 1])
def test_multi_context_matches_one_context(kind, mode):
    """acb_multi_*_ragged over two contexts on one GPU, split by streams (mode 0) or channels (mode 1), with a
    acb_multi_reset_stream mid-run: the merged messages and every chain state are those of one context."""
    rng = np.random.default_rng(71 + mode)
    S = 5
    K = _K(kind)
    sched = _schedule(kind, S, 7, rng)
    for c in sched[:2]:
        c[3] = c[4] = 0                                  # the second part of a stream split sits these out
        c[0] = max(c[0], 1)
    length = max(sum(c[s] for c in sched) for s in range(S)) * (1024 * K if kind in U8 else 1)
    sig = _signal(kind, S, max(length, 1024 * K), seed=19)
    _, fd, fc = _freqs(kind)
    kf = FLAG_REAL if kind == "real" else FLAG_CS16 if kind in ("cs16", "planar") else 0
    u = _unit(kind)
    out = []
    for multi in (False, True):
        ctx = api.MultiContext(K, S, NCH, MAXBLK, [0, 0], mode=mode, flags=kf) if multi else _make(kind, S, 0, 0)
        if multi:
            for s in range(S):
                if kind in U8:
                    ctx.set_plan(s, fd)
                elif kind == "real":
                    ctx.set_plan_air(s, fd)
                else:
                    ctx.set_plan_cs16(s, fd, 1 if kind == "planar" else 0, fc)
        off = [0] * S
        rows_all = []
        for i, counts in enumerate(sched):
            if i == 4:
                ctx.reset_stream(2)
            parts = [sig[s][off[s] * u:(off[s] + counts[s]) * u] for s in range(S)]
            w = max(counts)
            if kind in U8:
                buf = np.zeros((S, w * u), dtype=np.uint8)
            elif kind == "real":
                buf = np.zeros((S, w), dtype=np.float32)
            else:
                buf = np.zeros((S, w, 2), dtype=np.int16)
            for s, p in enumerate(parts):
                buf[s, :len(p)] = p
            if kind in U8:
                ctx.submit_host(buf, counts=counts)
            elif kind == "real":
                rows_all.append(list(ctx.submit_real(buf, counts=counts)))
            elif kind == "cs16":
                rows_all.append(list(ctx.submit_cs16(buf, counts=counts)))
            else:
                rows_all.append(list(ctx.submit_cs16_planar(np.ascontiguousarray(buf[..., 0]), np.ascontiguousarray(buf[..., 1]),
                                                             counts=counts)))
            off = [o + c for o, c in zip(off, counts)]
            if i % 3 == 2:
                ctx.collect()
        ctx.sync()
        out.append(([(m.stream,) + _full(m) for m in ctx.drain()], rows_all,
                    [bytes(ctx.get_state(s, ch)) for s in range(S) for ch in range(NCH)]))
        ctx.close()
    assert out[0][0] == out[1][0] and len(out[0][0]) > 0
    assert out[0][1] == out[1][1]
    assert out[0][2] == out[1][2]
