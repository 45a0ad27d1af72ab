"""Input and envelope levels on the device (ACB_FLAG_LEVEL_STATS: k_level_in, k_level_dm) against the float64
definition (tests/level_stats_refs.py): every input kind, host and device submits, taps = K and taps > K, every
channelizer form, lockstep and ragged counts, envelope input, cut independence, determinism, the flag's absence,
coverage and resets, and several contexts (acb_multi_*)."""
import copy
import zlib

import numpy as np
import pytest

import level_stats_refs as lr
import test_gpu_ragged as rg
from acarsdec_b200 import api
from common import msg_tuple

pytestmark = pytest.mark.gpu

LEVEL = api.FLAG_LEVEL_STATS
NCH, MAXBLK = rg.NCH, rg.MAXBLK
BASE = {"u8": "u8", "u8g": "u8", "cs16": "cs16", "planar": "cs16", "real": "real"}
FC, FF, FFR, FW, FWR = 8, 16, 32, 64, 128


def _taps(kind):
    return {"u8": 2 * 160 + 48, "u8g": 2 * 164 + 40, "cs16": 2 * 160 + 48, "planar": 2 * 160 + 48, "real": 2 * 200 + 40}[kind]


# (kind, form): the flags that select it at taps = K and at taps > K
FORMS = {
    "u8": {"exact": 0, "fast": FC | FF, "wb": FW},
    "u8g": {"generic": 0},
    "cs16": {"exact": 0, "fast": FC | FF, "wb": FW},
    "planar": {"exact": 0, "fast": FC | FF, "wb": FW},
    "real": {"exact": 0, "fast": FC | FFR, "wb": FWR},
}
CASES = [(k, f, t, c) for k, fs in FORMS.items() for f in fs for t in ("K", "long") for c in ("lockstep", "ragged")]


def _inject(kind, sig, rng):
    """full-scale codes (and codes just inside full scale) at random places of every stream"""
    out = []
    for x in sig:
        x = x.copy()
        n = len(x)
        pos = rng.choice(n, size=max(8, n // 2000), replace=False)
        if BASE[kind] == "u8":
            x[pos] = rng.choice(np.array([0, 255, 1, 254], np.uint8), size=len(pos))
        elif BASE[kind] == "cs16":
            comp = rng.integers(0, 2, size=len(pos))
            x[pos, comp] = rng.choice(np.array([-32768, 32767, -32767, 32766], np.int16), size=len(pos))
        else:
            x[pos] = rng.choice(np.array([-1.0, 1.0, 2047 / 2048, -2047 / 2048, 2046 / 2048, -1.25], np.float32), size=len(pos))
        out.append(x)
    return out


def _samples(kind, part):
    """a submit's part of one stream as (n, 2) components (u8 / CS16) or (n,) real samples"""
    return part.reshape(-1, 2) if BASE[kind] == "u8" else part


def _lockstep(ctx, kind, parts, dev, store):
    """the lockstep calls (no counts): every part has the same length"""
    S, K = len(parts), rg._K(kind)
    buf = np.ascontiguousarray(np.stack(parts))
    if kind in rg.U8:
        nblk = buf.shape[1] // (1024 * K * 2)
        if dev:
            t = store.put(buf)
            ctx.submit_device(t.data_ptr(), nblk, buf.shape[1])
        else:
            ctx.submit_host(buf, nblk)
        return np.full(S, nblk * 1024)
    if dev:
        r = ctx.submit_tensor(store.put(buf[..., 0]), store.put(buf[..., 1])) if kind == "planar" else ctx.submit_tensor(store.put(buf))
    elif kind == "real":
        r = ctx.submit_real(buf)
    elif kind == "cs16":
        r = ctx.submit_cs16(buf)
    else:
        r = ctx.submit_cs16_planar(np.ascontiguousarray(buf[..., 0]), np.ascontiguousarray(buf[..., 1]))
    return np.full(S, r)


def _sched(kind, S, nsub, rng, ragged):
    """counts per submit; the first submit brings every stream at least one whole window (1024 rows)"""
    K = rg._K(kind)
    big = MAXBLK if kind in rg.U8 else int(rng.integers(1024 * K, MAXBLK * 1024 * K - K))
    if ragged:
        sched = rg._schedule(kind, S, nsub, rng)
        sched[0] = [big] * S if kind in rg.U8 else [int(rng.integers(1024 * K, MAXBLK * 1024 * K - K)) for _ in range(S)]
        return sched
    if kind in rg.U8:
        return [[big] * S] + [[int(rng.integers(1, MAXBLK + 1))] * S for _ in range(nsub - 1)]
    return [[big] * S] + [[int(rng.choice([rng.integers(1, K), rng.integers(K, 3000), rng.integers(3000, MAXBLK * 1024 * K - K)]))] * S
                          for _ in range(nsub - 1)]


class Refs:
    """the definition for every stream and chain of a context"""

    def __init__(self, kind, S):
        self.kind = kind
        self.inp = [lr.InputLevels(BASE[kind], rg._K(kind)) for _ in range(S)]
        self.ch = [[lr.ChanLevels() for _ in range(NCH)] for _ in range(S)]

    def feed(self, s, part, dm_rows):
        if part is not None:
            self.inp[s].feed(_samples(self.kind, part))
        for c in range(NCH):
            self.ch[s][c].feed(dm_rows[:, c])

    def reset_stream(self, s):
        self.inp[s] = lr.InputLevels(BASE[self.kind], rg._K(self.kind))
        self.ch[s] = [lr.ChanLevels() for _ in range(NCH)]

    def clear(self):
        for s in range(len(self.inp)):
            self.inp[s].clear()
            for c in self.ch[s]:
                c.clear()

    def check(self, inp, ch, streams=None, input_table=True):
        for s in range(len(self.inp)) if streams is None else streams:
            if input_table:
                lr.check_input(inp[s], self.inp[s])
            else:
                assert int(inp[s]["samples"]) == 0 and int(inp[s]["clipped"]) == 0 and float(inp[s]["power_sum"]) == 0.0
            for c in range(NCH):
                lr.check_chan(ch[s, c], self.ch[s][c])


def _feed(ctx, kind, sig, sched, ragged, store, refs=None, off=None):
    """run the schedule (host and device submits alternating); refs follow every submit's samples and envelope"""
    S = len(sig)
    u = rg._unit(kind)
    off = [0] * S if off is None else off
    for i, counts in enumerate(sched):
        parts = [sig[s][off[s] * u:(off[s] + counts[s]) * u] for s in range(S)]
        dev = i % 2 == 1
        rows = rg._submit(ctx, kind, parts, counts, dev, store, stride_pad=3) if ragged else _lockstep(ctx, kind, parts, dev, store)
        if refs is not None:
            dm = ctx.read_dm(int(max(rows)))
            for s in range(S):
                refs.feed(s, parts[s], dm[s, :int(rows[s])])
        for s in range(S):
            off[s] += counts[s]
    return off


def _signal(kind, S, sched, rng):
    n = max(sum(c[s] for c in sched) for s in range(S)) * (1024 * rg._K(kind) if kind in rg.U8 else 1)
    return _inject(kind, rg._signal(kind, S, max(n, 1024 * rg._K(kind)), seed=int(rng.integers(1 << 20))), rng)


@pytest.mark.parametrize("kind,form,taps,counts", CASES)
def test_levels_match_the_definition(kind, form, taps, counts):
    rng = np.random.default_rng(zlib.crc32(f"{kind}{form}{taps}{counts}".encode()))
    S, ragged = 3, counts == "ragged"
    sched = _sched(kind, S, 4, rng, ragged)
    sig = _signal(kind, S, sched, rng)
    store = rg.Dev()
    refs = Refs(kind, S)
    with rg._make(kind, S, LEVEL | FORMS[kind][form], _taps(kind) if taps == "long" else 0) as ctx:
        _feed(ctx, kind, sig, sched, ragged, store, refs)
        ctx.sync()
        inp, ch = ctx.level_stats()
        refs.check(inp, ch)
        assert inp["samples"].sum() > 0 and inp["clipped"].sum() > 0 and ch["windows"].sum() > 0


def test_envelope_input_fills_the_chain_table_only():
    rng = np.random.default_rng(7)
    S = 2
    refs = Refs("u8", S)
    with api.Context(160, S, NCH, MAXBLK, flags=LEVEL | 1) as ctx:          # NO_INPUT_STAGING: envelope input only
        for n in (700, 1500, 2048, 900):
            dm = (rng.random((S, n, NCH)) * rng.choice([0.5, 4.0])).astype(np.float32)
            ctx.submit_dm(dm)
            for s in range(S):
                refs.feed(s, None, dm[s])
        ctx.sync()
        inp, ch = ctx.level_stats()
    refs.check(inp, ch, input_table=False)


@pytest.mark.parametrize("kind", ["u8", "real", "cs16"])
def test_cut_independence(kind):
    """stream 0 fed in one submit, and the same samples in ragged cuts beside a busy stream 1"""
    rng = np.random.default_rng(11)
    K = rg._K(kind)
    total = MAXBLK if kind in rg.U8 else MAXBLK * 1024 * K - K
    cuts = [1, 2] if kind in rg.U8 else [total // 5, 2 * total // 5, total - total // 5 - 2 * total // 5]
    sched_b = [[c, int(rng.integers(1, MAXBLK + 1)) if kind in rg.U8 else int(rng.integers(K, total))] for c in cuts]
    sig = _signal(kind, 2, sched_b, rng)
    store = rg.Dev()
    with rg._make(kind, 1, LEVEL, 0) as a, rg._make(kind, 2, LEVEL, 0) as b:
        _feed(a, kind, sig[:1], [[total]], False, store)
        _feed(b, kind, sig, sched_b, True, store)
        a.sync()
        b.sync()
        ia, ca = a.level_stats()
        ib, cb = b.level_stats()
    for f in ("samples", "clipped", "peak"):
        assert ia[f][0] == ib[f][0], f
    for f in ("rows", "windows", "peak"):
        assert np.array_equal(ca[f][0], cb[f][0]), f
    assert np.allclose(ia["power_sum"][0], ib["power_sum"][0], rtol=1e-10, atol=0)
    for f in ("power_sum", "floor"):
        assert np.allclose(ca[f][0], cb[f][0], rtol=1e-10, atol=0), f


@pytest.mark.parametrize("kind", ["u8", "real", "planar"])
def test_same_inputs_same_bits(kind):
    rng = np.random.default_rng(5)
    sched = _sched(kind, 3, 4, rng, True)
    sig = _signal(kind, 3, sched, rng)
    store = rg.Dev()
    tabs = []
    for _ in range(2):
        with rg._make(kind, 3, LEVEL | FORMS[kind]["fast"], 0) as ctx:
            _feed(ctx, kind, sig, sched, True, store)
            ctx.sync()
            tabs.append(ctx.level_stats())
    assert tabs[0][0].tobytes() == tabs[1][0].tobytes() and tabs[0][1].tobytes() == tabs[1][1].tobytes()


@pytest.mark.parametrize("kind", ["u8", "real"])
def test_flag_changes_nothing_else(kind):
    rng = np.random.default_rng(3)
    S = 3
    sched = _sched(kind, S, 4, rng, True)
    sig = _signal(kind, S, sched, rng)
    store = rg.Dev()
    out = []
    for flags in (api.FLAG_DECODE_STATS, api.FLAG_DECODE_STATS | LEVEL):
        with rg._make(kind, S, flags | FORMS[kind]["fast"], 0) as ctx:
            env = []
            u, off = rg._unit(kind), [0] * S
            for i, counts in enumerate(sched):
                parts = [sig[s][off[s] * u:(off[s] + counts[s]) * u] for s in range(S)]
                rows = rg._submit(ctx, kind, parts, counts, i % 2 == 1, store)
                env.append(ctx.read_dm(int(max(rows))).copy())
                off = [off[s] + counts[s] for s in range(S)]
            ctx.sync()
            msgs = [msg_tuple(m) for m in ctx.drain()]
            states = [bytes(ctx.get_state(s, c)) for s in range(S) for c in range(NCH)]
            if not flags & LEVEL:
                lib = ctx.lib
                a = np.zeros(S, api.INPUT_LEVEL_DTYPE)
                assert lib.acb_get_level_stats(ctx.h, a.ctypes.data, S, None, 0, 0) == -1        # ACB_ERR_ARG
            out.append((env, msgs, states, ctx.decode_stats().tobytes()))
    (e0, m0, s0, d0), (e1, m1, s1, d1) = out
    assert len(m0) > 0 and m0 == m1 and s0 == s1 and d0 == d1
    assert all(np.array_equal(a, b) for a, b in zip(e0, e1))


def test_coverage_and_resets():
    kind, S = "real", 3
    rng = np.random.default_rng(21)
    K = rg._K(kind)
    sched = [[int(rng.integers(300 * K, 2500 * K))] * S for _ in range(9)]      # windows straddle the submits
    sig = _signal(kind, S, sched, rng)
    store = rg.Dev()
    refs = Refs(kind, S)
    with rg._make(kind, S, LEVEL, 0) as ctx:
        off = _feed(ctx, kind, sig, sched[:1], False, store, refs)
        first = copy.deepcopy(refs)
        refs.clear()
        off = _feed(ctx, kind, sig, sched[1:3], False, store, refs, off=off)
        ctx.collect()                                 # covers submit 0 only
        first.check(*ctx.level_stats())
        first.check(*ctx.level_stats(reset=True))
        inp, ch = ctx.level_stats()
        assert not inp["samples"].any() and not ch["rows"].any()
        ctx.sync()                                    # submits 1 and 2, their windows counted from the stream start
        refs.check(*ctx.level_stats())
        ctx.reset()                                   # everything restarts, the windows too
        inp, ch = ctx.level_stats()
        assert not inp["samples"].any() and not ch["rows"].any()
        refs = Refs(kind, S)
        off = _feed(ctx, kind, sig, sched[3:5], False, store, refs, off=off)
        ctx.sync()
        refs.check(*ctx.level_stats())
        # acb_reset_stream(1) between two submits: stream 1 counts from its new start, streams 0 and 2 go on
        off = _feed(ctx, kind, sig, sched[5:6], False, store, refs, off=off)
        ctx.reset_stream(1)
        refs.reset_stream(1)
        # stream 1's carry restarted, so equal counts give it its own rows: the ragged call reports each stream's
        _feed(ctx, kind, sig, sched[6:9], True, store, refs, off=off)
        ctx.sync()
        refs.check(*ctx.level_stats())


@pytest.mark.parametrize("kind", ["u8", "real"])
@pytest.mark.parametrize("mode", [0, 1])
def test_several_contexts(kind, mode):
    import torch
    ngpu = torch.cuda.device_count()
    devices = [0, 1 % ngpu]
    rng = np.random.default_rng(31 + mode)
    S = 3
    sched = _sched(kind, S, 3, rng, False)
    sig = _signal(kind, S, sched, rng)
    fm, fd, fc = rg._freqs(kind)
    K = rg._K(kind)
    kf = rg.FLAG_REAL if kind == "real" else 0
    with api.Context(K, S, NCH, MAXBLK, flags=LEVEL | kf) as one, \
            api.MultiContext(K, S, NCH, MAXBLK, devices, mode=mode, flags=LEVEL | kf) as m:
        for s in range(S):
            if kind == "real":
                one.set_plan_air(s, fd)
                m.set_plan_air(s, fd)
            else:
                one.set_plan(s, fd)
                m.set_plan(s, fd)
        u, off = rg._unit(kind), [0] * S
        for counts in sched:
            buf = np.ascontiguousarray(np.stack([sig[s][off[s] * u:(off[s] + counts[s]) * u] for s in range(S)]))
            if kind == "real":
                one.submit_real(buf)
                m.submit_real(buf)
            else:
                one.submit_host(buf, counts[0])
                m.submit_host(buf, counts[0])
            off = [off[s] + counts[s] for s in range(S)]
        one.sync()
        m.sync()
        i1, c1 = one.level_stats()
        im, cm = m.level_stats()
        if mode == 1:
            parts = [m.part_input_levels(i) for i in range(m.parts())]
            assert all(p.tobytes() == parts[0].tobytes() for p in parts)
    assert i1.tobytes() == im.tobytes()
    for f in ("rows", "windows", "peak"):
        assert np.array_equal(c1[f], cm[f]), f
    for f in ("power_sum", "floor"):
        assert np.allclose(c1[f], cm[f], rtol=1e-10, atol=0), f
    assert c1["windows"].sum() > 0
