"""Frequency-error sums on the device (ACB_FLAG_FREQ_STATS: k_freq_in, k_freq_fin) against the float64 definition
(tests/freq_stats_refs.py): every input kind and channelizer form at taps = K and taps > K, host and device submits,
lockstep and ragged counts, the planners' record, determinism and cut independence, the flag's absence, coverage and
resets, stream moves, several contexts and wide shapes.

Bound: s_re, s_im and mag_sum within 1e-5 of the definition's mag_sum, power_sum within 1e-5 of its own value (a_m and
b_m are float sums on the device)."""
import zlib

import numpy as np
import pytest

import freq_stats_refs as fr
import test_gpu_level_stats as lt
import test_gpu_ragged as rg
from acarsdec_b200 import api
from common import msg_tuple

pytestmark = pytest.mark.gpu

FREQ = api.FLAG_FREQ_STATS
NCH = rg.NCH


class Refs:
    """the definition for every stream of a context, with the steps its planners recorded"""

    def __init__(self, kind, table):
        self.kind = lt.BASE[kind]
        self.K = rg._K(kind)
        self.st = [fr.ChainFreq(self.kind, self.K, table["step"][s]) for s in range(len(table))]

    def feed(self, s, part, dm_rows=None):
        self.st[s].feed(part)

    def check(self, table, streams=None):
        for s in range(len(self.st)) if streams is None else streams:
            for c in range(table.shape[1]):
                fr.check_chain(table[s, c], self.st[s], c)


def _check_plan(kind, table):
    _, fd, fc = rg._freqs(kind)
    freq, step = fr.plan_record(lt.BASE[kind], rg._K(kind), fd, fc)
    for s in range(len(table)):
        assert np.array_equal(table["freq_hz"][s], freq) and np.array_equal(table["step"][s], step)


@pytest.mark.parametrize("kind,form,taps,counts", lt.CASES)
def test_sums_match_the_definition(kind, form, taps, counts):
    rng = np.random.default_rng(zlib.crc32(f"freq{kind}{form}{taps}{counts}".encode()))
    S, ragged = 3, counts == "ragged"
    sched = lt._sched(kind, S, 4, rng, ragged)
    sig = lt._signal(kind, S, sched, rng)
    store = rg.Dev()
    with rg._make(kind, S, FREQ | lt.FORMS[kind][form], lt._taps(kind) if taps == "long" else 0) as ctx:
        t0 = ctx.freq_stats()
        _check_plan(kind, t0)
        assert not t0["pairs"].any()
        refs = Refs(kind, t0)
        lt._feed(ctx, kind, sig, sched, ragged, store, refs)
        ctx.sync()
        t = ctx.freq_stats()
    refs.check(t)
    assert t["pairs"].min() > 0 and (np.hypot(t["s_re"], t["s_im"]) / t["mag_sum"]).max() > 0.1


@pytest.mark.parametrize("kind", ["u8", "real", "cs16"])
def test_same_bits_and_cut_independence(kind):
    rng = np.random.default_rng(11)
    K = rg._K(kind)
    total = rg.MAXBLK if kind in rg.U8 else rg.MAXBLK * 1024 * K - K
    cuts = [1, 2] if kind in rg.U8 else [total // 5, 2 * total // 5, total - total // 5 - 2 * total // 5]
    sched_b = [[c, int(rng.integers(1, rg.MAXBLK + 1)) if kind in rg.U8 else int(rng.integers(K, total))] for c in cuts]
    sig = lt._signal(kind, 2, sched_b, rng)
    store = rg.Dev()
    tabs = []
    for _ in range(2):
        with rg._make(kind, 1, FREQ, 0) as a, rg._make(kind, 2, FREQ, 0) as b:
            lt._feed(a, kind, sig[:1], [[total]], False, store)
            lt._feed(b, kind, sig, sched_b, True, store)
            a.sync()
            b.sync()
            tabs.append((a.freq_stats(), b.freq_stats()))
    assert tabs[0][0].tobytes() == tabs[1][0].tobytes() and tabs[0][1].tobytes() == tabs[1][1].tobytes()
    ta, tb = tabs[0][0][0], tabs[0][1][0]
    assert np.array_equal(ta["pairs"], tb["pairs"])
    for f in ("s_re", "s_im", "mag_sum", "power_sum"):
        assert np.allclose(ta[f], tb[f], rtol=1e-10, atol=0), f


@pytest.mark.parametrize("kind", ["u8", "real", "planar"])
def test_flag_changes_nothing_else(kind):
    rng = np.random.default_rng(3)
    S = 3
    sched = lt._sched(kind, S, 4, rng, True)
    sig = lt._signal(kind, S, sched, rng)
    store = rg.Dev()
    out = []
    base = api.FLAG_DECODE_STATS | api.FLAG_LEVEL_STATS | lt.FORMS[kind]["fast"]
    for flags in (base, base | FREQ):
        with rg._make(kind, S, flags, 0) as ctx:
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
            if not flags & FREQ:
                a = np.zeros((S, NCH), api.CHAN_FREQ_DTYPE)
                assert ctx.lib.acb_get_freq_stats(ctx.h, a.ctypes.data, a.size, 0) == -1        # ACB_ERR_ARG
            lv = ctx.level_stats()
            out.append((env, msgs, states, ctx.decode_stats().tobytes(), lv[0].tobytes() + lv[1].tobytes()))
    (e0, m0, s0, d0, l0), (e1, m1, s1, d1, l1) = out
    assert len(m0) > 0 and m0 == m1 and s0 == s1 and d0 == d1 and l0 == l1
    assert all(np.array_equal(a, b) for a, b in zip(e0, e1))


def test_coverage_resets_and_replans():
    kind, S = "real", 3
    rng = np.random.default_rng(21)
    K = rg._K(kind)
    sched = [[int(rng.integers(300 * K, 2500 * K))] * S for _ in range(9)]
    sig = lt._signal(kind, S, sched, rng)
    store = rg.Dev()
    with rg._make(kind, S, FREQ, 0) as ctx:
        refs = Refs(kind, ctx.freq_stats())
        off = lt._feed(ctx, kind, sig, sched[:1], False, store, refs)
        first = [np.array([st.sums(c) for c in range(NCH)]) for st in refs.st]
        for st in refs.st:
            st.clear()
        off = lt._feed(ctx, kind, sig, sched[1:3], False, store, refs, off=off)
        ctx.collect()                                 # covers submit 0 only
        t = ctx.freq_stats(reset=True)
        for s in range(S):
            for c in range(NCH):
                assert abs(t["s_re"][s, c] - first[s][c, 0]) <= 1e-5 * first[s][c, 2]
        t = ctx.freq_stats()
        assert not t["pairs"].any() and not t["mag_sum"].any() and t["freq_hz"].all()     # the plan stays
        ctx.sync()
        refs.check(ctx.freq_stats())
        ctx.reset()
        t = ctx.freq_stats()
        assert not t["pairs"].any() and t["freq_hz"].all()
        refs = Refs(kind, t)
        off = lt._feed(ctx, kind, sig, sched[3:5], False, store, refs, off=off)
        ctx.reset_stream(1)
        refs.st[1] = fr.ChainFreq(refs.kind, K, ctx.freq_stats()["step"][1])
        off = lt._feed(ctx, kind, sig, sched[5:6], True, store, refs, off=off)
        # a re-plan of stream 0 two channels higher: the rows after it are measured against the new plan
        _, fd, fc = rg._freqs(kind)
        ctx.set_plan_air_at(0, [int(f) + 25000 for f in fd], fc)
        t = ctx.freq_stats()
        freq, step = fr.plan_record("real", K, [int(f) + 25000 for f in fd], fc)
        assert np.array_equal(t["freq_hz"][0], freq) and np.array_equal(t["step"][0], step)
        refs.st[0].replan(step)
        lt._feed(ctx, kind, sig, sched[6:9], True, store, refs, off=off)
        ctx.sync()
        refs.check(ctx.freq_stats())


def test_envelope_input_and_caller_tables_are_not_measured():
    rng = np.random.default_rng(7)
    S = 2
    with api.Context(160, S, NCH, rg.MAXBLK, flags=FREQ | 1) as ctx:        # NO_INPUT_STAGING: envelope input only
        for n in (700, 1500):
            ctx.submit_dm(rng.random((S, n, NCH)).astype(np.float32))
        ctx.sync()
        t = ctx.freq_stats()
    assert not t["pairs"].any() and not t["mag_sum"].any()
    kind = "u8"
    sched = [[2, 2, 2]] * 2
    sig = lt._signal(kind, 3, sched, rng)
    store = rg.Dev()
    with rg._make(kind, 3, FREQ, 0, wf_streams=(1,)) as ctx:
        lt._feed(ctx, kind, sig, sched, False, store)
        ctx.sync()
        t = ctx.freq_stats()
    assert not t["pairs"][1].any() and not t["mag_sum"][1].any() and not t["freq_hz"][1].any() and not t["step"][1].any()
    assert t["pairs"][0].all() and t["pairs"][2].all()


@pytest.mark.parametrize("kind", ["u8", "real", "cs16"])
def test_moved_streams_continue_bit_for_bit(kind):
    rng = np.random.default_rng(41)
    S = 3
    sched = lt._sched(kind, S, 4, rng, False)
    sig = lt._signal(kind, S, sched, rng)
    store = rg.Dev()
    flags = FREQ | api.FLAG_LEVEL_STATS
    perm = [2, 0, 1]                                  # stream s of a continues in slot perm[s] of b
    with rg._make(kind, S, flags, 0) as a, rg._make(kind, S, flags, 0) as b, rg._make(kind, S, api.FLAG_LEVEL_STATS, 0) as c:
        off = lt._feed(a, kind, sig, sched[:2], False, store)
        blob = a.save_streams([0, 1, 2])
        b.load_streams(perm, blob)
        with pytest.raises(api.AcbError):
            c.load_streams([0, 1, 2], blob)           # a flagged blob into a flagless context
        with pytest.raises(api.AcbError):
            a.load_streams([0, 1, 2], c.save_streams([0, 1, 2]))
        inv = [perm.index(i) for i in range(S)]
        off_b = [off[inv[i]] for i in range(S)]
        lt._feed(a, kind, sig, sched[2:], False, store, off=off)
        lt._feed(b, kind, [sig[inv[i]] for i in range(S)], sched[2:], False, store, off=off_b)
        a.sync()
        b.sync()
        ta, tb = a.freq_stats(), b.freq_stats()
    for s in range(S):
        assert ta[s].tobytes() == tb[perm[s]].tobytes(), s
    assert ta["pairs"].all()


@pytest.mark.parametrize("kind", ["u8", "real"])
@pytest.mark.parametrize("mode", [0, 1])
def test_several_contexts(kind, mode):
    import torch
    devices = [0, 1 % torch.cuda.device_count()]
    rng = np.random.default_rng(31 + mode)
    S = 3
    sched = lt._sched(kind, S, 3, rng, False)
    sig = lt._signal(kind, S, sched, rng)
    _, fd, _ = rg._freqs(kind)
    K = rg._K(kind)
    kf = rg.FLAG_REAL if kind == "real" else 0
    with api.Context(K, S, NCH, rg.MAXBLK, flags=FREQ | kf) as one, \
            api.MultiContext(K, S, NCH, rg.MAXBLK, devices, mode=mode, flags=FREQ | kf) as m:
        for s in range(S):
            for x in (one, m):
                (x.set_plan_air if kind == "real" else x.set_plan)(s, fd)
        u, off = rg._unit(kind), [0] * S
        for counts in sched:
            buf = np.ascontiguousarray(np.stack([sig[s][off[s] * u:(off[s] + counts[s]) * u] for s in range(S)]))
            for x in (one, m):
                x.submit_real(buf) if kind == "real" else x.submit_host(buf, counts[0])
            off = [off[s] + counts[s] for s in range(S)]
        one.sync()
        m.sync()
        t1, tm = one.freq_stats(), m.freq_stats()
    assert t1["pairs"].all() and t1.tobytes() == tm.tobytes()


def _wide(kind, K, S, nch, flags, nblk, seed):
    """a context of nch channels on the 25 kHz raster around fc, its input (noise and one carrier per stream), and
    the definition fed with it"""
    rng = np.random.default_rng(seed)
    fc = 130_000_000
    half = min(nch // 2 + 1, (K * 12500 // 2 - 50000) // 25000)
    ks = [k for k in range(-half, half + 1) if k][:nch]
    freqs = [fc + 25000 * k for k in ks]
    kf = {"u8": 0, "cs16": rg.FLAG_CS16, "real": rg.FLAG_REAL}[kind]
    ctx = api.Context(K, S, nch, nblk, flags=FREQ | flags | kf)
    for s in range(S):
        if kind == "u8":
            ctx.set_plan_at(s, freqs, fc)
        elif kind == "cs16":
            ctx.set_plan_cs16(s, freqs, 0, fc)
        else:
            ctx.set_plan_air_at(s, freqs, fc)
    n = nblk * 1024 * K
    t = np.arange(n) / (K * 12500)
    sig = []
    for s in range(S):
        tone = 20 * np.exp(2j * np.pi * ((freqs[s % nch] - fc) + 900.0) * t)
        if kind == "u8":
            x = np.clip(np.floor(np.stack([tone.real, tone.imag], 1) + rng.normal(0, 2, (n, 2)) + 128), 0, 255).astype(np.uint8)
            sig.append(x.reshape(-1))
        elif kind == "cs16":
            sig.append(np.round(np.stack([tone.real, tone.imag], 1) * 64 + rng.normal(0, 100, (n, 2))).astype(np.int16))
        else:
            sig.append((rng.normal(0, 0.01, n)).astype(np.float32))
    return ctx, sig


@pytest.mark.parametrize("kind,K,S,nch,flags,nblk", [
    ("cs16", 1600, 1, 256, rg.FAST_WIDEBAND, 2),     # the CS16 wideband shape: 32 chain tiles
    ("real", 800, 1, 200, rg.FAST_WIDEBAND_REAL, 2),
    ("u8", 161, 2, 5, 0, 2),                         # odd K: the row's last sample is not used
    ("u8", 160, 300, 13, rg.FAST_CHANNELIZER, 1),    # many streams, a partial chain tile
])
def test_wide_shapes(kind, K, S, nch, flags, nblk):
    ctx, sig = _wide(kind, K, S, nch, flags, nblk, seed=K + S)
    store = rg.Dev()
    with ctx:
        t0 = ctx.freq_stats()
        refs = [fr.ChainFreq(kind, K, t0["step"][s]) for s in range(S)]
        buf = np.ascontiguousarray(np.stack(sig))
        if kind == "u8":
            ctx.submit_host(buf, nblk)
        elif kind == "cs16":
            ctx.submit_cs16(buf)
        else:
            ctx.submit_real(buf)
        ctx.sync()
        t = ctx.freq_stats()
    for s in range(S):
        refs[s].feed(sig[s])
        for c in range(nch):
            fr.check_chain(t[s, c], refs[s], c)
    assert int(t["pairs"].min()) == nblk * 1024
