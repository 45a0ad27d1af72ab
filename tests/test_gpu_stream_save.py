"""Moving streams (acb_save_streams / acb_load_streams): a stream saved from one context and loaded into another slot,
context or process continues bit for bit as if it had stayed.

The reference run is one context in which stream s takes submits 1..n with ragged cuts.  In the moved run a source
context takes submits 1..j and saves s, at a cut where one of its chains is inside a frame (Acarsstate TXT, CRC1 or
CRC2) and, for the streaming kinds, its carry is non-zero and a level window is partly filled.  The blob loads into stream
t != s of a target of another nstreams whose other streams are busy with their own data at other positions, and the
target takes submits j+1..n.  Stream s of the reference must equal the source's output up to j followed by the target's
from j on: messages (every field, stream renamed), the last submit's envelope rows, chain states, decode and level
statistics.  The source itself, continued after the save, must equal the reference (the save changes nothing), and the
target's other streams must equal those of a twin target that never saw the load."""
import ctypes
import os
import pickle
import subprocess
import sys
import zlib
from pathlib import Path

import numpy as np
import pytest

import test_gpu_ragged as rg
from acarsdec_b200 import api

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
DECODE, LEVEL = api.FLAG_DECODE_STATS, api.FLAG_LEVEL_STATS
FC, FF, FFR, FW, FWR = 8, 16, 32, 64, 128
NCH, MAXBLK = rg.NCH, rg.MAXBLK
S, T, SRC, DST = 3, 5, 1, 3                    # source and target stream counts, the moved stream and its new slot
OPEN = (3, 4, 5)                               # F_TXT, F_CRC1, F_CRC2: a frame is being assembled


def _long(kind):
    return {"u8": 2 * 160 + 48, "u8g": 2 * 164 + 40, "real": 2 * 200 + 40}.get(kind, 2 * 160 + 48)


def _kflag(kind):
    return rg.FLAG_REAL if kind == "real" else rg.FLAG_CS16 if kind in ("cs16", "planar") else 0


def _full(m, stream=None):
    return (m.stream if stream is None else stream, m.chn, m.len, m.err, np.float32(m.lvl).tobytes(), m.block, m.pos, m.soh_pos,
            bytes(m.txt), bytes(m.crc))


def _state(ctx, s):
    return [bytes(ctx.get_state(s, ch)) for ch in range(NCH)]


def _stats(ctx, s, flags):
    out = []
    if flags & DECODE:
        out.append(ctx.decode_stats()[s].tobytes())
    if flags & LEVEL:
        inp, ch = ctx.level_stats()
        out += [inp[s].tobytes(), ch[s].tobytes()]
    return out


class Feed:
    """One context's streams, each reading its own signal from its own offset"""

    def __init__(self, ctx, kind, sigs, devmode, store):
        self.ctx, self.kind, self.sigs, self.devmode, self.store = ctx, kind, sigs, devmode, store
        self.off = [0] * len(sigs)
        self.i = 0
        self.rows = None

    def submit(self, counts, src=None):
        """src[k] = (signal, offset) overrides stream k's source (the moved stream continues its own signal)"""
        u = rg._unit(self.kind) if self.kind in rg.U8 else 1
        parts = []
        for k, c in enumerate(counts):
            sig, o = (self.sigs[k], self.off[k]) if not src or k not in src else src[k]
            parts.append(sig[o * u:(o + c) * u])
        dev = self.devmode == "dev" or (self.devmode == "mix" and self.i % 2 == 1)
        self.rows = rg._submit(self.ctx, self.kind, parts, counts, dev and self.store is not None, self.store, stride_pad=3)
        for k, c in enumerate(counts):
            if not src or k not in src:
                self.off[k] += c
        self.i += 1
        return self.rows


def _schedule(kind, rng, nsub, early):
    sched = rg._schedule(kind, S, nsub, rng, stall=0)
    K = rg._K(kind)
    if early:                                   # the stream is saved within H samples of its start
        sched[0][SRC] = 0 if kind in rg.U8 else K // 2 + 3
        sched[1][SRC] = 0 if kind in rg.U8 else K + 5
    for c in sched[-2:]:                        # the last submits give the moved stream rows to compare
        c[SRC] = max(c[SRC], 1 if kind in rg.U8 else 3 * K + 7)
    return sched


def _rows_of(kind, counts_upto):
    K = rg._K(kind)
    return counts_upto * 1024 if kind in rg.U8 else counts_upto // K


def _cut_ok(kind, ctx, sched, j, early):
    """the save point: a frame open on some chain, and (streaming kinds) a carry and a partly filled level window"""
    if early:
        return j == 2
    tot = sum(c[SRC] for c in sched[:j])
    if kind not in rg.U8 and (tot % rg._K(kind) == 0 or _rows_of(kind, tot) % 1024 == 0):
        return False
    return any(ctx.get_state(SRC, ch).Acarsstate in OPEN for ch in range(NCH))


def _target_counts(kind, rng, n):
    return [[int(x) for x in row] for row in rg._schedule(kind, T, n, rng, stall=0)]


def _make(kind, nstreams, flags, taps, unit):
    ctx = rg._make(kind, nstreams, flags, taps)
    if unit and kind not in rg.U8:
        ctx.set_emission_groups(*unit)
    return ctx


def _source(kind, flags, taps, devmode, unit, seed, early=False, nsub=9):
    """Reference and source runs.  Returns what the target needs and what it is compared with."""
    rng = np.random.default_rng(seed)
    sched = _schedule(kind, rng, nsub, early)
    length = max(sum(c[s] for c in sched) for s in range(S)) * (1024 * rg._K(kind) if kind in rg.U8 else 1)
    sig = rg._signal(kind, S, max(length, 1024 * rg._K(kind)), seed=int(rng.integers(1 << 20)))
    store = rg.Dev()
    ref = Feed(_make(kind, S, flags, taps, unit), kind, sig, devmode, store)
    for c in sched:
        ref.submit(c)
    last = ref.ctx.read_dm(int(max(ref.rows)))[SRC, :int(ref.rows[SRC])]
    ref.ctx.sync()
    ref_msgs = ref.ctx.drain()
    want = dict(msgs=[_full(m) for m in ref_msgs if m.stream == SRC], last=last, state=_state(ref.ctx, SRC),
                stats=_stats(ref.ctx, SRC, flags), all=[_full(m) for m in ref_msgs],
                all_states=[_state(ref.ctx, s) for s in range(S)])
    ref.ctx.close()
    src = Feed(_make(kind, S, flags, taps, unit), kind, sig, devmode, store)
    j = None
    for i, c in enumerate(sched[:-2]):
        src.submit(c)
        if i >= 1 and _cut_ok(kind, src.ctx, sched, i + 1, early):
            j = i + 1
            break
    assert j is not None, "no cut with a frame open"
    blob = src.ctx.save_streams([SRC])
    pre = src.ctx.drain()
    for c in sched[j:]:
        src.submit(c)
    src.ctx.sync()
    # the save changed nothing: the source continued equals the reference, every stream
    assert [_full(m) for m in pre + src.ctx.drain()] == want["all"]
    assert [_state(src.ctx, s) for s in range(S)] == want["all_states"]
    src.ctx.close()
    want["pre"] = [_full(m) for m in pre if m.stream == SRC]
    return dict(blob=blob, sched=sched, j=j, sig=sig, want=want, store=store)


def _continue(kind, flags, taps, devmode, unit, run, seed, load=True, ctx=None):
    """The target: its other streams busy before and after; stream DST loads the blob (or, load=False, the twin, stays
    idle) and continues the moved stream's schedule.  Returns (messages, last rows, states, stats, others)."""
    rng = np.random.default_rng(seed)
    sched, j, sig = run["sched"], run["j"], run["sig"]
    rest = sched[j:]
    own = _target_counts(kind, rng, 2 + len(rest))
    length = max(sum(c[k] for c in own) for k in range(T)) * (1024 * rg._K(kind) if kind in rg.U8 else 1)
    tsig = rg._signal(kind, T, max(length, 1024 * rg._K(kind)), seed=int(rng.integers(1 << 20)))
    tgt = Feed(ctx or _make(kind, T, flags, taps, unit), kind, tsig, devmode, run["store"])
    for c in own[:2]:
        c[DST] = 0
        if max(c) == 0:
            c[0] = 1
        tgt.submit(c)
    _replan(tgt.ctx, kind, DST)                 # the slot's own tables differ from the blob's until the load
    if load:
        tgt.ctx.load_streams([DST], run["blob"])
    off = sum(c[SRC] for c in sched[:j])
    for c, mine in zip(rest, own[2:]):
        mine[DST] = c[SRC] if load else 0
        if max(mine) == 0:
            mine[0] = 1
        tgt.submit(mine, src={DST: (sig[SRC], off)} if load else None)
        off += c[SRC]
    last = tgt.ctx.read_dm(int(max(tgt.rows)))[DST, :int(tgt.rows[DST])] if hasattr(tgt.ctx, "read_dm") else None
    tgt.ctx.sync()
    msgs = tgt.ctx.drain()
    others = ([_full(m) for m in msgs if m.stream != DST], [_state(tgt.ctx, k) for k in range(T) if k != DST])
    out = ([_full(m, SRC) for m in msgs if m.stream == DST], last, _state(tgt.ctx, DST), _stats(tgt.ctx, DST, flags), others)
    tgt.ctx.close()
    return out


def _replan(ctx, kind, s):
    """plan stream s with the channels in the other order: other exact tables, twiddles, residues and wideband plan"""
    _, fd, fc = rg._freqs(kind)
    fd2 = list(fd[::-1])
    if isinstance(ctx, api.MultiContext):
        ctx.set_plan(s, fd2) if kind in rg.U8 else ctx.set_plan_cs16(s, fd2, 0, fc)
    elif kind in rg.U8:
        ctx.set_plan_at(s, fd2, fc)
    elif kind == "real":
        ctx.set_plan_air_at(s, fd2, fc)
    else:
        ctx.set_plan_cs16(s, fd2, 1 if kind == "planar" else 0, fc)


def _same_levels(a, b):
    """channel level tables of contexts with different channel counts: k_level_dm tiles the channels by the context's
    count, so the float64 sums may differ in the last bits (as acb_multi_get_level_stats states); the rest is exact"""
    a, b = np.frombuffer(a, api.CHAN_LEVEL_DTYPE), np.frombuffer(b, api.CHAN_LEVEL_DTYPE)
    return all(np.array_equal(a[f], b[f]) for f in ("rows", "windows", "peak")) and \
        all(np.allclose(a[f], b[f], rtol=1e-10, atol=0) for f in ("power_sum", "floor"))


def _assert_moved(run, got, flags, check_env=True, chan_split=False):
    want = run["want"]
    msgs, last, state, stats, _ = got
    assert want["pre"] + msgs == want["msgs"], "messages"
    assert any(True for _ in want["msgs"]), "no message to compare"
    if check_env:
        assert last.shape == want["last"].shape and np.array_equal(last.view(np.uint32), want["last"].view(np.uint32)), "envelope"
    assert state == want["state"], "chain states"
    if chan_split and flags & LEVEL:
        assert stats[:-1] == want["stats"][:-1] and _same_levels(stats[-1], want["stats"][-1]), "statistics"
    else:
        assert stats == want["stats"], "statistics"


# (kind, flags): every form each kind has; taps = K and taps > K
FORMS = {
    "u8": {"exact": 0, "dft": FC, "ovl": FF, "wb": FW},
    "u8g": {"generic": 0},
    "cs16": {"exact": 0, "dft": FC, "ovl": FF, "wb": FW},
    "planar": {"exact": 0, "dft": FC, "ovl": FF, "wb": FW},
    "real": {"exact": 0, "rdft": FC, "ovl": FFR, "wb": FWR},
}
CASES = [(k, f, t) for k, fs in FORMS.items() for f in fs for t in ("K", "long")
         if not (f == "ovl" and t == "K") and not (f == "dft" and t == "long") and not (f == "rdft" and t == "long")
         and not (k == "u8g" and t == "K")]


@pytest.mark.parametrize("kind,form,taps", CASES)
def test_moved_stream_continues_bit_for_bit(kind, form, taps):
    flags = FORMS[kind][form] | DECODE | LEVEL
    tp = _long(kind) if taps == "long" else 0
    seed = zlib.crc32(f"{kind} {form} {taps}".encode())
    devmode = ("host", "mix", "dev")[seed % 3]
    unit = (2, 4093) if kind not in rg.U8 else None
    run = _source(kind, flags, tp, devmode, unit, seed)
    got = _continue(kind, flags, tp, devmode, unit, run, seed + 1)
    _assert_moved(run, got, flags)
    twin = _continue(kind, flags, tp, devmode, unit, run, seed + 1, load=False)
    assert got[4] == twin[4], "the target's other streams changed"


@pytest.mark.parametrize("kind", ["u8", "u8g", "cs16", "real"])
def test_save_near_the_stream_start(kind):
    """taps > K, saved while the stream is within H samples of its start: the pre-start terms stay omitted after the move"""
    flags = {"u8": FF, "u8g": 0, "cs16": FW, "real": 0}[kind] | DECODE
    run = _source(kind, flags, _long(kind), "host", None, 11, early=True)
    _assert_moved(run, _continue(kind, flags, _long(kind), "host", None, run, 12), flags)


@pytest.mark.parametrize("kind", ["u8", "real"])
def test_several_streams_in_one_call(kind):
    """a round trip of several streams in one call; saving and loading into the same slots changes nothing"""
    flags = DECODE | LEVEL
    rng = np.random.default_rng(5)
    sched = rg._schedule(kind, S, 8, rng, stall=0)
    length = max(sum(c[s] for c in sched) for s in range(S)) * (1024 * rg._K(kind) if kind in rg.U8 else 1)
    sig = rg._signal(kind, S, max(length, 1024 * rg._K(kind)), seed=9)
    res = []
    for roundtrip in (False, True):
        f = Feed(_make(kind, S, flags, 0, None), kind, sig, "host", None)
        for i, c in enumerate(sched):
            f.submit(c)
            if roundtrip and i in (2, 5):
                order = [2, 0, 1]
                blob = f.ctx.save_streams(order)
                assert api.blob_info(blob).count == 3
                f.ctx.load_streams(order, blob)
        f.ctx.sync()
        res.append(([_full(m) for m in f.ctx.drain()], [_state(f.ctx, s) for s in range(S)],
                    [_stats(f.ctx, s, flags) for s in range(S)]))
        f.ctx.close()
    assert res[0] == res[1]
    # records are per stream: two streams saved together load into two other slots of a bigger context
    with _make(kind, S, flags, 0, None) as a, _make(kind, T, flags, 0, None) as b:
        fa = Feed(a, kind, sig, "host", None)
        for c in sched[:4]:
            fa.submit(c)
        blob = a.save_streams([0, 2])
        b.load_streams([4, 1], blob)
        assert [_state(b, 4), _state(b, 1)] == [_state(a, 0), _state(a, 2)]
        assert _stats(b, 4, flags) == _stats(a, 0, flags) and _stats(b, 1, flags) == _stats(a, 2, flags)


def test_load_restores_the_raster_plan():
    """a slot given a caller's table (not on the raster) runs its context EXACT; loading a raster-planned stream into it
    restores fast_ok, and the fast form runs again"""
    kind = "u8"
    with _make(kind, S, FC, 0, None) as a, _make(kind, T, FC, 0, None) as b:
        b.set_wf(DST, api.build_wf(rg._K(kind), rg.U8_FM))
        sig = rg._signal(kind, T, MAXBLK * 1024 * rg._K(kind), seed=3)
        fb = Feed(b, kind, sig, "host", None)
        fb.submit([1] * T)
        b.sync()
        assert b.stats().fast_chan_launches == 0
        b.load_streams([DST], a.save_streams([SRC]))
        fb.submit([1] * T)
        b.sync()
        assert b.stats().fast_chan_launches == 1


def test_load_into_a_live_slot():
    """the slot's messages from submits made before the load are still delivered; no other stream's bits change"""
    kind, flags = "u8", DECODE
    run = _source(kind, flags, 0, "host", None, 31)
    res = {}
    for load in (False, True):
        rng = np.random.default_rng(77)
        tsig = rg._signal(kind, T, 6 * MAXBLK * 1024 * rg._K(kind), seed=123)
        tgt = Feed(_make(kind, T, flags, 0, None), kind, tsig, "host", None)
        for _ in range(3):                      # slot DST busy with its own receiver, submits left in flight
            tgt.submit([int(x) for x in rng.integers(1, MAXBLK + 1, size=T)])
        if load:
            tgt.ctx.load_streams([DST], run["blob"])
        tgt.ctx.sync()
        msgs = tgt.ctx.drain()
        res[load] = ([_full(m) for m in msgs], [_state(tgt.ctx, k) for k in range(T) if k != DST])
        if load:
            assert _state(tgt.ctx, DST) == [bytes(s) for s in _state_from_blob(run)]
        tgt.ctx.close()
    assert res[True] == res[False], "messages of submits before the load, or other streams, changed"


def _state_from_blob(run):
    """the moved stream's chain states as the source had them at the save (read from a context loaded with it)"""
    with _make("u8", 1, DECODE, 0, None) as c:
        c.load_streams([0], run["blob"])
        return _state(c, 0)


def _child(path):
    """a fresh process: load the saved stream and continue it (test_restart_in_another_process)"""
    with open(path, "rb") as f:
        args = pickle.load(f)
    run = args["run"]
    run["store"] = rg.Dev()
    got = _continue(args["kind"], args["flags"], args["taps"], "host", args["unit"], run, args["seed"])
    with open(path + ".out", "wb") as f:
        pickle.dump(got, f)


def test_restart_in_another_process(tmp_path):
    kind, flags, taps, unit = "cs16", FW | DECODE | LEVEL, _long("cs16"), (2, 4093)
    run = _source(kind, flags, taps, "host", unit, 41)
    (tmp_path / "stream.blob").write_bytes(run["blob"])
    blob = (tmp_path / "stream.blob").read_bytes()
    args = dict(run={k: v for k, v in run.items() if k != "store"}, kind=kind, flags=flags, taps=taps, unit=unit, seed=42)
    args["run"]["blob"] = blob
    path = str(tmp_path / "args.pkl")
    with open(path, "wb") as f:
        pickle.dump(args, f)
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(ROOT), str(ROOT / "tests")]))
    subprocess.run([sys.executable, "-c", f"import test_gpu_stream_save as t; t._child({path!r})"], check=True, env=env, cwd=str(ROOT),
                   timeout=600)
    with open(path + ".out", "rb") as f:
        got = pickle.load(f)
    _assert_moved(run, got, flags)


def _multi(kind, nstreams, flags, devices, mode=0):
    m = api.MultiContext(rg._K(kind), nstreams, NCH, MAXBLK, devices, mode=mode, flags=flags | _kflag(kind))
    _, fd, fc = rg._freqs(kind)
    for s in range(nstreams):
        if kind in rg.U8:
            m.set_plan(s, fd)
        else:
            m.set_plan_cs16(s, fd, 0, fc)
    return m


def _without_level_sums(blob, nch):
    """a one-record DECODE | LEVEL blob with its CRC, open-window carries and channel level table zeroed"""
    b = bytearray(blob)
    rec = len(b) - 64
    lch = 64 + rec - nch * 40
    lcarry = lch - 32 - nch * 120 - nch * 16
    b[12:16] = bytes(4)
    b[lcarry:lcarry + nch * 16] = bytes(nch * 16)
    b[lch:] = bytes(len(b) - lch)
    return bytes(b)


def _multi_continued(kind, flags, run, mode):
    """a multi-context fed the source schedule, saved at the cut and continued: its blob, and whether its whole output
    (every stream, through the merge) equals the single reference's"""
    with _multi(kind, S, flags, [0, 0], mode) as m:
        f = Feed(m, kind, run["sig"], "host", None)
        for c in run["sched"][:run["j"]]:
            f.submit(c)
        blob = m.save_streams([SRC])
        for c in run["sched"][run["j"]:]:
            f.submit(c)
        m.sync()
        assert [_full(x) for x in m.drain()] == run["want"]["all"], "the save changed the multi-context's output"
        assert [_state(m, s) for s in range(S)] == run["want"]["all_states"]
    return blob


@pytest.mark.parametrize("kind,form", [("u8", 0), ("u8", FC), ("cs16", FW)])
def test_multi_contexts(kind, form):
    """single contexts, stream splits and channel splits (two contexts on one device) exchange the same blobs"""
    flags = form | DECODE | LEVEL
    run = _source(kind, flags, 0, "host", None, 51)
    seed = 52
    _assert_moved(run, _continue(kind, flags, 0, "host", None, run, seed), flags)
    # a stream split as the source gives the single context's blob byte for byte; a channel split too, but for the
    # envelope level sums, which follow its parts' channel tiling
    assert _multi_continued(kind, flags, run, 0) == run["blob"]
    blob_cs = _multi_continued(kind, flags, run, 1)
    assert _without_level_sums(blob_cs, NCH) == _without_level_sums(run["blob"], NCH)
    # single -> stream split, single -> channel split, channel split -> stream split
    for mode in (0, 1):
        _assert_moved(run, _continue(kind, flags, 0, "host", None, run, seed, ctx=_multi(kind, T, flags, [0, 0], mode)), flags,
                      check_env=False, chan_split=mode == 1)
    run_cs = dict(run, blob=blob_cs)
    _assert_moved(run_cs, _continue(kind, flags, 0, "host", None, run_cs, seed, ctx=_multi(kind, T, flags, [0, 0], 0)), flags,
                  check_env=False, chan_split=True)
    with _multi(kind, T, flags, [0, 0], 1) as m2:
        m2.load_streams([DST], run["blob"])
        assert m2.save_streams([DST]) == run["blob"]


@pytest.mark.parametrize("kind", ["u8", "cs16"])
def test_move_across_devices(kind):
    """a single context's stream continued in multi-contexts whose parts sit on two GPUs"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: the move across devices needs two")
    flags, seed = DECODE | LEVEL, 52
    run = _source(kind, flags, 0, "host", None, 51)
    for mode in (0, 1):
        _assert_moved(run, _continue(kind, flags, 0, "host", None, run, seed, ctx=_multi(kind, T, flags, [0, 1], mode)), flags,
                      check_env=False, chan_split=mode == 1)


def test_refusals_leave_the_context_unchanged():
    lib = api.load()
    kind, flags = "real", DECODE
    run = _source(kind, flags, 0, "host", (2, 4093), 61)
    blob = run["blob"]
    others = {}
    with rg._make("real", 1, flags, 0) as c:
        others["group"] = c.save_streams([0])                               # ACB_GROUP_SUBMIT, not (2, 4093)
    for name, (k, fl, tp) in {"taps": ("real", flags, _long("real")), "form": ("real", flags | FC, 0),
                              "decode": ("real", 0, 0), "level": ("real", flags | LEVEL, 0), "kind": ("cs16", flags, 0)}.items():
        with _make(k, 1, fl, tp, (2, 4093)) as c:
            others[name] = c.save_streams([0])
    with _make("real", 1, flags, 0, (2, 4000)) as c:
        others["period"] = c.save_streams([0])                              # the group unit alone matches
    with api.Context(240, 1, NCH, MAXBLK, flags=flags | rg.FLAG_REAL) as c:
        c.set_emission_groups(2, 4093)
        others["K"] = c.save_streams([0])
    with api.Context(200, 1, NCH + 1, MAXBLK, flags=flags | rg.FLAG_REAL) as c:
        c.set_emission_groups(2, 4093)
        others["nch"] = c.save_streams([0])
    bad_crc = bytearray(blob)
    bad_crc[len(blob) // 2] ^= 0x40
    res = []
    for refuse in (False, True):
        tgt = _make(kind, T, flags, 0, (2, 4093))
        if refuse:
            one = np.array([DST], np.int32)
            for name, b in others.items():
                assert lib.acb_load_streams(tgt.h, one.ctypes.data, 1, b, len(b)) == -1, name
            for b in (bytes(bad_crc), blob[:-1]):
                assert lib.acb_load_streams(tgt.h, one.ctypes.data, 1, b, len(b)) == -1
            for lst in ([DST, DST], [T], [-1], [DST, 0]):
                a = np.array(lst, np.int32)
                assert lib.acb_load_streams(tgt.h, a.ctypes.data, len(a), blob, len(blob)) == -1, lst
            two, small = np.array([0, 1], np.int32), ctypes.create_string_buffer(10)
            assert lib.acb_save_streams(tgt.h, two.ctypes.data, 2, small, 10) == -1        # cap too small
        res.append(_continue(kind, flags, 0, "host", (2, 4093), run, 62, ctx=tgt))
    (m0, e0, st0, ds0, o0), (m1, e1, st1, ds1, o1) = res
    assert (m0, st0, ds0, o0) == (m1, st1, ds1, o1) and np.array_equal(e0.view(np.uint32), e1.view(np.uint32))
