"""Overlapping-window channelizer (taps > K) on the GPU: envelope bit-exact against its CPU definition
(tests/host/ovl_oracle.c) for every input kind and kernel form, invariant to how the stream is cut into submits (the
history carried across them, omitted terms after a reset), end to end with frames and demodulator states, acb_multi in
both split modes, and the weak-channel scenario the feature exists for."""
import numpy as np
import pytest

import ovl_refs
import refs
from acarsdec_b200 import api, synth
from common import bits_equal
from test_ovl_oracle import decode_oracle, weak_strong_scenario

pytestmark = pytest.mark.gpu

FLAG_REAL, FLAG_CS16, FLAG_FAST = 2, 4, 8


def rand_tables(rng, nch, taps):
    w = rng.standard_normal((nch, 2 * taps)) / taps
    return w.astype(np.float32)


def oracle_dm(kind, x, K, wf):
    if kind == "u8":
        return ovl_refs.channelize_ovl(x, K, wf)
    if kind == "real":
        return ovl_refs.channelize_ovl_real(x, K, wf)
    return ovl_refs.channelize_ovl_cs16(x, K, wf)


def run_stream_kind(ctx, kind, x, cuts, planar=False):
    """Feed (nstreams, n[, 2]) input through submits of the given sizes; returns (nstreams, rows, nch) envelopes."""
    out, p = [], 0
    for n in cuts:
        part = np.ascontiguousarray(x[:, p:p + n])
        p += n
        if kind == "real":
            got = ctx.submit_real(part)
        elif planar:
            got = ctx.submit_cs16_planar(np.ascontiguousarray(part[..., 0]), np.ascontiguousarray(part[..., 1]))
        else:
            got = ctx.submit_cs16(part)
        if got:
            out.append(ctx.read_dm(got))
    return np.concatenate(out, axis=1)


# (kind, K, taps, nch, variant): every input kind, pipeline and generic kernels, both real-input row forms
CASES = [
    ("u8", 160, 168, 8, None), ("u8", 192, 2 * 192, 5, None), ("u8", 200, 4 * 200 - 3, 64, None),
    ("u8", 1600, 16 * 1600, 8, None), ("u8", 44, 4 * 44 - 3, 5, None),
    ("cs16", 160, 2 * 160, 8, None), ("cs16", 1600, 1600 + 8, 5, None), ("cs16", 192, 4 * 192 - 3, 64, "planar"),
    ("cs16", 42, 2 * 42, 5, None),
    ("real", 200, 16 * 200, 8, None), ("real", 160, 160 + 8, 64, None), ("real", 200, 2 * 200, 5, "rows2"),
    ("real", 202, 4 * 202 - 3, 5, None),
]


@pytest.mark.parametrize("kind,K,taps,nch,variant", CASES)
def test_ovl_envelope_bit_exact(native, kind, K, taps, nch, variant, monkeypatch):
    if variant == "rows2":
        monkeypatch.setenv("ACB_REAL_ROWS", "2")
    rng = np.random.default_rng(K * 7 + taps)
    S, nblk = 2, 2
    wf = rand_tables(rng, nch, taps)
    if kind == "u8":
        x = rng.integers(0, 256, size=(S, 3 * nblk * 2048 * K), dtype=np.uint8)
        with api.Context(K, S, nch, nblk, taps=taps) as ctx:
            for s in range(S):
                ctx.set_wf(s, wf)
            got = []
            for i in range(3):                                   # three submits: the history crosses two boundaries
                ctx.submit_host(np.ascontiguousarray(x[:, i * nblk * 2048 * K:(i + 1) * nblk * 2048 * K]), nblk)
                got.append(ctx.read_dm(nblk * 1024))
            got = np.concatenate(got, axis=1)
    else:
        n = 2 * nblk * 1024 * K + K // 3
        if kind == "real":
            x = (rng.standard_normal((S, n)) * 100).astype(np.float32)
        else:
            x = rng.integers(-32768, 32768, size=(S, n, 2), dtype=np.int16)
        cuts = [nblk * 1024 * K - 5, K // 2, taps - K - 1 if taps > K + 1 else 3, n]
        cuts[-1] = n - sum(cuts[:-1])
        flags = FLAG_REAL if kind == "real" else FLAG_CS16
        with api.Context(K, S, nch, nblk + 1, flags=flags, taps=taps) as ctx:
            for s in range(S):
                ctx.set_wf(s, wf)
            got = run_stream_kind(ctx, kind, x, cuts, planar=variant == "planar")
    for s in range(S):
        want = oracle_dm(kind, x[s], K, wf)
        assert got.shape[1] == want.shape[1]
        assert bits_equal(got[s], want.T.copy()), s


def _frames_plan(K, nblk, seed, nch=8):
    fm = synth.DEFAULT_FREQS_MHZ[:nch]
    fd, _, fc = api.plan(K, fm)
    plan = synth.make_plan(K, fm, fc, seconds=nblk * 1024 / 12500, seed=seed, msgs_per_chan_per_sec=3.0,
                           text_len=(5, 30), amp=(6.0, 12.0))
    return fm, plan


def oracle_path(iq_stream, K, wf):
    """channelize_ovl -> orc_demod -> FEC on one stream: (frames, per-channel states, envelope)."""
    orc = refs.OracleLib()
    dm = ovl_refs.channelize_ovl(iq_stream, K, wf)
    sink = refs.Sink()
    chans = []
    for c in range(wf.shape[0]):
        ch = orc.new_chan(c)
        orc.demod(ch, dm[c], sink)
        chans.append(ch.vec())
    want = []
    for m in sink.msgs():
        f = orc.fec(m)
        if f is not None:
            want.append((f.chn, f.len, f.err, bytes(f.txt[:f.len]), bytes(f.crc)))
    return sorted(want), chans, dm


def ctx_result(ctx, S, nch):
    ctx.sync()
    msgs = sorted((m.stream,) + m.as_tuple() for m in ctx.drain())
    return msgs, [[ctx.get_state(s, c).vec() for c in range(nch)] for s in range(S)]


@pytest.mark.parametrize("K,taps", [(160, 8 * 160), (192, 2 * 192 + 5)])
def test_ovl_chunking_invariance_u8(native, oracle, K, taps):
    """One submit, block by block, random block counts with collect/sync in between, host and device submits alternated
    (dense and ring pitch), an input buffer overwritten as soon as the N+2 submit returns: identical envelope bits,
    frames and states, all equal to the oracle over the whole stream."""
    S, nblk, nch = 2, 8, 8
    fm, plan = _frames_plan(K, nblk, seed=K)
    one = synth.render_blocks(plan, 0, nblk).reshape(-1)
    iq = np.stack([one, np.roll(one, 12345 * 2)])                   # two different streams
    wf = api.build_wf_lp(K, taps, fm)
    bb = 2048 * K
    wants = [oracle_path(iq[s], K, wf) for s in range(S)]
    want_msgs = sorted((s,) + m for s in range(S) for m in wants[s][0])
    assert len(want_msgs) >= 10

    def fresh():
        ctx = api.Context(K, S, nch, nblk, taps=taps)
        for s in range(S):
            ctx.set_plan(s, [int(round(f * 1e6)) for f in fm])
        return ctx

    schedules = {"one": [nblk], "blocks": [1] * nblk, "random": [3, 1, 2, 2]}
    results = {}
    for name, sched in schedules.items():
        with fresh() as ctx:
            p, env = 0, []
            for i, n in enumerate(sched):
                ctx.submit_host(np.ascontiguousarray(iq[:, p * bb:(p + n) * bb]), n)
                env.append(ctx.read_dm(n * 1024))
                if name == "random" and i % 2:
                    ctx.collect()
                p += n
            results[name] = ctx_result(ctx, S, nch) + (np.concatenate(env, axis=1),)
    # host / device alternated, ring pitch, and a device buffer overwritten as soon as submit N+2 has returned (no
    # read-back in between: the submits stay in flight)
    with fresh() as ctx:
        pitch = 3 * bb + 4096
        dev = [ctx.device_alloc(S * pitch) for _ in range(3)]
        for b in range(nblk):
            blk = np.ascontiguousarray(iq[:, b * bb:(b + 1) * bb])
            if b % 2:
                slot = (b // 2) % 3
                staged = np.zeros((S, pitch), dtype=np.uint8)
                staged[:, :bb] = blk
                ctx.copy_to_device(dev[slot], staged)
                ctx.submit_device(dev[slot], 1, pitch)
            else:
                ctx.submit_host(blk, 1)
            if b >= 2 and (b - 2) % 2:
                # submit b-2 went through dev[((b-2)//2) % 3]: it has been read, scribble over it
                ctx.copy_to_device(dev[((b - 2) // 2) % 3], np.full((S, pitch), 0xA5, dtype=np.uint8))
        results["mixed"] = ctx_result(ctx, S, nch) + (None,)
        for d in dev:
            ctx.device_free(d)
    for name, (msgs, states, env) in results.items():
        assert msgs == want_msgs, name
        for s in range(S):
            assert env is None or bits_equal(env[s], wants[s][2].T.copy()), (name, s)
            assert states[s] == wants[s][1], (name, s)


def test_ovl_reset_restarts_history(native):
    """After a mid-run acb_reset the first rows omit the terms before the new stream start (u8: not the zero bytes of a
    cleared buffer, not the previous stream's tail) — for every input kind."""
    rng = np.random.default_rng(5)
    K, taps, nch = 160, 5 * 160 + 3, 8
    wf = rand_tables(rng, nch, taps)
    a = rng.integers(0, 256, size=(1, 2048 * K), dtype=np.uint8)
    b = rng.integers(0, 256, size=(1, 2048 * K), dtype=np.uint8)
    with api.Context(K, 1, nch, 1, taps=taps) as ctx:
        ctx.set_wf(0, wf)
        ctx.submit_host(a, 1)
        ctx.sync()
        ctx.reset()
        ctx.submit_host(b, 1)
        got = ctx.read_dm(1024)[0]
    assert bits_equal(got, ovl_refs.channelize_ovl(b[0], K, wf).T.copy())
    for kind, flags in (("real", FLAG_REAL), ("cs16", FLAG_CS16)):
        if kind == "real":
            xa, xb = (rng.standard_normal((2, 1, 3000 * K)) * 50).astype(np.float32)
        else:
            xa, xb = rng.integers(-32768, 32768, size=(2, 1, 3000 * K, 2), dtype=np.int16)
        with api.Context(K, 1, nch, 3, flags=flags, taps=taps) as ctx:
            ctx.set_wf(0, wf)
            run_stream_kind(ctx, kind, xa, [1000 * K + 17])
            ctx.sync()
            ctx.reset()
            got = run_stream_kind(ctx, kind, xb, [7, K - 7, 2999 * K])[0]
        assert bits_equal(got, oracle_dm(kind, xb[0], K, wf).T.copy()), kind


@pytest.mark.parametrize("kind,variant", [("cs16", 0), ("cs16", 1), ("real", None)])
def test_ovl_streaming_frames_and_planners(native, kind, variant):
    """The streaming front-ends end to end with their planners' low-pass tables, ragged submits (below K and below H):
    frames and states equal the oracle's over the whole stream."""
    K = 200 if kind == "real" else 160
    taps, nblk, nch = 8 * K, 6, 8
    fm, plan = _frames_plan(K, nblk, seed=11 + (variant or 0))
    n = nblk * 1024 * K
    with api.Context(K, 1, nch, nblk, flags=FLAG_REAL if kind == "real" else FLAG_CS16, taps=taps) as ctx:
        if kind == "real":
            fd, fc, _ = api.air_plan(K * 12500, fm)
            plan = synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, bursts=plan.bursts, seed=plan.seed)
            x = synth.render_real(plan, 0, n).reshape(1, -1)
            ctx.set_plan_air(0, fd)
            wf = api.build_wf_air_lp(K * 12500, taps, fm)
        else:
            fd = list(plan.freqs_hz)
            x = synth.render_cs16(plan, 0, n).reshape(1, n, 2)
            fc = ctx.set_plan_cs16(0, fd, variant)
            wf = api.build_wf_cs16_lp(variant, K, taps, fd, fc)
        cuts = [K - 3, taps - K - 5, 3 * 1024 * K + 11]
        cuts.append(n - sum(cuts))
        env = run_stream_kind(ctx, kind, x, cuts)
        msgs, states = ctx_result(ctx, 1, nch)
    orc = refs.OracleLib()
    dm = oracle_dm(kind, x[0], K, wf)
    assert bits_equal(env[0], dm.T.copy())
    sink = refs.Sink()
    chans = []
    for c in range(nch):
        ch = orc.new_chan(c)
        orc.demod(ch, dm[c], sink)
        chans.append(ch.vec())
    want = sorted((0,) + (f.chn, f.len, f.err, bytes(f.txt[:f.len]), bytes(f.crc))
                  for f in (orc.fec(m) for m in sink.msgs()) if f is not None)
    assert msgs == want and len(want) >= 5
    assert states[0] == chans


def test_ovl_multi_equals_one_context(native):
    """acb_multi in channel-split and stream-split modes (two contexts on one GPU) equals one context, message for
    message; ACB_FLAG_FAST_CHANNELIZER with taps > K runs the exact kernel."""
    K, taps, nblk, S, nch = 160, 4 * 160 + 8, 4, 2, 8
    fm, plan = _frames_plan(K, nblk, seed=21)
    one = synth.render_blocks(plan, 0, nblk).reshape(-1)
    iq = np.stack([one, np.roll(one, 777 * 2)])
    freqs = [int(round(f * 1e6)) for f in fm]
    with api.Context(K, S, nch, nblk, flags=FLAG_FAST, taps=taps) as ctx:
        for s in range(S):
            ctx.set_plan(s, freqs)
        for h in range(2):
            ctx.submit_host(np.ascontiguousarray(iq[:, h * 2 * 2048 * K:(h + 1) * 2 * 2048 * K]), 2)
        ctx.sync()
        ref = [(m.stream, m.chn, m.len, m.err, bytes(m.txt[:m.len]), m.pos) for m in ctx.drain()]
        assert ctx.stats().fast_chan_launches == 0
    assert len(ref) >= 4
    for mode in (0, 1):
        with api.MultiContext(K, S, nch, nblk, [0, 0], mode=mode, taps=taps) as mc:
            for s in range(S):
                mc.set_plan(s, freqs)
            for h in range(2):
                mc.submit_host(np.ascontiguousarray(iq[:, h * 2 * 2048 * K:(h + 1) * 2 * 2048 * K]), 2)
            mc.sync()
            got = [(m.stream, m.chn, m.len, m.err, bytes(m.txt[:m.len]), m.pos) for m in mc.drain()]
        assert got == ref, mode


def test_weak_channel_next_to_strong_neighbour_gpu(native, oracle):
    """Scenario of tests/test_ovl_oracle.py on the GPU: the 8K-tap context decodes the frames the CPU oracle decodes,
    the boxcar context does not."""
    K = 160
    iq, fm, sent = weak_strong_scenario(K)
    nblk = iq.size // (2048 * K)
    want = sorted(m.as_tuple() for m in decode_oracle(oracle, ovl_refs.channelize_ovl(iq, K, api.build_wf_lp(K, 8 * K, fm)[:1])[0]))
    assert len(want) == len(sent)
    freqs = [int(round(f * 1e6)) for f in fm]
    got = {}
    for taps in (0, 8 * K):
        with api.Context(K, 1, 2, nblk, taps=taps) as ctx:
            ctx.set_plan(0, freqs)
            ctx.submit_host(iq.reshape(1, -1), nblk)
            ctx.sync()
            got[taps] = sorted(m.as_tuple() for m in ctx.drain() if m.chn == 0)
    assert got[8 * K] == want
    assert not any(m[2] == 0 for m in got[0])
