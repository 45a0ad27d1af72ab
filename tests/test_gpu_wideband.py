"""Wideband fast form (ACB_FLAG_FAST_WIDEBAND) on the GPU: k_channelize_wb's envelope bit-exact to its definitions
(orc_channelize_dft8* at taps = K, orc_channelize_ovl_fast* at taps > K) for u8 and CS16 input at any K % 8 == 0 and any
channel count, invariant to how the stream is cut into submits, messages identical to the exact form's, and what ran
before wherever the form does not apply."""
import numpy as np
import pytest

from acarsdec_b200 import api
from common import bits_equal
from test_gpu_ovl import ctx_result, rand_tables, run_stream_kind
from test_wideband_oracle import FC, fast_envelope, planner, raster, wideband_fixture

pytestmark = pytest.mark.gpu

FLAG_REAL, FLAG_CS16, FLAG_FAST, FLAG_FAST_FILTER, FLAG_WB = 2, 4, 8, 16, api.FLAG_FAST_WIDEBAND


def freqs_for(K, nch, shift=0):
    """nch channels on the raster around FC, every residue present; `shift` moves those above FC up (other bins per
    stream)"""
    step = max(1, (K // 2 - 4 - 2 * shift) // (2 * nch + 2))
    return [f + 25_000 * shift if f > FC else f for f in raster(nch, step)]


def want(oracle, L, kind, x, K, taps, freqs, variant=-1):
    k, tw = planner(L, kind, variant, K, freqs)
    return fast_envelope(oracle, kind, x, K, taps, k, tw)


U8_CASES = [(56, 56, 13), (160, 160, 8), (192, 2 * 192 + 3, 64), (200, 208, 13), (800, 800, 256), (800, 8 * 800, 64),
            (1600, 1600, 256), (1600, 2 * 1600 + 3, 256), (2048, 16 * 2048, 8), (2048, 2048, 1), (192, 16 * 192, 64),
            (1600, 4 * 1600, 300)]


@pytest.mark.parametrize("K,taps,nch", U8_CASES)
def test_u8_bit_exact(native, oracle, K, taps, nch):
    """Host submits, then device submits with a ring pitch, two streams with different centres: the envelope equals the
    definition bit for bit."""
    S, nblk = 2, 1
    fs = [freqs_for(K, nch, s) for s in range(S)]
    bb = 2048 * K
    x = np.random.default_rng(K + taps + nch).integers(0, 256, size=(S, 3 * nblk * bb), dtype=np.uint8)
    with api.Context(K, S, nch, nblk, flags=FLAG_WB, taps=taps) as ctx:
        for s in range(S):
            ctx.set_plan_at(s, fs[s], FC)
        got = []
        for i in range(2):
            ctx.submit_host(np.ascontiguousarray(x[:, i * nblk * bb:(i + 1) * nblk * bb]), nblk)
            got.append(ctx.read_dm(nblk * 1024))
        pitch = nblk * bb + 4096
        d = ctx.device_alloc(S * pitch)
        staged = np.zeros((S, pitch), dtype=np.uint8)
        staged[:, :nblk * bb] = x[:, 2 * nblk * bb:]
        ctx.copy_to_device(d, staged)
        ctx.submit_device(d, nblk, pitch)
        got.append(ctx.read_dm(nblk * 1024))
        ctx.sync()
        ctx.device_free(d)
        assert ctx.stats().fast_chan_launches == 3
    got = np.concatenate(got, axis=1)
    for s in range(S):
        assert bits_equal(got[s], want(oracle, native, "u8", x[s], K, taps, fs[s]).T.copy()), s


CS16_CASES = [(56, 56, 8, 0, False), (160, 2 * 160 + 3, 13, 1, True), (200, 200, 64, 1, False), (800, 800 + 8, 128, 0, True),
              (1600, 1600, 256, 0, False), (1600, 16 * 1600, 13, 1, False), (2048, 8 * 2048, 256, 1, True), (192, 192, 1, 0, True),
              (1600, 1600, 300, 1, False)]


@pytest.mark.parametrize("K,taps,nch,variant,planar", CS16_CASES)
def test_cs16_bit_exact_ragged(native, oracle, K, taps, nch, variant, planar):
    """Interleaved and planar CS16, both variants, two streams: submits shorter than K and than H, and partial blocks."""
    S = 2
    fs = [freqs_for(K, nch, s) for s in range(S)]
    n = 1024 * K + 40 * K + K // 3
    x = np.random.default_rng(taps + variant + nch).integers(-32768, 32768, size=(S, n, 2), dtype=np.int16)
    cuts = [600 * K - 5, K // 2, max(1, taps - K - 1), 7]
    cuts.append(n - sum(cuts))
    with api.Context(K, S, nch, 2, flags=FLAG_CS16 | FLAG_WB, taps=taps) as ctx:
        for s in range(S):
            ctx.set_plan_cs16(s, fs[s], variant, FC)
        got = run_stream_kind(ctx, "cs16", x, cuts, planar=planar)
        assert ctx.stats().fast_chan_launches >= 2
    for s in range(S):
        assert bits_equal(got[s], want(oracle, native, "cs16", x[s], K, taps, fs[s], variant).T.copy()), s


@pytest.mark.parametrize("K", [160, 192])
@pytest.mark.parametrize("taps_mul", [1, 8])
def test_same_envelope_as_narrow_kernels(native, K, taps_mul):
    """At K = 160 / 192 with 8 channels the new bit alone gives the narrow kernels' envelope (FAST_CHANNELIZER at
    taps = K, FAST_FILTER at taps > K), on u8 and CS16."""
    taps = taps_mul * K
    narrow = FLAG_FAST if taps == K else FLAG_FAST_FILTER
    freqs = freqs_for(K, 8)
    rng = np.random.default_rng(K + taps)
    x = rng.integers(0, 256, size=(1, 2 * 2048 * K), dtype=np.uint8)
    env = {}
    for flags in (narrow, FLAG_WB):
        with api.Context(K, 1, 8, 2, flags=flags, taps=taps) as ctx:
            ctx.set_plan_at(0, freqs, FC)
            ctx.submit_host(x, 2)
            env[flags] = ctx.read_dm(2048)
            ctx.sync()
            assert ctx.stats().fast_chan_launches == 1
    assert bits_equal(env[narrow], env[FLAG_WB])
    xc = rng.integers(-32768, 32768, size=(1, 1500 * K + 5, 2), dtype=np.int16)
    for flags in (narrow, FLAG_WB):
        with api.Context(K, 1, 8, 2, flags=FLAG_CS16 | flags, taps=taps) as ctx:
            ctx.set_plan_cs16(0, freqs, 1, FC)
            env[flags] = run_stream_kind(ctx, "cs16", xc, [xc.shape[1]])
    assert bits_equal(env[narrow], env[FLAG_WB])


def test_u8_chunking_and_reset(native, oracle):
    """Block by block, and host / device submits alternated with the input overwritten as soon as submit N+2 returns,
    give the bits of one submit; after a mid-run reset the first rows omit the terms before the new start."""
    K, taps, nch, S, nblk = 800, 5 * 800 + 3, 64, 2, 4
    fs = [freqs_for(K, nch, s) for s in range(S)]
    bb = 2048 * K
    iq = np.random.default_rng(4).integers(0, 256, size=(S, nblk * bb), dtype=np.uint8)
    wants = [want(oracle, native, "u8", iq[s], K, taps, fs[s]).T.copy() for s in range(S)]

    def fresh():
        ctx = api.Context(K, S, nch, nblk, flags=FLAG_WB, taps=taps)
        for s in range(S):
            ctx.set_plan_at(s, fs[s], FC)
        return ctx

    with fresh() as ctx:
        env = []
        for b in range(nblk):
            ctx.submit_host(np.ascontiguousarray(iq[:, b * bb:(b + 1) * bb]), 1)
            env.append(ctx.read_dm(1024))
        env = np.concatenate(env, axis=1)
        for s in range(S):
            assert bits_equal(env[s], wants[s]), s
        blocks = ctx_result(ctx, S, nch)
    with fresh() as ctx:
        ctx.submit_host(iq, nblk)
        assert ctx_result(ctx, S, nch) == blocks
    with fresh() as ctx:
        pitch = bb + 4096
        dev = [ctx.device_alloc(S * pitch) for _ in range(3)]
        for b in range(nblk):
            blk = np.ascontiguousarray(iq[:, b * bb:(b + 1) * bb])
            if b % 2:
                staged = np.zeros((S, pitch), dtype=np.uint8)
                staged[:, :bb] = blk
                ctx.copy_to_device(dev[b % 3], staged)
                ctx.submit_device(dev[b % 3], 1, pitch)
            else:
                ctx.submit_host(blk, 1)
            if b >= 2 and (b - 2) % 2:
                ctx.copy_to_device(dev[(b - 2) % 3], np.full((S, pitch), 0xA5, dtype=np.uint8))
        assert ctx_result(ctx, S, nch) == blocks
        for d in dev:
            ctx.device_free(d)
        ctx.sync()
        ctx.reset()
        ctx.submit_host(np.ascontiguousarray(iq[:, bb:2 * bb]), 1)
        got = ctx.read_dm(1024)
    for s in range(S):
        assert bits_equal(got[s], want(oracle, native, "u8", iq[s, bb:2 * bb], K, taps, fs[s]).T.copy()), s


def test_cs16_reset(native, oracle):
    K, taps, nch = 1600, 3 * 1600 + 8, 32
    fs = freqs_for(K, nch)
    rng = np.random.default_rng(8)
    xa, xb = rng.integers(-32768, 32768, size=(2, 1, 700 * K, 2), dtype=np.int16)
    with api.Context(K, 1, nch, 1, flags=FLAG_CS16 | FLAG_WB, taps=taps) as ctx:
        ctx.set_plan_cs16(0, fs, 0, FC)
        run_stream_kind(ctx, "cs16", xa, [300 * K + 17])
        ctx.sync()
        ctx.reset()
        got = run_stream_kind(ctx, "cs16", xb, [7, K - 7, 699 * K])[0]
    assert bits_equal(got, want(oracle, native, "cs16", xb[0], K, taps, fs, 0).T.copy())


def _msgs(ctx):
    ctx.sync()
    return sorted((m.stream, m.chn, m.len, m.err, bytes(m.txt[:m.len]), bytes(m.crc), m.pos, m.block) for m in ctx.drain())


@pytest.mark.parametrize("taps_mul", [1, 8])
def test_messages_and_states_equal_exact_form(native, taps_mul):
    """The K = 1600, 256-channel fixture (two weak channels next to neighbours 20 dB stronger): the same messages, and
    every chain in the same framing state, as an exact context (the float demodulator states follow the envelope, which
    differs within the tolerance); every frame sent on the weak channels decodes with err = 0."""
    K = 1600
    iq, freqs, busy, sent = wideband_fixture(K)
    nblk = iq.size // (2048 * K)
    out = {}
    for flags in (0, FLAG_WB):
        with api.Context(K, 1, len(freqs), nblk, flags=flags, taps=taps_mul * K) as ctx:
            ctx.set_plan_at(0, freqs, FC)
            ctx.submit_host(iq.reshape(1, -1), nblk)
            msgs = _msgs(ctx)
            out[flags] = (msgs, [ctx.get_state(0, c).Acarsstate for c in range(len(freqs))])
            assert (ctx.stats().fast_chan_launches > 0) == (flags != 0)
    assert out[0] == out[FLAG_WB]
    weak = [m for m in out[0][0] if m[1] in busy]
    assert len(weak) == len(sent) >= 4 and all(m[3] == 0 for m in weak)


def test_fallbacks_run_what_ran_before(native):
    """acb_set_wf tables, a plan off the raster, taps < K, K % 8 != 0 and real input: no fast launch, and the envelope of
    a context without the bit."""
    rng = np.random.default_rng(3)
    nch = 16

    def u8_env(K, taps, plan_fn, flags):
        x = np.random.default_rng(K + taps).integers(0, 256, size=(1, 2048 * K), dtype=np.uint8)
        with api.Context(K, 1, nch, 1, flags=flags, taps=taps) as ctx:
            plan_fn(ctx)
            ctx.submit_host(x, 1)
            got = ctx.read_dm(1024)
            ctx.sync()
            launches = ctx.stats().fast_chan_launches
        return got, launches

    K = 800
    freqs = freqs_for(K, nch)
    wf_tab = rand_tables(rng, nch, 2 * K)
    off = [f + 12_500 for f in freqs]
    wf_short = rand_tables(rng, nch, K - 8)
    cases = [(K, 2 * K, lambda c: c.set_wf(0, wf_tab)), (K, 2 * K, lambda c: c.set_plan_at(0, off, FC)),
             (K, K - 8, lambda c: c.set_wf(0, wf_short)), (164, 164, lambda c: c.set_plan_at(0, freqs_for(164, nch), FC))]
    for K_, taps, fn in cases:
        ref, _ = u8_env(K_, taps, fn, 0)
        got, launches = u8_env(K_, taps, fn, FLAG_WB)
        assert launches == 0 and bits_equal(got, ref), (K_, taps)
    K = 200
    x = (rng.standard_normal((1, 2 * 1024 * K)) * 100).astype(np.float32)
    from acarsdec_b200 import synth
    fda, _, _ = api.air_plan(K * 12500, synth.DEFAULT_FREQS_MHZ)
    env = []
    for flags in (FLAG_REAL, FLAG_REAL | FLAG_WB):
        with api.Context(K, 1, 8, 2, flags=flags, taps=4 * K) as ctx:
            ctx.set_plan_air(0, fda)
            env.append(run_stream_kind(ctx, "real", x, [x.shape[1]]))
            assert ctx.stats().fast_chan_launches == 0
    assert bits_equal(env[0], env[1])


@pytest.mark.parametrize("taps_mul", [1, 4])
def test_multi_equals_one_context(native, taps_mul):
    """acb_multi, stream split and channel split, with the flag: message for message one wideband context."""
    K = 1600
    iq, freqs, _, _ = wideband_fixture(K)
    nblk = iq.size // (2048 * K)
    S, taps = 2, taps_mul * K
    x = np.stack([iq, np.roll(iq, 555 * 2)])
    key = lambda m: (m.stream, m.chn, m.len, m.err, bytes(m.txt[:m.len]), m.pos)
    with api.Context(K, S, len(freqs), nblk, flags=FLAG_WB, taps=taps) as ctx:
        for s in range(S):
            ctx.set_plan(s, freqs)
        ctx.submit_host(x, nblk)
        ctx.sync()
        ref = sorted(key(m) for m in ctx.drain())
        assert ctx.stats().fast_chan_launches == 1
    assert len(ref) >= 4
    for mode in (0, 1):
        with api.MultiContext(K, S, len(freqs), nblk, [0, 0], mode=mode, flags=FLAG_WB, taps=taps) as mc:
            for s in range(S):
                mc.set_plan(s, freqs)
            mc.submit_host(x, nblk)
            mc.sync()
            got = sorted(key(m) for m in mc.drain())
        assert got == ref, mode
