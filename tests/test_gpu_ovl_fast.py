"""Polyphase fast form of the overlapping-window channelizer (ACB_FLAG_FAST_FILTER) on the GPU: envelope bit-exact to
its CPU restatement (orc_channelize_ovl_fast{,_cs16}) for u8 and CS16 input, invariant to how the stream is cut into
submits, messages identical to the exact form's, and the exact kernel wherever the fast form does not apply."""
import numpy as np
import pytest

import ovl_fast_refs
import ovl_refs
from acarsdec_b200 import api, synth
from common import bits_equal
from test_gpu_ovl import _frames_plan, ctx_result, rand_tables, run_stream_kind
from test_ovl_fast_oracle import fast_plan
from test_ovl_oracle import weak_strong_scenario

pytestmark = pytest.mark.gpu

FLAG_REAL, FLAG_CS16, FLAG_FAST, FLAG_FAST_FILTER = 2, 4, 8, 16


def raster(nch):
    """nch channels 50 kHz apart above a centre of 131.0 MHz: every offset a whole even number of 12.5 kHz steps"""
    return [131_050_000 + 25_000 * i for i in range(nch)], 131_000_000


def want_fast(kind, x, K, taps, freqs, fc, variant=None):
    h = api.build_lowpass(K, taps)
    k, tw = fast_plan(kind, variant, K, freqs, fc)
    if kind == "u8":
        return ovl_fast_refs.channelize_ovl_fast(x, K, h, k, tw)
    return ovl_fast_refs.channelize_ovl_fast_cs16(x, K, h, k, tw)


U8_CASES = [(160, 168, 8), (160, 2 * 160 + 3, 13), (192, 4 * 192 - 5, 1), (192, 8 * 192, 8), (160, 16 * 160, 13),
            (192, 16 * 192 - 1, 8)]


@pytest.mark.parametrize("K,taps,nch", U8_CASES)
def test_u8_bit_exact(native, K, taps, nch):
    """Host submits, then device submits with a ring pitch: the envelope of both streams equals the restatement."""
    S, nblk = 2, 2
    freqs, fc = raster(nch)
    bb = 2048 * K
    x = np.random.default_rng(K + taps).integers(0, 256, size=(S, 4 * nblk * bb), dtype=np.uint8)
    with api.Context(K, S, nch, nblk, flags=FLAG_FAST_FILTER, taps=taps) as ctx:
        for s in range(S):
            ctx.set_plan_at(s, freqs, fc)
        got = []
        for i in range(2):
            ctx.submit_host(np.ascontiguousarray(x[:, i * nblk * bb:(i + 1) * nblk * bb]), nblk)
            got.append(ctx.read_dm(nblk * 1024))
        pitch = nblk * bb + 4096
        d = ctx.device_alloc(S * pitch)
        for i in range(2, 4):
            staged = np.zeros((S, pitch), dtype=np.uint8)
            staged[:, :nblk * bb] = x[:, i * nblk * bb:(i + 1) * nblk * bb]
            ctx.copy_to_device(d, staged)
            ctx.submit_device(d, nblk, pitch)
            got.append(ctx.read_dm(nblk * 1024))
        ctx.sync()
        ctx.device_free(d)
        assert ctx.stats().fast_chan_launches == 4
    got = np.concatenate(got, axis=1)
    for s in range(S):
        assert bits_equal(got[s], want_fast("u8", x[s], K, taps, freqs, fc).T.copy()), s


CS16_CASES = [(160, 160 + 8, 8, 0, False), (160, 2 * 160 + 3, 13, 1, True), (192, 4 * 192 - 2, 1, 0, True),
              (192, 8 * 192 + 4, 8, 1, False), (160, 16 * 160, 8, 1, False), (192, 16 * 192, 13, 0, True)]


@pytest.mark.parametrize("K,taps,nch,variant,planar", CS16_CASES)
def test_cs16_bit_exact_ragged(native, K, taps, nch, variant, planar):
    """Interleaved and planar CS16, both variants, submits below K and below H and partial blocks."""
    S = 2
    freqs, fc = raster(nch)
    n = 2 * 1024 * K + K // 3
    x = np.random.default_rng(taps + variant).integers(-32768, 32768, size=(S, n, 2), dtype=np.int16)
    cuts = [1024 * K - 5, K // 2, taps - K - 1, 7]
    cuts.append(n - sum(cuts))
    with api.Context(K, S, nch, 3, flags=FLAG_CS16 | FLAG_FAST_FILTER, taps=taps) as ctx:
        for s in range(S):
            ctx.set_plan_cs16(s, freqs, variant, fc)
        got = run_stream_kind(ctx, "cs16", x, cuts, planar=planar)
        assert ctx.stats().fast_chan_launches >= 2
    for s in range(S):
        assert bits_equal(got[s], want_fast("cs16", x[s], K, taps, freqs, fc, variant).T.copy()), s


def test_u8_chunking_invariance(native, oracle):
    """One submit, block by block, random block counts with collects between, host / device alternated with an input
    buffer overwritten as soon as submit N+2 returns: the envelope equals the whole-stream restatement bit for bit and
    the frames are the same in every schedule."""
    K, taps, S, nblk, nch = 160, 8 * 160, 2, 8, 8
    fm, plan = _frames_plan(K, nblk, seed=31)
    fd, _, fc = api.plan(K, fm)
    one = synth.render_blocks(plan, 0, nblk).reshape(-1)
    iq = np.stack([one, np.roll(one, 4321 * 2)])
    bb = 2048 * K
    want = [want_fast("u8", iq[s], K, taps, fd, fc) for s in range(S)]

    def fresh():
        ctx = api.Context(K, S, nch, nblk, flags=FLAG_FAST_FILTER, taps=taps)
        for s in range(S):
            ctx.set_plan(s, fd)
        return ctx

    results = {}
    for name, sched in {"one": [nblk], "blocks": [1] * nblk, "random": [3, 1, 2, 2]}.items():
        with fresh() as ctx:
            p, env = 0, []
            for i, n in enumerate(sched):
                ctx.submit_host(np.ascontiguousarray(iq[:, p * bb:(p + n) * bb]), n)
                env.append(ctx.read_dm(n * 1024))
                if name == "random" and i % 2:
                    ctx.collect()
                p += n
            env = np.concatenate(env, axis=1)
            for s in range(S):
                assert bits_equal(env[s], want[s].T.copy()), (name, s)
            results[name] = ctx_result(ctx, S, nch)[0]
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
                ctx.copy_to_device(dev[((b - 2) // 2) % 3], np.full((S, pitch), 0xA5, dtype=np.uint8))
        results["mixed"] = ctx_result(ctx, S, nch)[0]
        for d in dev:
            ctx.device_free(d)
    assert len(results["one"]) >= 10
    for name, msgs in results.items():
        assert msgs == results["one"], name


def test_reset_restarts_history(native):
    """After a mid-run acb_reset the first ceil(H/K) rows omit the terms before the new start (u8: not the zero bytes of
    the cleared history), on both input kinds."""
    K, taps, nch = 160, 5 * 160 + 3, 8
    freqs, fc = raster(nch)
    rng = np.random.default_rng(9)
    a, b = rng.integers(0, 256, size=(2, 1, 2048 * K), dtype=np.uint8)
    with api.Context(K, 1, nch, 1, flags=FLAG_FAST_FILTER, taps=taps) as ctx:
        ctx.set_plan_at(0, freqs, fc)
        ctx.submit_host(a, 1)
        ctx.sync()
        ctx.reset()
        ctx.submit_host(b, 1)
        got = ctx.read_dm(1024)[0]
    assert bits_equal(got, want_fast("u8", b[0], K, taps, freqs, fc).T.copy())
    xa, xb = rng.integers(-32768, 32768, size=(2, 1, 3000 * K, 2), dtype=np.int16)
    with api.Context(K, 1, nch, 3, flags=FLAG_CS16 | FLAG_FAST_FILTER, taps=taps) as ctx:
        ctx.set_plan_cs16(0, freqs, 0, fc)
        run_stream_kind(ctx, "cs16", xa, [1000 * K + 17])
        ctx.sync()
        ctx.reset()
        got = run_stream_kind(ctx, "cs16", xb, [7, K - 7, 2999 * K])[0]
    assert bits_equal(got, want_fast("cs16", xb[0], K, taps, freqs, fc, 0).T.copy())


def _msgs(ctx):
    ctx.sync()
    return sorted((m.stream, m.chn, m.len, m.err, bytes(m.txt[:m.len]), bytes(m.crc), m.pos, m.block) for m in ctx.drain())


def test_messages_equal_exact_form(native):
    """4 streams x 8 channels x 8 blocks at 8K taps, and the weak-channel fixture: the same messages as an exact taps > K
    context on the same input; on the weak channel every frame decodes with err = 0."""
    K, taps, S, nblk, nch = 160, 8 * 160, 4, 8, 8
    fm, plan = _frames_plan(K, nblk, seed=41)
    fd = api.plan(K, fm)[0]
    one = synth.render_blocks(plan, 0, nblk).reshape(-1)
    iq = np.stack([np.roll(one, 999 * 2 * s) for s in range(S)])
    out = {}
    for flags in (0, FLAG_FAST_FILTER):
        with api.Context(K, S, nch, nblk, flags=flags, taps=taps) as ctx:
            for s in range(S):
                ctx.set_plan(s, fd)
            ctx.submit_host(iq, nblk)
            out[flags] = _msgs(ctx)
            assert (ctx.stats().fast_chan_launches > 0) == (flags != 0)
    assert out[0] == out[FLAG_FAST_FILTER] and len(out[0]) >= 20
    iq, fm, sent = weak_strong_scenario(K)
    nblk = iq.size // (2048 * K)
    fd = api.plan(K, fm)[0]
    for flags in (0, FLAG_FAST_FILTER):
        with api.Context(K, 1, 2, nblk, flags=flags, taps=8 * K) as ctx:
            ctx.set_plan(0, fd)
            ctx.submit_host(iq.reshape(1, -1), nblk)
            out[flags] = [m for m in _msgs(ctx) if m[1] == 0]
    assert out[0] == out[FLAG_FAST_FILTER] and len(out[0]) == len(sent) and all(m[3] == 0 for m in out[0])


def test_fallbacks_run_the_exact_kernel(native):
    """acb_set_wf tables, a plan off the raster, u8 at K = 200 and real input take the exact kernel (envelope bit-exact to
    orc_channelize_ovl*, no fast launch); at taps <= K the flag changes nothing."""
    rng = np.random.default_rng(3)
    nch = 8

    def u8_run(K, taps, plan_fn):
        x = rng.integers(0, 256, size=(1, 2048 * K), dtype=np.uint8)
        with api.Context(K, 1, nch, 1, flags=FLAG_FAST_FILTER, taps=taps) as ctx:
            wf = plan_fn(ctx)
            ctx.submit_host(x, 1)
            got = ctx.read_dm(1024)[0]
            ctx.sync()
            assert ctx.stats().fast_chan_launches == 0
        return got, x[0], wf

    K, taps = 160, 4 * 160
    freqs, fc = raster(nch)
    wf_tab = rand_tables(rng, nch, taps)
    got, x, _ = u8_run(K, taps, lambda c: c.set_wf(0, wf_tab))
    assert bits_equal(got, ovl_refs.channelize_ovl(x, K, wf_tab).T.copy())
    off = [f + 12_500 for f in freqs]                      # odd number of 12.5 kHz steps: off the fast raster
    got, x, _ = u8_run(K, taps, lambda c: c.set_plan_at(0, off, fc))
    L = api.load()
    wf_off = np.empty((nch, 2 * taps), dtype=np.float32)
    for i, f in enumerate(off):
        L.acb_build_wf_lp(L.acb_stored_fr(f), fc, K, taps, wf_off[i].ctypes.data)
    assert bits_equal(got, ovl_refs.channelize_ovl(x, K, wf_off).T.copy())
    fm = synth.DEFAULT_FREQS_MHZ
    fd200, _, _ = api.plan(200, fm)
    got, x, _ = u8_run(200, 2 * 200, lambda c: c.set_plan(0, fd200))
    assert bits_equal(got, ovl_refs.channelize_ovl(x, 200, api.build_wf_lp(200, 400, fm)).T.copy())
    # real input
    K = 200
    x = (rng.standard_normal((1, 2 * 1024 * K)) * 100).astype(np.float32)
    with api.Context(K, 1, nch, 2, flags=FLAG_REAL | FLAG_FAST_FILTER, taps=4 * K) as ctx:
        fda, _, _ = api.air_plan(K * 12500, fm)
        ctx.set_plan_air(0, fda)
        got = run_stream_kind(ctx, "real", x, [x.shape[1]])[0]
        assert ctx.stats().fast_chan_launches == 0
    assert bits_equal(got, ovl_refs.channelize_ovl_real(x[0], K, api.build_wf_air_lp(K * 12500, 4 * K, fm)).T.copy())
    # taps <= K: the flag changes nothing (taps = K with and without it, the boxcar's envelope)
    K = 160
    x = rng.integers(0, 256, size=(1, 2048 * K), dtype=np.uint8)
    env = []
    for flags in (0, FLAG_FAST_FILTER):
        with api.Context(K, 1, nch, 1, flags=flags) as ctx:
            ctx.set_plan_at(0, freqs, fc)
            ctx.submit_host(x, 1)
            env.append(ctx.read_dm(1024))
            ctx.sync()
            assert ctx.stats().fast_chan_launches == 0
    assert bits_equal(env[0], env[1])


def test_multi_equals_one_context(native):
    """acb_multi, stream split and channel split, with the flag: message for message one fast context."""
    K, taps, nblk, S, nch = 160, 4 * 160 + 8, 4, 2, 8
    fm, plan = _frames_plan(K, nblk, seed=23)
    one = synth.render_blocks(plan, 0, nblk).reshape(-1)
    iq = np.stack([one, np.roll(one, 555 * 2)])
    fd = api.plan(K, fm)[0]
    with api.Context(K, S, nch, nblk, flags=FLAG_FAST_FILTER, taps=taps) as ctx:
        for s in range(S):
            ctx.set_plan(s, fd)
        ctx.submit_host(iq, nblk)
        ctx.sync()
        ref = [(m.stream, m.chn, m.len, m.err, bytes(m.txt[:m.len]), m.pos) for m in ctx.drain()]
        assert ctx.stats().fast_chan_launches == 1
    assert len(ref) >= 4
    for mode in (0, 1):
        with api.MultiContext(K, S, nch, nblk, [0, 0], mode=mode, flags=FLAG_FAST_FILTER, taps=taps) as mc:
            for s in range(S):
                mc.set_plan(s, fd)
            mc.submit_host(iq, nblk)
            mc.sync()
            got = [(m.stream, m.chn, m.len, m.err, bytes(m.txt[:m.len]), m.pos) for m in mc.drain()]
        assert got == ref, mode
