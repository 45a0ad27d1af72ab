"""Wideband fast form for real input (ACB_FLAG_FAST_WIDEBAND_REAL) on the GPU: k_channelize_wb_real's envelope bit-exact
to its definitions (orc_channelize_rdft at taps = K, orc_ovl_presum_real then orc_channelize_rdft at taps > K) at any
K % 8 == 0 and any channel count, the narrow kernels' envelope where they apply, invariant to how the stream is cut into
submits, messages identical to the exact form's, and what ran before wherever the form does not apply."""
import numpy as np
import pytest

import test_gpu_stream_stress as stress
from acarsdec_b200 import api, synth
from common import bits_equal
from test_gpu_ovl import ctx_result, rand_tables, run_stream_kind
from test_gpu_scale import nsm  # noqa: F401  (fixture)
from test_ovl_fast_real_oracle import frames_plan
from test_wideband_real_oracle import air_fc, air_freqs, fast_envelope, fast_plan_air, wideband_real_fixture

pytestmark = pytest.mark.gpu

FLAG_REAL, FLAG_CS16, FLAG_FAST, FLAG_FAST_FILTER_REAL = 2, 4, 8, 32
FLAG_WB, FLAG_WBR = api.FLAG_FAST_WIDEBAND, api.FLAG_FAST_WIDEBAND_REAL
WB_CTILE = 256                      # channels per channel tile (acb_internal.h)


def want(oracle, x, K, taps, freqs, sel=None):
    """the definition's envelope (nch, rows) of one stream; `sel`: only those channels"""
    k, tw = fast_plan_air(K, freqs)
    if sel is not None:
        k, tw = k[sel], tw[sel]
    return fast_envelope(oracle, x, K, taps, k, tw)


def wbr_ctx(K, S, fs, max_blocks, taps, flags=FLAG_REAL | FLAG_WBR):
    ctx = api.Context(K, S, len(fs[0]), max_blocks, flags=flags, taps=taps)
    for s in range(S):
        assert ctx.set_plan_air(s, fs[s]) == air_fc(fs[s])
    return ctx


CASES = [(56, 56, 13), (56, 4 * 56 + 3, 20), (200, 200, 40), (200, 16 * 200, 8), (800, 800, 200), (800, 2 * 800 + 3, 100),
         (1600, 1600, 300), (1600, 4 * 1600, 300), (1608, 2 * 1608 + 3, 64), (2048, 2048, 1), (2048, 16 * 2048, 300)]


@pytest.mark.parametrize("K,taps,nch", CASES)
def test_bit_exact_ragged(native, oracle, K, taps, nch):
    """Two streams on different bins, submits below K, below H, partial blocks and one of exactly max_blocks * 1024
    rows: the envelope of both streams equals the definition over the whole stream."""
    S, max_blocks = 2, 2
    fs = [air_freqs(K, nch, s) for s in range(S)]
    H = taps - K
    cuts = [K // 3, max(1, H - 1), 1024 * K + 13]
    cuts.append(max_blocks * 1024 * K - sum(cuts) % K)          # carry + this = exactly max_blocks * 1024 rows
    cuts += [5 * K + 7, 3 * K]
    x = (np.random.default_rng(K + taps + nch).standard_normal((S, sum(cuts))) * 50).astype(np.float32)
    with wbr_ctx(K, S, fs, max_blocks, taps) as ctx:
        got = run_stream_kind(ctx, "real", x, cuts)
        ctx.sync()
        st = ctx.stats()
        assert st.fast_chan_launches == st.chan_launches >= 4
    assert got.shape[1] == sum(cuts) // K
    for s in range(S):
        assert bits_equal(got[s], want(oracle, x[s], K, taps, fs[s]).T.copy()), s


# on the raster; the first four are consecutive 12.5 kHz steps (every residue k mod 4)
NARROW_FM = (131.525, 131.5375, 131.55, 131.5625, 131.725, 131.825, 131.45, 131.475, 131.4875, 131.6)


@pytest.mark.parametrize("K", [200, 240, 400, 480, 800])
@pytest.mark.parametrize("taps_mul", [1, 4])
def test_same_envelope_as_narrow_kernels(native, K, taps_mul):
    """At the five Airspy K with 8 and 10 channels the new bit alone gives the envelope of ACB_FLAG_FAST_CHANNELIZER
    (taps = K) and of ACB_FLAG_FAST_FILTER_REAL (taps > K) bit for bit; with both bits the narrow kernel runs."""
    taps = taps_mul * K
    narrow = FLAG_FAST if taps == K else FLAG_FAST_FILTER_REAL
    x = (np.random.default_rng(K + taps).standard_normal((1, 2500 * K + 11)) * 80).astype(np.float32)
    for nch in (8, 10):
        fd = api.air_plan(K * 12500, NARROW_FM[:nch])[0]
        env = {}
        for flags in (narrow, FLAG_WBR, narrow | FLAG_WBR):
            with wbr_ctx(K, 1, [fd], 2, taps, flags=FLAG_REAL | flags) as ctx:
                env[flags] = run_stream_kind(ctx, "real", x, [1500 * K + 7, x.shape[1] - 1500 * K - 7])
                ctx.sync()
                st = ctx.stats()
                assert st.fast_chan_launches == st.chan_launches == 2
        assert bits_equal(env[narrow], env[FLAG_WBR]), nch
        assert bits_equal(env[narrow], env[narrow | FLAG_WBR]), nch


def test_chunking_invariance_and_reset(native, oracle):
    """One submit, many small ones and a seeded random schedule: identical envelope, messages and states, the envelope
    equal to the whole-stream definition and the messages equal to an exact context's.  After a mid-run acb_reset the
    rows equal the definition of the new input alone."""
    K, taps, S = 800, 4 * 800 + 3, 2
    fm = synth.DEFAULT_FREQS_MHZ
    fd = api.air_plan(K * 12500, fm)[0]
    secs = 0.5
    n = int(secs * K * 12500)
    one = synth.render_real(frames_plan(K, fm, secs, seed=41, amp=(6.0, 14.0), gap=0.02), 0, n)
    x = np.stack([one, np.roll(one, 54321)])
    wants = [want(oracle, x[s], K, taps, fd) for s in range(S)]
    max_blocks = n // K // 1024 + 2
    rng = np.random.default_rng(6)
    rand = []
    while sum(rand) < n:
        rand.append(int(min(rng.integers(1, 700 * K), n - sum(rand))))
    schedules = {"one": [n], "small": [37 * K + 11] * (n // (37 * K + 11)) + [n % (37 * K + 11)], "random": rand}
    results = {}
    for name, cuts in schedules.items():
        cuts = [c for c in cuts if c]
        with wbr_ctx(K, S, [fd] * S, max_blocks, taps) as ctx:
            env = run_stream_kind(ctx, "real", x, cuts)
            for s in range(S):
                assert bits_equal(env[s], wants[s].T.copy()), (name, s)
            results[name] = ctx_result(ctx, S, len(fm))
            assert ctx.stats().fast_chan_launches == ctx.stats().chan_launches
    with wbr_ctx(K, S, [fd] * S, max_blocks, taps, flags=FLAG_REAL) as ctx:
        run_stream_kind(ctx, "real", x, [n])
        exact_msgs = ctx_result(ctx, S, len(fm))[0]
    assert len(results["one"][0]) >= 10
    for name, r in results.items():
        assert r == results["one"], name
    assert results["one"][0] == exact_msgs
    # reset mid-run
    rng = np.random.default_rng(9)
    a, b = (rng.standard_normal((2, 1, 1500 * K)) * 30).astype(np.float32)
    with wbr_ctx(K, 1, [fd], 2, taps) as ctx:
        run_stream_kind(ctx, "real", a, [1000 * K + 17, 499 * K])
        ctx.sync()
        ctx.reset()
        got = run_stream_kind(ctx, "real", b, [7, K - 7, 3, 1499 * K - 3])[0]
    assert bits_equal(got, want(oracle, b[0], K, taps, fd).T.copy())


def test_pipelined_ragged_walk(native, oracle, monkeypatch):
    """tests/test_gpu_stream_stress.py's seeded random walk (pipelined ragged submits, collects, syncs, resets, sources
    overwritten as soon as the input-lifetime rule frees them) for a real-input context at taps > K with the new bit
    alone, against the definition."""
    name = "real-gt-wideband-real"
    monkeypatch.setitem(stress.CASES, name, stress.Case("real", "gt", FLAG_WBR, group=(stress.GROUP_OUTPUTS, 1024)))
    stress.test_stream_random_walk(native, oracle, name)


@pytest.mark.parametrize("K,taps,nch", [(1600, 8 * 1600, 64), (800, 800, 100)])
def test_any_scale(native, oracle, K, taps, nch):
    """The same input scaled by 2^-70 .. 2^70: bit-exact to the definition and finite."""
    fs = [air_freqs(K, nch)]
    n = 2 * 1024 * K + 5 * K
    x1 = synth.render_real(frames_plan(K, (131.525, 131.5375, 131.55, 131.5625), n / (K * 12500) + 0.05, seed=77), 0, n)
    x1 += (np.random.default_rng(K).standard_normal(n) * 0.1).astype(np.float32)
    for e in (-70, -40, 0, 40, 70):
        x = x1 * np.float32(2.0 ** e)
        with wbr_ctx(K, 1, fs, 3, taps) as ctx:
            got = run_stream_kind(ctx, "real", x[None, :], [n])[0]
            ctx.sync()
            assert ctx.stats().fast_chan_launches == 1
        assert np.isfinite(got).all() and bits_equal(got, want(oracle, x, K, taps, fs[0]).T.copy()), e


@pytest.mark.parametrize("taps_mul", [1, 8])
def test_messages_and_states_equal_exact_form(native, taps_mul):
    """The K = 1600, 160-channel real fixture (two weak channels next to neighbours 20 dB stronger): the same messages
    (stream, channel, text, CRC, position, block) and every chain in the same framing state as an exact context; with the
    8K filter every frame sent on the weak channels decodes with err = 0."""
    K = 1600
    x, freqs, busy, sent = wideband_real_fixture(K)
    out = {}
    for flags in (FLAG_REAL, FLAG_REAL | FLAG_WBR):
        with wbr_ctx(K, 1, [freqs], x.size // (1024 * K) + 2, taps_mul * K, flags=flags) as ctx:
            run_stream_kind(ctx, "real", x[None, :], [x.size])
            ctx.sync()
            msgs = sorted((m.stream, m.chn, m.len, m.err, bytes(m.txt[:m.len]), bytes(m.crc), m.pos, m.block) for m in ctx.drain())
            out[flags] = (msgs, [ctx.get_state(0, c).Acarsstate for c in range(len(freqs))])
            assert (ctx.stats().fast_chan_launches > 0) == (flags != FLAG_REAL)
    assert out[FLAG_REAL] == out[FLAG_REAL | FLAG_WBR]
    weak = [m for m in out[FLAG_REAL][0] if m[1] in busy]
    if taps_mul > 1:
        assert len(weak) == len(sent) >= 4 and all(m[3] == 0 for m in weak)


def test_fallbacks_run_what_ran_before(native):
    """acb_set_wf tables, a plan off the raster, taps < K, K % 8 != 0, the bit on u8 and CS16 contexts, and
    ACB_FLAG_FAST_WIDEBAND alone on a real context: no fast launch, and the envelope of a context without the bit."""
    rng = np.random.default_rng(3)
    nch = 16

    def real_env(K, taps, plan_fn, flags):
        x = (np.random.default_rng(K + taps).standard_normal((1, 1500 * K + 11)) * 100).astype(np.float32)
        with api.Context(K, 1, nch, 2, flags=FLAG_REAL | flags, taps=taps) as ctx:
            plan_fn(ctx)
            got = run_stream_kind(ctx, "real", x, [x.shape[1] // 3, x.shape[1] - x.shape[1] // 3])
            ctx.sync()
            return got, ctx.stats().fast_chan_launches

    K = 800
    freqs = air_freqs(K, nch)
    off = [f + 5000 for f in freqs]                       # 5 kHz off the 12.5 kHz raster
    assert api.load().acb_fast_plan_air(np.asarray(off, np.uint32).ctypes.data, nch, K, air_fc(off), None, None) == 0
    wf_tab, wf_short = rand_tables(rng, nch, 2 * K), rand_tables(rng, nch, K - 8)
    cases = {"set_wf": (K, 2 * K, lambda c: c.set_wf(0, wf_tab)), "off_raster": (K, 2 * K, lambda c: c.set_plan_air(0, off)),
             "taps_lt_K": (K, K - 8, lambda c: c.set_wf(0, wf_short)),
             "K204": (204, 2 * 204, lambda c: c.set_plan_air(0, air_freqs(204, nch)))}
    for name, (K_, taps, fn) in cases.items():
        ref, _ = real_env(K_, taps, fn, 0)
        for flags in (FLAG_WBR, FLAG_WB):
            got, launches = real_env(K_, taps, fn, flags)
            assert launches == 0 and bits_equal(got, ref), (name, flags)
    # ACB_FLAG_FAST_WIDEBAND alone on a real context that the new bit would take
    ref, _ = real_env(K, 2 * K, lambda c: c.set_plan_air(0, freqs), 0)
    got, launches = real_env(K, 2 * K, lambda c: c.set_plan_air(0, freqs), FLAG_WB)
    assert launches == 0 and bits_equal(got, ref)
    # u8 and CS16 contexts: the new bit changes nothing
    from test_gpu_wideband import freqs_for
    from test_wideband_oracle import FC
    fu = freqs_for(K, nch)
    xu = rng.integers(0, 256, size=(1, 2048 * K), dtype=np.uint8)
    xc = rng.integers(-32768, 32768, size=(1, 1500 * K + 7, 2), dtype=np.int16)
    for base in (0, FLAG_WB):
        env = []
        for flags in (base, base | FLAG_WBR):
            with api.Context(K, 1, nch, 1, flags=flags, taps=2 * K) as ctx:
                ctx.set_plan_at(0, fu, FC)
                ctx.submit_host(xu, 1)
                env.append(ctx.read_dm(1024))
                ctx.sync()
                env.append(ctx.stats().fast_chan_launches)
            with api.Context(K, 1, nch, 2, flags=FLAG_CS16 | flags, taps=2 * K) as ctx:
                ctx.set_plan_cs16(0, fu, 0, FC)
                env.append(run_stream_kind(ctx, "cs16", xc, [xc.shape[1]]))
                env.append(ctx.stats().fast_chan_launches)
        assert bits_equal(env[0], env[4]) and bits_equal(env[2], env[6]), base
        assert env[1] == env[5] == (1 if base else 0) and env[3] == env[7] == (1 if base else 0), base


# ------------------------------------------------------------------ production launch sizes

def wbr_rows(K):
    """kernels.cu (wbr_rows): rows per tile, the most (a multiple of 4, at most 32) that leaves two CTAs per SM"""
    return min(32, (113 * 1024 - 8 * K) // (4 * K) // 4 * 4)


def wbr_tiles_per_cta(K, nsamp, nstreams, nch, nsm):
    """kernels.cu (wb_tiles_per_cta, shared with k_channelize_wb): tiles per CTA of a k_channelize_wb_real launch"""
    tiles = -(-nsamp // wbr_rows(K)) * nstreams * -(-nch // WB_CTILE)
    return max(1, min(8, tiles // (8 * nsm)))


def test_restated_heuristics_at_h100_size():
    assert wbr_rows(800) == 32 and wbr_rows(848) == 32 and wbr_rows(856) == 28 and wbr_rows(1600) == 16 and wbr_rows(1808) == 12
    assert wbr_rows(2048) == 12 and wbr_rows(56) == 32
    assert wbr_tiles_per_cta(800, 12 * 1024 - 5, 8, 16, 132) == 2
    assert wbr_tiles_per_cta(2048, 1024, 2, 300, 132) == 1


def subset(k, extra=10, seed=0):
    """channels covering every column (k mod 4 = 0, 2, odd) and both signs of the odd ones in every channel tile, plus
    a few at random"""
    sel = set()
    for z in range(0, len(k), WB_CTILE):
        kz = k[z:z + WB_CTILE]
        for r in range(4):
            idx = np.flatnonzero(kz % 4 == r)
            if len(idx):
                sel.update((z + idx[[0, -1]]).tolist())
    sel.update(np.random.default_rng(seed).choice(len(k), size=min(extra, len(k)), replace=False).tolist())
    return sorted(sel)


@pytest.mark.parametrize("K,taps,nch,S,want_tpc", [(800, 800, 16, 8, lambda t: 2 <= t < 8),
                                                    (2048, 2 * 2048 + 3, 300, 2, lambda t: t >= 2)],
                         ids=["K800-16ch-tpc2to7", "K2048-300ch-tpc2plus"])
def test_several_tiles_per_cta(native, oracle, nsm, K, taps, nch, S, want_tpc):
    """A submit sized from the restated rule to run several tiles per CTA, its last CTA short and ending in a partial
    tile; at K = 2048 (12-row tiles) with 300 channels, two channel tiles: bit-exact to the definition over every
    residue class and both channel tiles, and equal to one-tile-per-CTA submits of the same stream."""
    T = wbr_rows(K)
    rows = next(r for r in range(T + 1, 64 * 1024)
                if want_tpc(wbr_tiles_per_cta(K, r, S, nch, nsm))
                and r % (wbr_tiles_per_cta(K, r, S, nch, nsm) * T) and r % T)
    small = 1
    while wbr_tiles_per_cta(K, small + 1, S, nch, nsm) == 1 and small < rows:
        small += 1
    max_blocks = -(-rows // 1024)
    fs = [air_freqs(K, nch, s % 2) for s in range(S)]
    x = (np.random.default_rng(K + nch).standard_normal((S, rows * K)) * 20).astype(np.float32)
    with wbr_ctx(K, S, fs, max_blocks, taps) as ctx:
        big = run_stream_kind(ctx, "real", x, [rows * K])
    with wbr_ctx(K, S, fs, max_blocks, taps) as ctx:
        pieces = [small * K] * (rows // small) + ([rows % small * K] if rows % small else [])
        parts = run_stream_kind(ctx, "real", x, pieces)
    assert bits_equal(big, parts)
    for s in range(S):
        k, _ = fast_plan_air(K, fs[s])
        sel = subset(k, seed=s) if nch > 64 else list(range(nch))
        assert bits_equal(big[s][:, sel], want(oracle, x[s], K, taps, fs[s], sel).T.copy()), s
