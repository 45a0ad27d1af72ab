"""Polyphase fast form of the overlapping-window channelizer for real input (ACB_FLAG_FAST_FILTER_REAL) on the GPU:
envelope bit-exact to its CPU restatement (orc_ovl_presum_real, then orc_channelize_rdft), invariant to how the stream is
cut into submits, messages identical to the exact form's, and the exact kernel wherever the fast form does not apply."""
import numpy as np
import pytest

import ovl_fast_real_refs
from acarsdec_b200 import api, synth
from common import bits_equal
from test_gpu_ovl import ctx_result, rand_tables, run_stream_kind
from test_ovl_fast_oracle import f64_rows
from test_ovl_fast_real_oracle import frames_plan, setup, weak_strong_real

pytestmark = pytest.mark.gpu

FLAG_REAL, FLAG_CS16, FLAG_FAST, FLAG_FAST_FILTER, FLAG_FAST_FILTER_REAL = 2, 4, 8, 16, 32
# on the raster; the first four are consecutive 12.5 kHz steps (every residue k mod 4), ten channels make two groups
FREQS_MHZ = (131.525, 131.5375, 131.55, 131.5625, 131.725, 131.825, 131.45, 131.475, 131.4875, 131.6)


def want_fast(oracle, x, K, taps, fm):
    _, h, k, tw, _ = setup(K, taps, fm)
    return ovl_fast_real_refs.channelize_ovl_rdft(oracle, x, K, h, k, tw)


def real_ctx(K, S, fm, max_blocks, taps, flags=FLAG_REAL | FLAG_FAST_FILTER_REAL):
    ctx = api.Context(K, S, len(fm), max_blocks, flags=flags, taps=taps)
    fd, fc, _ = api.air_plan(K * 12500, fm)
    for s in range(S):
        assert ctx.set_plan_air(s, fd) == fc
    return ctx


CASES = [(200, 16 * 200, 10), (200, 200 + 4, 3), (240, 2 * 240 + 3, 8), (400, 400 + 4, 1), (480, 4 * 480, 3),
         (800, 8 * 800, 10), (800, 16 * 800, 8)]


@pytest.mark.parametrize("K,taps,nch", CASES)
def test_bit_exact_ragged(native, oracle, K, taps, nch):
    """Two streams of different data, submits below K, below H, partial blocks and one of exactly max_blocks * 1024 rows:
    the envelope of both streams equals the restatement over the whole stream."""
    S, max_blocks = 2, 2
    fm = FREQS_MHZ[:nch]
    H = taps - K
    cuts = [K // 3, max(1, H - 1), 1024 * K + 13]
    fed = sum(cuts)
    cuts.append(max_blocks * 1024 * K - fed % K)                # carry + this = exactly max_blocks * 1024 rows
    cuts += [5 * K + 7, 3 * K]
    x = (np.random.default_rng(K + taps).standard_normal((S, sum(cuts))) * 50).astype(np.float32)
    with real_ctx(K, S, fm, max_blocks, taps) as ctx:
        got = run_stream_kind(ctx, "real", x, cuts)
        ctx.sync()
        st = ctx.stats()
        assert st.fast_chan_launches == st.chan_launches >= 4
    nout = sum(cuts) // K
    assert got.shape[1] == nout
    for s in range(S):
        assert bits_equal(got[s], want_fast(oracle, x[s], K, taps, fm).T.copy()), s


def test_chunking_invariance(native, oracle):
    """One submit, many small ones and a random schedule: identical envelope, messages and states, the envelope equal to
    the whole-stream restatement; the messages equal an exact taps > K context's on the same input."""
    K, taps, S = 200, 8 * 200, 2
    fm = synth.DEFAULT_FREQS_MHZ
    secs = 0.6
    n = int(secs * K * 12500)
    one = synth.render_real(frames_plan(K, fm, secs, seed=31, amp=(6.0, 14.0), gap=0.02), 0, n)
    x = np.stack([one, np.roll(one, 43210)])
    nout = n // K
    want = [want_fast(oracle, x[s], K, taps, fm) for s in range(S)]
    max_blocks = nout // 1024 + 2
    rng = np.random.default_rng(5)
    rand = []
    while sum(rand) < n:
        rand.append(int(min(rng.integers(1, 700 * K), n - sum(rand))))
    schedules = {"one": [n], "small": [37 * K + 11] * (n // (37 * K + 11)) + [n % (37 * K + 11)], "random": rand}
    results = {}
    for name, cuts in schedules.items():
        cuts = [c for c in cuts if c]
        with real_ctx(K, S, fm, max_blocks, taps) as ctx:
            env = run_stream_kind(ctx, "real", x, cuts)
            for s in range(S):
                assert bits_equal(env[s], want[s].T.copy()), (name, s)
            results[name] = ctx_result(ctx, S, len(fm))
    with real_ctx(K, S, fm, max_blocks, taps, flags=FLAG_REAL) as ctx:
        run_stream_kind(ctx, "real", x, [n])
        exact_msgs = ctx_result(ctx, S, len(fm))[0]
    assert len(results["one"][0]) >= 10
    for name, r in results.items():
        assert r == results["one"], name
    assert results["one"][0] == exact_msgs


def test_reset_restarts_history(native, oracle):
    """After a mid-run acb_reset the rows equal the restatement of the new input alone."""
    K, taps, fm = 400, 5 * 400 + 3, FREQS_MHZ[:8]
    rng = np.random.default_rng(9)
    a, b = (rng.standard_normal((2, 1, 1500 * K)) * 30).astype(np.float32)
    with real_ctx(K, 1, fm, 2, taps) as ctx:
        run_stream_kind(ctx, "real", a, [1000 * K + 17, 499 * K])
        ctx.sync()
        ctx.reset()
        got = run_stream_kind(ctx, "real", b, [7, K - 7, 3, 1499 * K - 3])[0]
    assert bits_equal(got, want_fast(oracle, b[0], K, taps, fm).T.copy())


@pytest.mark.parametrize("K,taps", [(200, 4 * 200), (800, 16 * 800)])
def test_any_scale(native, oracle, K, taps):
    """The same capture scaled by 2^-70 .. 2^70: bit-exact to the restatement, finite, within 1e-6 * S of float64."""
    fm = FREQS_MHZ[:8]
    n = 2 * 1024 * K + 5 * K
    x1 = synth.render_real(frames_plan(K, fm, n / (K * 12500), seed=77), 0, n)
    _, h, k, tw, w64 = setup(K, taps, fm)
    for e in (-70, -40, 0, 40, 70):
        x = x1 * np.float32(2.0 ** e)
        with real_ctx(K, 1, fm, 3, taps) as ctx:
            got = run_stream_kind(ctx, "real", x[None, :], [n])[0]
            ctx.sync()
            assert ctx.stats().fast_chan_launches == 1
        assert bits_equal(got, ovl_fast_real_refs.channelize_ovl_rdft(oracle, x, K, h, k, tw).T.copy()), e
        ideal, S = f64_rows(x.astype(np.float64).astype(np.complex128), K, w64)
        assert np.isfinite(got).all() and np.all(np.abs(got.T.astype(np.float64) - ideal) <= 1e-6 * S), e


def _env(K, taps, flags, x, plan_fn, nch=8):
    """(envelope, stats) of one context of the given flags fed x (1, n[, 2]) in two submits"""
    kind = "real" if flags & FLAG_REAL else "cs16"
    with api.Context(K, 1, nch, 2, flags=flags, taps=taps) as ctx:
        plan_fn(ctx)
        n = x.shape[1]
        got = run_stream_kind(ctx, kind, x, [n // 3, n - n // 3])
        ctx.sync()
        return got, ctx.stats()


def test_switch_runs_what_ran_before(native, oracle):
    """The new bit where the fast form does not apply: u8 and CS16 contexts, acb_set_wf tables, a plan off the raster,
    real K = 160 and 202, taps = K (alone and with ACB_FLAG_FAST_CHANNELIZER) — bit-identical envelope to the context
    without it and no extra fast launch.  With ACB_FLAG_FAST_FILTER as well, a real context runs the fast form."""
    rng = np.random.default_rng(3)
    nch = 8
    # u8
    K, taps = 160, 4 * 160
    fd, _, _ = api.plan(K, synth.DEFAULT_FREQS_MHZ)
    x = rng.integers(0, 256, size=(1, 2048 * K), dtype=np.uint8)
    env = []
    for flags in (0, FLAG_FAST_FILTER_REAL):
        with api.Context(K, 1, nch, 1, flags=flags, taps=taps) as ctx:
            ctx.set_plan(0, fd)
            ctx.submit_host(x, 1)
            env.append(ctx.read_dm(1024))
            ctx.sync()
            assert ctx.stats().fast_chan_launches == 0
    assert bits_equal(env[0], env[1])
    # CS16
    xc = rng.integers(-32768, 32768, size=(1, 1500 * K + 7, 2), dtype=np.int16)
    out = [_env(K, 2 * K + 3, FLAG_CS16 | f, xc, lambda c: c.set_plan_cs16(0, fd, 0)) for f in (0, FLAG_FAST_FILTER_REAL)]
    assert bits_equal(out[0][0], out[1][0]) and out[1][1].fast_chan_launches == 0
    # real input
    fm = synth.DEFAULT_FREQS_MHZ

    def air(K):
        fda = api.air_plan(K * 12500, fm)[0]
        return lambda c: c.set_plan_air(0, fda)

    def real_pair(K, taps, plan_fn, extra=0):
        xr = (rng.standard_normal((1, 1500 * K + 11)) * 100).astype(np.float32)
        return [_env(K, taps, FLAG_REAL | extra | f, xr, plan_fn) for f in (0, FLAG_FAST_FILTER_REAL)]

    wf = rand_tables(rng, nch, 4 * 200)
    off = [f + 5000 for f in api.air_plan(200 * 12500, fm)[0]]        # 5 kHz off the 12.5 kHz raster
    assert api.load().acb_fast_plan_air(np.asarray(off, np.uint32).ctypes.data, nch, 200,
                                        api.air_plan(200 * 12500, fm)[1], None, None) == 0
    for name, (K, taps, plan_fn) in {"set_wf": (200, 4 * 200, lambda c: c.set_wf(0, wf)),
                                     "off_raster": (200, 4 * 200, lambda c: c.set_plan_air(0, off)),
                                     "K160": (160, 4 * 160, air(160)), "K202": (202, 2 * 202, air(202)),
                                     "taps_K": (200, 200, air(200))}.items():
        a, b = real_pair(K, taps, plan_fn)
        assert bits_equal(a[0], b[0]) and b[1].fast_chan_launches == 0, name
    a, b = real_pair(200, 200, air(200), extra=FLAG_FAST)
    assert bits_equal(a[0], b[0]) and b[1].fast_chan_launches == a[1].fast_chan_launches == a[1].chan_launches > 0
    # ACB_FLAG_FAST_FILTER alone selects nothing on a real context; with the new bit the fast form runs
    K, taps = 240, 4 * 240
    xr = (rng.standard_normal((1, 1500 * K + 11)) * 100).astype(np.float32)
    alone = _env(K, taps, FLAG_REAL | FLAG_FAST_FILTER, xr, air(K))
    assert alone[1].fast_chan_launches == 0
    assert bits_equal(alone[0], _env(K, taps, FLAG_REAL, xr, air(K))[0])
    both = _env(K, taps, FLAG_REAL | FLAG_FAST_FILTER | FLAG_FAST_FILTER_REAL, xr, air(K))
    assert both[1].fast_chan_launches == both[1].chan_launches > 0
    n = (xr.shape[1] // K) * K
    assert bits_equal(both[0][0], want_fast(oracle, xr[0, :n], K, taps, fm).T.copy())


def test_weak_channel_next_to_strong_neighbour(native):
    """The real-input weak/strong fixture at 8K taps: the fast context decodes every weak frame with err = 0, the same
    frames as an exact context."""
    K = 200
    x, fm, sent = weak_strong_real(K)
    out = {}
    for flags in (FLAG_REAL, FLAG_REAL | FLAG_FAST_FILTER_REAL):
        with real_ctx(K, 1, fm, x.size // (1024 * K) + 2, 8 * K, flags=flags) as ctx:
            run_stream_kind(ctx, "real", x[None, :], [x.size])
            out[flags] = [m for m in ctx_result(ctx, 1, 2)[0] if m[1] == 0]
            assert (ctx.stats().fast_chan_launches > 0) == (flags != FLAG_REAL)
    assert out[FLAG_REAL] == out[FLAG_REAL | FLAG_FAST_FILTER_REAL]
    assert len(out[FLAG_REAL]) == len(sent) and all(m[3] == 0 for m in out[FLAG_REAL])
