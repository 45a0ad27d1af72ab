"""The short channel filter (taps < K, tables from acb_set_wf) on the streaming front-ends on the GPU: float32 real input
(the 4-row kernel and ACB_REAL_ROWS=2), CS16 interleaved and CS16 planar, envelope bit-exact to the definition
(tests/host/fir_stream_oracle.c: the FIRST `taps` samples of each row) under ragged submits, and end to end: frames and
every chain's state equal the oracle's demodulation of the definition's envelope."""
import numpy as np
import pytest

import fir_stream_refs as fsr
import refs
from acarsdec_b200 import api, synth
from common import bits_equal

pytestmark = pytest.mark.gpu

FLAG_REAL, FLAG_CS16 = 2, 4
KINDS = ("real", "rows2", "cs16", "planar")


def definition(kind, x, K, wf):
    return fsr.channelize_fir_real(x, K, wf) if kind in ("real", "rows2") else fsr.channelize_fir_cs16(x, K, wf)


def submit(ctx, kind, part):
    """One streaming submit of (nstreams, n[, 2]) rows (a view: its row pitch is the stream stride; the planar planes are
    split into rows 13 samples wider than the submit)."""
    if kind in ("real", "rows2"):
        return ctx.submit_real(part)
    if kind == "planar":
        S, n = part.shape[:2]
        planes = np.zeros((2, S, n + 13), dtype=np.int16)
        planes[0, :, :n], planes[1, :, :n] = part[..., 0], part[..., 1]
        return ctx.submit_cs16_planar(planes[0, :, :n], planes[1, :, :n])
    return ctx.submit_cs16(part)


def rand_input(kind, rng, S, n, pad=0):
    """(S, n[, 2]) input as a view into rows of n + pad samples: pad > 0 makes the stream stride larger than n."""
    if kind in ("real", "rows2"):
        return (rng.standard_normal((S, n + pad)) * 100).astype(np.float32)[:, :n]
    return rng.integers(-32768, 32768, size=(S, n + pad, 2), dtype=np.int16)[:, :n]


# taps: less than one 16-byte unit (1, 3), exactly one unit of real input (4), one past it (5), a 20 / 21-tap filter,
# K/2 + 1 and K - 1; nch cycles through one channel, a partial group of 8, one group, one past it and eight groups
TAPS = (1, 3, 4, 5, 20, 21, "K/2+1", "K-1")
NCH = (1, 5, 8, 9, 64)


@pytest.mark.parametrize("K", [64, 42])                      # K % 4 == 0 (pipeline kernel) and K % 4 != 0 (generic)
@pytest.mark.parametrize("kind", KINDS)
def test_envelope_bit_exact_ragged(native, kind, K, monkeypatch):
    """Two streams with different tables, submits below one row, ending exactly on a row, and one that crosses a 1024-row
    block (pipeline and generic kernel in one submit), the last one from rows wider than the submit (stream stride >
    sample count): every envelope row equals the definition over the whole stream."""
    if kind == "rows2":
        monkeypatch.setenv("ACB_REAL_ROWS", "2")
    flags = FLAG_REAL if kind in ("real", "rows2") else FLAG_CS16
    S = 2
    for i, taps in enumerate(TAPS):
        taps = K // 2 + 1 if taps == "K/2+1" else K - 1 if taps == "K-1" else taps
        nch = NCH[i % len(NCH)]
        rng = np.random.default_rng(K * 1000 + taps * 10 + KINDS.index(kind))
        wf = [(rng.standard_normal((nch, 2 * taps)) / np.sqrt(taps)).astype(np.float32) for _ in range(S)]
        cuts = [K // 3, K - K // 3, 1029 * K + 7, 300 * K + 11]
        x = rand_input(kind, rng, S, sum(cuts))
        last = rand_input(kind, rng, S, cuts[-1], pad=37)
        x[:, sum(cuts[:-1]):] = last
        with api.Context(K, S, nch, 2, flags=flags, taps=taps) as ctx:
            for s in range(S):
                ctx.set_wf(s, wf[s])
            got, p = [], 0
            for j, n in enumerate(cuts):
                part = last if j == len(cuts) - 1 else x[:, p:p + n]
                rows = submit(ctx, kind, part)
                p += n
                if rows:
                    got.append(ctx.read_dm(rows))
            got = np.concatenate(got, axis=1)
        assert got.shape[1] == sum(cuts) // K
        for s in range(S):
            assert bits_equal(got[s], definition(kind, x[s], K, wf[s]).T.copy()), (taps, nch, s)


def _fixture(kind, K, nblk, seed, nch=8):
    """(input (1, n[, 2]), truncated planner tables (nch, 2*taps)) for a stream with frames on every channel: the planners'
    K-tap tables cut to their first 3K/4 + 1 taps (a shorter boxcar: a wider pass band, the same mixer)."""
    fm = synth.DEFAULT_FREQS_MHZ[:nch]
    n = nblk * 1024 * K
    taps = 3 * K // 4 + 1
    if kind in ("real", "rows2"):
        rate = K * 12500
        fd, fc, _ = api.air_plan(rate, fm)
        plan = synth.make_plan(K, fm, fc, seconds=n / rate, seed=seed, msgs_per_chan_per_sec=3.0, text_len=(5, 30),
                               amp=(6.0, 12.0))
        plan = synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, bursts=plan.bursts, seed=plan.seed)
        x = synth.render_real(plan, 0, n).reshape(1, -1)
        wf = api.build_wf_air(rate, fm)
    else:
        fd, _, fc = api.plan(K, fm)
        plan = synth.make_plan(K, fm, fc, seconds=n / (K * 12500), seed=seed, msgs_per_chan_per_sec=3.0, text_len=(5, 30),
                               amp=(6.0, 12.0))
        x = synth.render_cs16(plan, 0, n).reshape(1, n, 2)
        wf = api.build_wf_cs16(0 if kind == "cs16" else 1, K, fd, fc)
    return x, np.ascontiguousarray(wf[:, :2 * taps]), taps


@pytest.mark.parametrize("kind", ["real", "cs16", "planar"])
def test_frames_and_states_end_to_end(native, oracle, kind):
    K = 200 if kind == "real" else 160
    nblk, nch = 6, 8
    x, wf, taps = _fixture(kind, K, nblk, seed=40 + KINDS.index(kind))
    n = x.shape[1]
    cuts = [K - 3, 5, 2 * 1024 * K + 11]
    cuts.append(n - sum(cuts))
    with api.Context(K, 1, nch, nblk, flags=FLAG_REAL if kind == "real" else FLAG_CS16, taps=taps) as ctx:
        ctx.set_wf(0, wf)
        p, env = 0, []
        for c in cuts:
            rows = submit(ctx, kind, x[:, p:p + c])
            p += c
            if rows:
                env.append(ctx.read_dm(rows))
        ctx.sync()
        got = sorted(m.as_tuple() for m in ctx.drain())
        states = [ctx.get_state(0, c).vec() for c in range(nch)]
    dm = definition(kind, x[0], K, wf)
    assert bits_equal(np.concatenate(env, axis=1)[0], dm.T.copy())
    sink = refs.Sink()
    chans = []
    for c in range(nch):
        ch = oracle.new_chan(c)
        oracle.demod(ch, dm[c], sink)
        chans.append(ch.vec())
    want = sorted((f.chn, f.len, f.err, bytes(f.txt[:f.len]), bytes(f.crc))
                  for f in (oracle.fec(m) for m in sink.msgs()) if f is not None)
    assert got == want and len(want) >= 5
    assert states == chans
