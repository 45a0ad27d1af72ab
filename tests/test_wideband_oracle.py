"""CPU checks of the wideband fast form (ACB_FLAG_FAST_WIDEBAND): its single twiddle table E (acb_wb_twiddles) against
the fast planners' per-channel twiddles, and the two definitions it is held to bit for bit on the GPU — the folded
boxcar form (orc_channelize_dft8{,_cs16}) and the polyphase form (orc_channelize_ovl_fast{,_cs16}) — at wide shapes:
against the exact definition and the definition in float64 per output row relative to S = sum |x| * |w|, and the frames
the oracle demodulator decodes from each envelope."""
import ctypes as C

import numpy as np
import pytest

import ovl_fast_refs
import ovl_refs
from acarsdec_b200 import api, synth
from test_ovl_fast_oracle import f64_rows

TABLE_EPS = 1e-5          # (a) fast vs exact form
IDEAL_EPS = 1e-6          # (b) fast vs the float64 definition
FC = 120_000_000


@pytest.fixture(scope="module")
def lib():
    from acarsdec_b200 import build
    build.build()
    L = api.load()
    L.acb_wb_twiddles.restype = C.c_int
    L.acb_wb_twiddles.argtypes = [C.c_int, C.c_int, C.c_void_p]
    return L


def wb_table(L, variant, K):
    """E (2K - 1, 2) float32, E[r + K - 1] for r in (-K, K); variant -1: u8"""
    E = np.zeros((2 * K - 1, 2), dtype=np.float32)
    assert L.acb_wb_twiddles(variant, K, E.ctypes.data) == 1
    return E


def raster(nch, step=1):
    """nch channels at 25 kHz * step apart, alternating above and below FC: k = +-2 step, +-4 step, ..."""
    j = np.array([(i // 2 + 1) * (1 if i % 2 == 0 else -1) for i in range(nch)]) * step
    return [int(FC + 25_000 * v) for v in j]


def planner(L, kind, variant, K, freqs):
    f = np.asarray(freqs, dtype=np.uint32)
    k = np.zeros(len(f), dtype=np.int32)
    tw = np.zeros((len(f), K // 4, 2), dtype=np.float32)
    if kind == "u8":
        ok = L.acb_fast_plan(f.ctypes.data, len(f), K, FC, k.ctypes.data, tw.ctypes.data)
    else:
        ok = L.acb_fast_plan_cs16(variant, f.ctypes.data, len(f), K, FC, k.ctypes.data, tw.ctypes.data)
    assert ok == 1
    return k, tw


@pytest.mark.parametrize("K", [56, 160, 192, 800, 1600, 2048])
@pytest.mark.parametrize("kind,variant", [("u8", -1), ("cs16", 0), ("cs16", 1)])
def test_table_reproduces_planners(lib, K, kind, variant):
    """Every admissible bin k (even, non-zero, |k| < K/2): E[(k*n2) % K] is the planner's twiddle T_k[n2], bit for bit,
    for every n2 < K/4."""
    E = wb_table(lib, variant, K)
    freqs = raster(2 * (K // 4 - 1))
    k, tw = planner(lib, kind, variant, K, freqs)
    assert sorted(k.tolist()) == sorted([v for v in range(-(K // 2) + 2, K // 2, 2) if v != 0])
    n2 = np.arange(K // 4, dtype=np.int64)
    r = np.fmod(k.astype(np.int64)[:, None] * n2[None, :], K)        # C remainder: the sign of k
    assert np.array_equal(E[r + K - 1].view(np.uint32), tw.view(np.uint32))


def u8_inputs(K, n, rng):
    fm = synth.DEFAULT_FREQS_MHZ
    plan = synth.make_plan(K, fm, api.plan(K, fm)[2], seconds=(n // K + 1024) / 12500, seed=K, msgs_per_chan_per_sec=20.0)
    t = np.arange(n)
    sq = np.empty(2 * n, np.uint8)
    sq[0::2] = np.where((t // 7) % 2, 255, 0)
    sq[1::2] = np.where((t // 3) % 2, 0, 255)
    frames = synth.render_blocks(plan, 0, (n + 1024 * K - 1) // (1024 * K)).reshape(-1)[:2 * n]
    return {"frames": frames, "uniform": rng.integers(0, 256, 2 * n, dtype=np.uint8),
            "zeros": np.zeros(2 * n, np.uint8), "ones255": np.full(2 * n, 255, np.uint8), "square": sq}


def cs16_inputs(n, rng):
    sat = rng.choice(np.array([-32768, 32767], np.int16), size=(n, 2))
    dc = np.empty((n, 2), np.int16)
    dc[:, 0], dc[:, 1] = 16384, -16384
    return {"saturation": sat, "dc": dc, "uniform": rng.integers(-32768, 32768, size=(n, 2), dtype=np.int16)}


def fast_envelope(oracle, kind, x, K, taps, k, tw):
    """the definition k_channelize_wb is held to: orc_channelize_dft8* at taps = K, orc_channelize_ovl_fast* above"""
    if taps == K:
        return oracle.channelize_dft(x, K, k, tw, fold8=True) if kind == "u8" else oracle.channelize_dft8_cs16(x, K, k, tw)
    h = api.build_lowpass(K, taps)
    if kind == "u8":
        return ovl_fast_refs.channelize_ovl_fast(x, K, h, k, tw)
    return ovl_fast_refs.channelize_ovl_fast_cs16(x, K, h, k, tw)


def tables(L, kind, variant, K, taps, freqs):
    """(exact table (nch, 2*taps) of the planner, float64 weights (nch, taps))"""
    nch = len(freqs)
    wf = np.zeros((nch, 2 * taps), dtype=np.float32)
    for i, f in enumerate(freqs):
        if kind == "u8":
            fr = L.acb_stored_fr(f)
            (L.acb_build_wf_lp(fr, FC, K, taps, wf[i].ctypes.data) if taps > K else L.acb_build_wf(fr, FC, K, wf[i].ctypes.data))
        elif taps > K:
            L.acb_cs16_build_wf_lp(variant, f, FC, K, taps, wf[i].ctypes.data)
        else:
            L.acb_cs16_build_wf(variant, f, FC, K, wf[i].ctypes.data)
    k, _ = planner(L, kind, variant, K, freqs)
    scale = 1 / 127.5 if kind == "u8" else (1 / 32768 if variant == 0 else 0.25)
    h = api.build_lowpass(K, taps).astype(np.float64) if taps > K else np.full(K, 1.0 / K)
    i = np.arange(taps) - (taps - K)
    return wf, h[None, :] * np.exp(-2j * np.pi * np.outer(k, i) / K) * scale


MEASURED = {}


def check(name, got, exact, ideal, S):
    ea = np.abs(got.astype(np.float64) - exact) / np.maximum(S, 1e-300)
    eb = np.abs(got.astype(np.float64) - ideal) / np.maximum(S, 1e-300)
    for key, v in (("fast_vs_exact", ea), ("fast_vs_f64", eb)):
        MEASURED[key] = max(MEASURED.get(key, 0.0), float(v.max()))
    assert np.all(np.abs(got.astype(np.float64) - exact) <= TABLE_EPS * S), (name, float(ea.max()))
    assert np.all(np.abs(got.astype(np.float64) - ideal) <= IDEAL_EPS * S), (name, float(eb.max()))


SHAPES = [(800, 256), (1600, 256), (2048, 256), (192, 64)]
TAPS = ("K", "K+8", "2K+3", "8K", "16K")


def taps_of(K, t):
    return {"K": K, "K+8": K + 8, "2K+3": 2 * K + 3, "8K": 8 * K, "16K": 16 * K}[t]


def rows_of(K, taps):
    return (taps + K - 1) // K + 6           # every row past the first window is a full window


@pytest.mark.parametrize("K,nch", SHAPES)
@pytest.mark.parametrize("t", TAPS)
def test_u8_within_bars(lib, oracle, K, nch, t):
    taps = taps_of(K, t)
    freqs = raster(nch, step=max(1, (K // 2 - 2) // (2 * nch)))
    k, tw = planner(lib, "u8", -1, K, freqs)
    wf, w64 = tables(lib, "u8", -1, K, taps, freqs)
    n = rows_of(K, taps) * K
    for name, iq in u8_inputs(K, n, np.random.default_rng(K + taps)).items():
        got = fast_envelope(oracle, "u8", iq, K, taps, k, tw)
        exact = ovl_refs.channelize_ovl(iq, K, wf)
        xc = (iq[0::2].astype(np.float32) - np.float32(127.37)).astype(np.float64) + 1j * (iq[1::2].astype(np.float32) - np.float32(127.37))
        if taps == K:
            # the boxcar's definition is the reference's arithmetic on the mid-scale 127.5 (rtl.c:334-354)
            xc = (iq[0::2].astype(np.float64) - 127.5) + 1j * (iq[1::2].astype(np.float64) - 127.5)
            exact = oracle.channelize(iq, K, wf)
        ideal, S = f64_rows(xc, K, w64)
        check((name, K, nch, taps), got, exact, ideal, S)


@pytest.mark.parametrize("K,nch", SHAPES)
@pytest.mark.parametrize("t", TAPS)
@pytest.mark.parametrize("variant", [0, 1])
def test_cs16_within_bars(lib, K, nch, t, variant, oracle):
    taps = taps_of(K, t)
    freqs = raster(nch, step=max(1, (K // 2 - 2) // (2 * nch)))
    k, tw = planner(lib, "cs16", variant, K, freqs)
    wf, w64 = tables(lib, "cs16", variant, K, taps, freqs)
    n = rows_of(K, taps) * K
    for name, x in cs16_inputs(n, np.random.default_rng(K + taps + variant)).items():
        got = fast_envelope(oracle, "cs16", x, K, taps, k, tw)
        exact = ovl_refs.channelize_ovl_cs16(x, K, wf)
        ideal, S = f64_rows(x[:, 0].astype(np.float64) + 1j * x[:, 1], K, w64)
        check((name, K, nch, taps, variant), got, exact, ideal, S)


def test_report_measured_maxima():
    """The worst ratios |error| / S over the two tests above (DESIGN.md §4 quotes them)."""
    if not MEASURED:
        pytest.skip("the tolerance tests did not run in this session")
    print("\nwideband fast form, max |error|/S:", {k: f"{v:.3g}" for k, v in sorted(MEASURED.items())})
    assert MEASURED["fast_vs_exact"] <= TABLE_EPS and MEASURED["fast_vs_f64"] <= IDEAL_EPS


def wideband_fixture(K=1600, nch=256, nblk=8, weak=3.0, strong=30.0, noise=0.5, seed=5):
    """K = 1600 (20 MS/s), 256 adjacent 25 kHz channels around FC.  Two channels (FC + 500 kHz, FC - 1.5 MHz) carry
    frames at amplitude `weak`; the channel 25 kHz above each carries an AM voice carrier (+1 kHz off its centre) of
    amplitude `strong`, 10x the frames (20 dB), peaking at 2 * strong * 1.8 = 108 LSB together: no clipping.  Returns
    (iq (nblk*1024*K*2,) u8, freqs, the two busy channels, the frames sent on them)."""
    freqs = raster(nch)
    busy, loud = [38, 119], [40, 117]              # raster indices: j = 20 / 21 and j = -60 / -59 (25 kHz steps)
    assert all(freqs[b] + 25_000 == freqs[n] for b, n in zip(busy, loud))
    plan = synth.StreamPlan(K=K, freqs_hz=tuple(freqs[c] for c in busy), fc_hz=FC, seed=seed, noise_sigma=noise)
    rng = np.random.default_rng(seed)
    sent = []
    for ch in range(len(busy)):
        t = 0.05 + 0.07 * ch
        while t < nblk * 1024 / 12500 - 0.2:
            fr = synth.frame_bytes(synth.random_text(rng, 30))
            plan.bursts.append(synth.Burst(chan=ch, t0=t, frame=fr, amp=weak, phase=float(rng.uniform(0, 2 * np.pi))))
            sent.append((ch, fr))
            t += len(fr) * 8 / 2400 + 0.03
    fs, ns = K * 12500, nblk * 1024 * K
    tt = np.arange(ns, dtype=np.float64) / fs
    x = np.zeros(ns, dtype=np.complex128)
    for i, c in enumerate(loud):
        audio = 0.5 * np.sin(2 * np.pi * 400 * tt + i) + 0.3 * np.sin(2 * np.pi * 1100 * tt + 1) + 0.2 * np.sin(2 * np.pi * 2300 * tt + 2)
        x += strong * (1 + 0.8 * audio) * np.exp(2j * np.pi * (freqs[c] + 1000 - FC) * tt + 1j * i)
    del tt
    for b in plan.bursts:
        lo, hi, v = synth.burst_samples(plan, b, 0, ns)
        x[lo:hi] += v
    iq = np.empty(2 * ns)
    iq[0::2], iq[1::2] = x.real, x.imag
    iq += np.random.default_rng([seed, 9]).standard_normal(2 * ns) * noise
    return np.clip(np.floor(iq + 128.0), 0, 255).astype(np.uint8), freqs, busy, sent


def test_wideband_fixture_frames_identical(lib, oracle):
    """The K = 1600, 256-channel fixture, the two weak channels next to neighbours 20 dB stronger: the oracle decodes the
    same frames from the fast and the exact envelopes, with the boxcar and with an 8K filter; with the filter that is
    every frame sent, all with err = 0."""
    from test_ovl_fast_oracle import _frames
    K = 1600
    iq, freqs, busy, sent = wideband_fixture(K)
    assert int(iq.min()) > 0 and int(iq.max()) < 255
    sel = [freqs[c] for c in busy]
    k, tw = planner(lib, "u8", -1, K, sel)
    for taps in (K, 8 * K):
        wf, _ = tables(lib, "u8", -1, K, taps, sel)
        exact = ovl_refs.channelize_ovl(iq, K, wf) if taps > K else oracle.channelize(iq, K, wf)
        fast = fast_envelope(oracle, "u8", iq, K, taps, k, tw)
        decoded = 0
        for c in range(len(sel)):
            want = _frames(oracle, exact[c])
            assert _frames(oracle, fast[c]) == want, (taps, c)
            if taps > K:
                assert len(want) == sum(ch == c for ch, _ in sent) and all(m[2] == 0 for m in want), c
            decoded += len(want)
        if taps > K:
            assert decoded == len(sent) and decoded >= 4
