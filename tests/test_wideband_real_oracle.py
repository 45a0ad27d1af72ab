"""CPU checks of the wideband fast form for real input (ACB_FLAG_FAST_WIDEBAND_REAL): the real variant of its single
twiddle table E (acb_wb_twiddles) against acb_fast_plan_air's per-channel twiddles, and the two definitions it is held to
bit for bit on the GPU — orc_channelize_rdft at taps = K, orc_ovl_presum_real then orc_channelize_rdft at taps > K — at
wide shapes: against the exact definition and the definition in float64 per output row relative to S = sum |x| * |w|,
and the frames the oracle demodulator decodes from each envelope."""
import ctypes as C

import numpy as np
import pytest

import ovl_fast_real_refs
import ovl_refs
from acarsdec_b200 import api, synth
from test_ovl_fast_oracle import f64_rows
from test_ovl_fast_real_oracle import _frames, frames_plan

TABLE_EPS = 1e-5          # (a) fast vs exact form
IDEAL_EPS = 1e-6          # (b) fast vs the float64 definition
FCR = 131_500_000         # on the 12.5 kHz raster
WB_TW_REAL = 2            # acb_wb_twiddles' real-input variant (acb_internal.h: ACB_WB_TW_REAL)


@pytest.fixture(scope="module")
def lib():
    from acarsdec_b200 import build
    build.build()
    L = api.load()
    L.acb_wb_twiddles.restype = C.c_int
    L.acb_wb_twiddles.argtypes = [C.c_int, C.c_int, C.c_void_p]
    return L


def wb_table(L, K):
    """E (2K - 1, 2) float32, E[r + K - 1] for r in (-K, K), real-input variant"""
    E = np.zeros((2 * K - 1, 2), dtype=np.float32)
    assert L.acb_wb_twiddles(WB_TW_REAL, K, E.ctypes.data) == 1
    return E


def air_freqs(K, nch, shift=0):
    """nch channels (Hz) on the 12.5 kHz raster around FCR, as far apart as the real band allows: offsets d of about
    round(linspace(-D, D - 1, nch)) raster steps, D = K/4 - 1 - shift, so acb_air_choose_fc picks about FCR and the bins
    k = K/4 - d lie in (0, K/2 + 3).  Where the spacing is 4 steps or more, channel i moves down to the offset = i mod 4,
    so that every residue k mod 4 occurs; closer spacings mix the residues themselves.  `shift` gives another stream
    other bins."""
    D = K // 4 - 1 - shift
    d = np.rint(np.linspace(-D, D - 1, nch)).astype(np.int64)
    if nch > 1 and (2 * D - 1) / (nch - 1) >= 4:
        d -= (d - np.arange(nch)) % 4
    assert len(np.unique(d)) == nch, (K, nch)
    return [int(FCR + 12_500 * v) for v in d]


def air_fc(freqs):
    return int(api.load().acb_air_choose_fc(min(freqs), max(freqs)))


def fast_plan_air(K, freqs, fc=None):
    """(kbin, tw (nch, K/4, 2) float32) of acb_fast_plan_air"""
    fc = air_fc(freqs) if fc is None else fc
    f = np.asarray(freqs, dtype=np.uint32)
    k = np.zeros(len(f), dtype=np.int32)
    tw = np.zeros((len(f), K // 4, 2), dtype=np.float32)
    assert api.load().acb_fast_plan_air(f.ctypes.data, len(f), K, fc, k.ctypes.data, tw.ctypes.data) == 1
    return k, tw


def exact_tables(K, taps, freqs, fc=None):
    """(exact table (nch, 2*taps) as acb_set_plan_air builds it, float64 weights (nch, taps), kbin, tw)"""
    L = api.load()
    fc = air_fc(freqs) if fc is None else fc
    rate = K * 12_500
    wf = np.zeros((len(freqs), 2 * taps), dtype=np.float32)
    for i, f in enumerate(freqs):
        if taps > K:
            L.acb_air_build_wf_lp(f, fc, rate, taps, wf[i].ctypes.data)
        else:
            L.acb_air_build_wf(f, fc, rate, wf[i].ctypes.data)
    k, tw = fast_plan_air(K, freqs, fc)
    h = api.build_lowpass(K, taps).astype(np.float64) if taps > K else np.full(K, 1.0 / K)
    i = np.arange(taps) - (taps - K)
    return wf, h[None, :] * np.exp(-2j * np.pi * np.outer(k, i) / K), k, tw


def fast_envelope(oracle, x, K, taps, k, tw):
    """the definition k_channelize_wb_real is held to: orc_channelize_rdft at taps = K, the pre-sum rows of
    orc_ovl_presum_real through it above"""
    if taps == K:
        return oracle.channelize_rdft(x, K, k, tw)
    return ovl_fast_real_refs.channelize_ovl_rdft(oracle, x, K, api.build_lowpass(K, taps), k, tw)


def exact_envelope(oracle, x, K, taps, wf):
    return ovl_refs.channelize_ovl_real(x, K, wf) if taps > K else oracle.channelize_real(x, K, wf)


@pytest.mark.parametrize("K", [56, 200, 800, 1600, 1808, 2048])
def test_table_reproduces_planner(lib, K):
    """Every admissible bin 0 < k < K: E[(k*n2) % K] is acb_fast_plan_air's twiddle T_k[n2], bit for bit, for every
    n2 < K/4."""
    E = wb_table(lib, K)
    rate = K * 12_500
    fc = FCR
    ks = np.arange(1, K)
    freqs = [fc + rate // 4 - 12_500 * int(v) for v in ks]          # air.c:278: k = (Fc - Fr + rate/4) / 12.5 kHz
    k, tw = fast_plan_air(K, freqs, fc)
    assert np.array_equal(k, ks)
    n2 = np.arange(K // 4, dtype=np.int64)
    r = (k.astype(np.int64)[:, None] * n2[None, :]) % K
    assert np.array_equal(E[r + K - 1].view(np.uint32), tw.view(np.uint32))


def test_other_variants_unchanged(lib):
    """The real variant is an addition: K % 8 != 0 is refused for it, and the u8 / CS16 variants still take K % 4 == 0."""
    E = np.zeros((2 * 204 - 1, 2), dtype=np.float32)
    assert lib.acb_wb_twiddles(WB_TW_REAL, 204, E.ctypes.data) == 0
    for v in (-1, 0, 1):
        assert lib.acb_wb_twiddles(v, 204, E.ctypes.data) == 1
    assert lib.acb_wb_twiddles(3, 200, E.ctypes.data) == 0


def rows_of(K, taps):
    return (taps + K - 1) // K + 6           # every row past the first window is a full window


def real_inputs(K, n, rng):
    frames = synth.render_real(frames_plan(K, (131.525, 131.5375, 131.55, 131.5625), n / (K * 12_500) + 0.05, seed=K,
                                           gap=0.005), 0, n)
    return {"frames": frames, "noise": (rng.standard_normal(n) * 100).astype(np.float32),
            "constant": np.full(n, 0.75, np.float32), "square": np.where(np.arange(n) % 2, -1.0, 1.0).astype(np.float32),
            "frames_2^-70": frames * np.float32(2.0 ** -70), "frames_2^70": frames * np.float32(2.0 ** 70)}


MEASURED = {}


def check(name, got, exact, ideal, S):
    ea = np.abs(got.astype(np.float64) - exact) / np.maximum(S, 1e-300)
    eb = np.abs(got.astype(np.float64) - ideal) / np.maximum(S, 1e-300)
    for key, v in (("fast_vs_exact", ea), ("fast_vs_f64", eb)):
        MEASURED[key] = max(MEASURED.get(key, 0.0), float(v.max()))
    assert np.isfinite(got).all(), name
    assert np.all(np.abs(got.astype(np.float64) - exact) <= TABLE_EPS * S), (name, float(ea.max()))
    assert np.all(np.abs(got.astype(np.float64) - ideal) <= IDEAL_EPS * S), (name, float(eb.max()))


SHAPES = [(800, 200), (1600, 256), (2048, 256)]
TAPS = {"K": lambda K: K, "K+4": lambda K: K + 4, "2K+3": lambda K: 2 * K + 3, "8K": lambda K: 8 * K,
        "16K": lambda K: 16 * K}


@pytest.mark.parametrize("K,nch", SHAPES)
@pytest.mark.parametrize("t", list(TAPS))
def test_real_within_bars(lib, oracle, K, nch, t):
    taps = TAPS[t](K)
    freqs = air_freqs(K, nch)
    wf, w64, k, tw = exact_tables(K, taps, freqs)
    assert len(set(int(v) % 4 for v in k)) == 4
    n = rows_of(K, taps) * K
    for name, x in real_inputs(K, n, np.random.default_rng(K + taps)).items():
        got = fast_envelope(oracle, x, K, taps, k, tw)
        exact = exact_envelope(oracle, x, K, taps, wf)
        ideal, S = f64_rows(x.astype(np.float64).astype(np.complex128), K, w64)
        check((name, K, nch, taps), got, exact, ideal, S)


def test_report_measured_maxima():
    """The worst ratios |error| / S over the test above (DESIGN.md §4 quotes them)."""
    if not MEASURED:
        pytest.skip("the tolerance test did not run in this session")
    print("\nreal-input wideband fast form, max |error|/S:", {k: f"{v:.3g}" for k, v in sorted(MEASURED.items())})
    assert MEASURED["fast_vs_exact"] <= TABLE_EPS and MEASURED["fast_vs_f64"] <= IDEAL_EPS


def wideband_real_fixture(K=1600, nch=160, nblk=8, weak=3.0, strong=30.0, noise=0.5, seed=5):
    """K = 1600 (20 MS/s real), nch adjacent 25 kHz channels around FCR.  Two channels carry frames at amplitude `weak`;
    the channel 25 kHz above each carries an AM voice carrier (+1 kHz off its centre) of amplitude `strong`, 10x the
    frames (20 dB).  Returns (x (nblk*1024*K,) float32, freqs, the two busy channels, the frames sent on them)."""
    freqs = [FCR + 25_000 * (i - nch // 2) for i in range(nch)]
    busy, loud = [30, 101], [31, 102]
    assert all(freqs[b] + 25_000 == freqs[n] for b, n in zip(busy, loud))
    fc, rate = air_fc(freqs), K * 12_500
    plan = synth.StreamPlan(K=K, freqs_hz=tuple(freqs[c] for c in busy), fc_hz=fc, seed=seed, noise_sigma=noise)
    rng = np.random.default_rng(seed)
    sent = []
    for ch in range(len(busy)):
        t = 0.05 + 0.07 * ch
        while t < nblk * 1024 / 12_500 - 0.2:
            fr = synth.frame_bytes(synth.random_text(rng, 30))
            plan.bursts.append(synth.Burst(chan=ch, t0=t, frame=fr, amp=weak, phase=float(rng.uniform(0, 2 * np.pi))))
            sent.append((ch, fr))
            t += len(fr) * 8 / 2400 + 0.03
    ns = nblk * 1024 * K
    x = synth.render_real(plan, 0, ns).astype(np.float64)
    tt = np.arange(ns, dtype=np.float64) / rate
    for i, c in enumerate(loud):
        audio = 0.5 * np.sin(2 * np.pi * 400 * tt + i) + 0.3 * np.sin(2 * np.pi * 1100 * tt + 1) + 0.2 * np.sin(2 * np.pi * 2300 * tt + 2)
        f_if = float(fc - (freqs[c] + 1000) + rate // 4)              # the neighbour's IF (air.c:278), 1 kHz off
        x += strong * (1 + 0.8 * audio) * np.cos(2 * np.pi * f_if * tt + i) / 256
    return x.astype(np.float32), freqs, busy, sent


def test_wideband_fixture_frames_identical(lib, oracle):
    """The K = 1600, 160-channel real fixture, two weak channels next to neighbours 20 dB stronger: the oracle decodes
    the same frames from the fast and the exact envelopes, with the boxcar and with an 8K filter; with the filter that
    is every frame sent, all with err = 0."""
    K = 1600
    x, freqs, busy, sent = wideband_real_fixture(K)
    fc = air_fc(freqs)
    sel = [freqs[c] for c in busy]
    for taps in (K, 8 * K):
        wf, _, k, tw = exact_tables(K, taps, sel, fc)
        exact = exact_envelope(oracle, x, K, taps, wf)
        fast = fast_envelope(oracle, x, K, taps, k, tw)
        decoded = 0
        for c in range(len(sel)):
            want = _frames(oracle, exact[c])
            assert _frames(oracle, fast[c]) == want, (taps, c)
            if taps > K:
                assert len(want) == sum(ch == c for ch, _ in sent) and all(m[2] == 0 for m in want), c
            decoded += len(want)
        if taps > K:
            assert decoded == len(sent) and decoded >= 4
