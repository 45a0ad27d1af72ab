"""CPU checks of the polyphase fast form of the overlapping-window channelizer for real input (ACB_FLAG_FAST_FILTER_REAL,
taps > K): its restatement (tests/host/ovl_fast_real_oracle.c: orc_ovl_presum_real, then the oracle's orc_channelize_rdft)
against the exact definition (orc_channelize_ovl_real) and against the definition evaluated in float64, per output row
relative to S = sum |x| * |w|, and the frames the oracle demodulator decodes from each envelope."""
import numpy as np
import pytest

import ovl_fast_real_refs
import ovl_refs
from acarsdec_b200 import api, synth
from test_ovl_fast_oracle import f64_rows
from test_ovl_oracle import decode_oracle

TABLE_EPS = 1e-5          # (a) fast vs exact form
IDEAL_EPS = 1e-6          # (b) fast vs the float64 definition
NROWS = 160
# on the 12.5 kHz raster around the Fc acb_air_choose_fc picks; four consecutive steps: every residue k mod 4
FREQS_MHZ = (131.525, 131.5375, 131.55, 131.5625, 131.725, 131.825, 131.45, 131.475)


@pytest.fixture(scope="module")
def lib():
    from acarsdec_b200 import build
    build.build()
    return api.load()


def fast_plan_air(K, freqs_hz, fc):
    """(kbin, tw (nch, K/4, 2) float32) of acb_fast_plan_air; the frequencies must be on the raster."""
    f = np.asarray(freqs_hz, dtype=np.uint32)
    k = np.zeros(len(f), dtype=np.int32)
    tw = np.zeros((len(f), K // 4, 2), dtype=np.float32)
    assert api.load().acb_fast_plan_air(f.ctypes.data, len(f), K, fc, k.ctypes.data, tw.ctypes.data) == 1
    return k, tw


def setup(K, taps, fm=FREQS_MHZ):
    """(exact table, prototype h, kbin, tw, f64 weights (nch, taps)) of acb_set_plan_air for the channels fm."""
    rate = K * 12500
    fd, fc, _ = api.air_plan(rate, fm)
    h = api.build_lowpass(K, taps)
    k, tw = fast_plan_air(K, fd, fc)
    wf = api.build_wf_air_lp(rate, taps, fm)
    i = np.arange(taps) - (taps - K)
    w64 = h.astype(np.float64)[None, :] * np.exp(-2j * np.pi * np.outer(k, i) / K)
    return wf, h, k, tw, w64


def fast_env(oracle, x, K, h, k, tw):
    return ovl_fast_real_refs.channelize_ovl_rdft(oracle, x, K, h, k, tw)


def frames_plan(K, fm, seconds, seed, amp=(10.0, 25.0), gap=0.05):
    rate = K * 12500
    fd, fc, _ = api.air_plan(rate, fm)
    plan = synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, seed=seed, noise_sigma=1.0)
    rng = np.random.default_rng(seed)
    for ch in range(len(fm)):
        t = 0.01 + 0.03 * ch
        while True:
            fr = synth.frame_bytes(synth.random_text(rng, int(rng.integers(8, 40))))
            dur = len(fr) * 8 / 2400
            if t + dur + 0.01 > seconds:
                break
            plan.bursts.append(synth.Burst(chan=ch, t0=t, frame=fr, amp=float(rng.uniform(*amp)), phase=float(rng.uniform(0, 6))))
            t += dur + gap
    return plan


def real_inputs(K, rng):
    n = NROWS * K
    frames = synth.render_real(frames_plan(K, FREQS_MHZ, n / (K * 12500), seed=K, gap=0.005), 0, n)
    return {"frames": frames, "noise": (rng.standard_normal(n) * 100).astype(np.float32),
            "constant": np.full(n, 0.75, np.float32), "square": np.where(np.arange(n) % 2, -1.0, 1.0).astype(np.float32),
            "frames_2^-70": frames * np.float32(2.0 ** -70), "frames_2^70": frames * np.float32(2.0 ** 70)}


MEASURED = {}


def check(name, got, exact, ideal, S):
    ea = np.abs(got.astype(np.float64) - exact) / np.maximum(S, 1e-300)
    eb = np.abs(got.astype(np.float64) - ideal) / np.maximum(S, 1e-300)
    ee = np.abs(exact.astype(np.float64) - ideal) / np.maximum(S, 1e-300)
    for key, v in (("fast_vs_exact", ea), ("fast_vs_f64", eb), ("exact_vs_f64", ee)):
        MEASURED[key] = max(MEASURED.get(key, 0.0), float(v.max()))
    assert np.isfinite(got).all(), name
    assert np.all(np.abs(got.astype(np.float64) - exact) <= TABLE_EPS * S), (name, float(ea.max()))
    assert np.all(np.abs(got.astype(np.float64) - ideal) <= IDEAL_EPS * S), (name, float(eb.max()))


TAPS = {"K+4": lambda K: K + 4, "2K+3": lambda K: 2 * K + 3, "4K": lambda K: 4 * K, "8K": lambda K: 8 * K,
        "16K": lambda K: 16 * K}
CASES = [(K, t) for K in (200, 800) for t in TAPS] + [(240, "K+4"), (240, "16K"), (400, "2K+3"), (400, "8K"),
                                                     (480, "4K"), (480, "16K")]


@pytest.mark.parametrize("K,t", CASES)
def test_fast_real_within_bars(lib, oracle, K, t):
    taps = TAPS[t](K)
    wf, h, k, tw, w64 = setup(K, taps)
    assert len(set(int(v) % 4 for v in k)) == 4
    for name, x in real_inputs(K, np.random.default_rng(K + taps)).items():
        got = fast_env(oracle, x, K, h, k, tw)
        exact = ovl_refs.channelize_ovl_real(x, K, wf)
        ideal, S = f64_rows(x.astype(np.float64).astype(np.complex128), K, w64)
        check((name, K, taps), got, exact, ideal, S)


def test_report_measured_maxima():
    """The worst ratios |error| / S over the test above (DESIGN.md §4 quotes them)."""
    if not MEASURED:
        pytest.skip("the tolerance test did not run in this session")
    print("\nreal-input polyphase fast form, max |error|/S:", {k: f"{v:.3g}" for k, v in sorted(MEASURED.items())})
    assert MEASURED["fast_vs_exact"] <= TABLE_EPS and MEASURED["fast_vs_f64"] <= IDEAL_EPS


def _frames(oracle, dm_row):
    """(chn, len, err, txt, crc) of the frames the oracle decodes, in decoding (time) order"""
    return [m.as_tuple() for m in decode_oracle(oracle, dm_row)]


def weak_strong_real(K: int = 200, seconds: float = 1.0, weak: float = 3.0, strong: float = 60.0, noise: float = 0.5,
                     seed: int = 3):
    """float32 real input (air.c front-end) of a weak channel (131.525 MHz) carrying frames and a strong AM voice carrier
    on its 25 kHz neighbour (131.550 MHz) with a +1 kHz carrier offset: returns (x, planned channel freqs in MHz, the
    frames sent)."""
    fm = (131.525, 131.550)
    rate = K * 12500
    fd, fc, _ = api.air_plan(rate, fm)
    plan = synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, seed=seed, noise_sigma=noise)
    rng = np.random.default_rng(seed)
    t, sent = 0.05, []
    while t < seconds - 0.2:
        fr = synth.frame_bytes(synth.random_text(rng, 30))
        plan.bursts.append(synth.Burst(chan=0, t0=t, frame=fr, amp=weak, phase=float(rng.uniform(0, 2 * np.pi))))
        sent.append(fr)
        t += len(fr) * 8 / 2400 + 0.03
    ns = int(seconds * rate) // K * K
    tt = np.arange(ns, dtype=np.float64) / rate
    audio = 0.5 * np.sin(2 * np.pi * 400 * tt) + 0.3 * np.sin(2 * np.pi * 1100 * tt + 1) + 0.2 * np.sin(2 * np.pi * 2300 * tt + 2)
    f_if = float(fc - (fd[1] + 1000) + rate // 4)                  # the neighbour's IF (air.c:278), 1 kHz off
    x = synth.render_real(plan, 0, ns).astype(np.float64)
    x += strong * (1 + 0.8 * audio) * np.cos(2 * np.pi * f_if * tt) / 256
    return x.astype(np.float32), fm, sent


def test_weak_channel_frames_identical(lib, oracle):
    """The real-input weak/strong fixture: the boxcar (taps = K) loses every weak frame; at 8K taps the exact and the fast
    envelope decode every frame, all with err = 0, and the same frames."""
    K = 200
    x, fm, sent = weak_strong_real(K)
    assert len(sent) >= 3
    box = decode_oracle(oracle, oracle.channelize_real(x, K, api.build_wf_air(K * 12500, fm)[:1])[0])
    assert len([m for m in box if m.err == 0]) == 0
    wf, h, k, tw, _ = setup(K, 8 * K, fm)
    exact = _frames(oracle, ovl_refs.channelize_ovl_real(x, K, wf[:1])[0])
    fast = _frames(oracle, fast_env(oracle, x, K, h, k[:1], tw[:1])[0])
    assert fast == exact and len(fast) == len(sent) and all(m[2] == 0 for m in fast)


def test_eight_channel_frames_identical(lib, oracle):
    """An 8-channel air stream at 8K taps: every channel decodes the same frames from both envelopes."""
    K, secs = 200, 0.6
    fm = synth.DEFAULT_FREQS_MHZ
    x = synth.render_real(frames_plan(K, fm, secs, seed=17, amp=(4.0, 12.0), gap=0.02), 0, int(secs * K * 12500))
    wf, h, k, tw, _ = setup(K, 8 * K, fm)
    exact = ovl_refs.channelize_ovl_real(x, K, wf)
    fast = fast_env(oracle, x, K, h, k, tw)
    total = 0
    for c in range(len(fm)):
        want = _frames(oracle, exact[c])
        assert _frames(oracle, fast[c]) == want, c
        total += len(want)
    assert total >= 10
