"""The frequency-error definition (tests/freq_stats_refs.py) against physical truth: synthetic receivers whose carriers
sit off the frequencies the context plans with, for every input kind.

The estimate reads about 1% short of the true offset.  The AM sidebands of the MSK subcarrier (1200 and 2400 Hz) sit on
either side of the carrier, and the half-row boxcar passes the one nearer the channel centre more strongly, which pulls
the rotation toward zero.  At the synthesizer's default noise (1.5 LSB) this file's run gave errors of 0.2 to 2.8 Hz at
0 Hz, 16 Hz at +1.7 kHz and 29 Hz at -3.2 kHz, and 23.28 ppm for 23.5 ppm.  So offsets are held to 3 Hz + 1.2% of the
offset and ppm to 0.3."""
import numpy as np
import pytest

import freq_stats_refs as fr
from acarsdec_b200 import api, synth

K = {"u8": 160, "real": 200, "soapy": 160, "sdrplay": 160}
BASE = {"u8": "u8", "real": "real", "soapy": "cs16", "sdrplay": "cs16"}
FM = (131.125, 131.450, 131.725)
OFF_TOL_HZ, OFF_TOL_REL, PPM_TOL = 3.0, 0.012, 0.3


def _planned(kind):
    """the nominal plan a context would be given: (freqs_hz, fc)"""
    k = K[kind]
    if kind == "real":
        fd, fc, _ = api.air_plan(k * 12500, FM)
        return [int(f) for f in fd], int(fc)
    fd, _, fc = api.plan(k, FM)
    return [int(f) for f in fd], int(fc)


def _render(kind, true_hz, fc, seconds=0.5, seed=3, drop=()):
    """the receiver's samples, one 0.4 s frame per channel with its carrier at true_hz; channels in `drop` carry none"""
    k = K[kind]
    rng = np.random.default_rng(seed)
    bursts = [synth.Burst(chan=c, t0=0.01 + 0.03 * c, frame=synth.frame_bytes(synth.random_text(rng, 100)), amp=float(rng.uniform(12, 30)),
                          phase=float(rng.uniform(0, 2 * np.pi))) for c in range(len(FM)) if c not in drop]
    p = synth.StreamPlan(K=k, freqs_hz=tuple(true_hz), fc_hz=fc, bursts=bursts, seed=seed)
    n = int(seconds * k * 12500) // (1024 * k) * (1024 * k)
    if kind == "u8":
        return synth.render_blocks(p, 0, n // (1024 * k)).reshape(-1)
    if kind == "real":
        return synth.render_real(p, 0, n)
    return synth.render_cs16(p, 0, n)


def _measure(kind, x, freqs_hz, fc):
    freq, step = fr.plan_record(BASE[kind], K[kind], freqs_hz, fc)
    ref = fr.ChainFreq(BASE[kind], K[kind], step)
    u = 2 if kind == "u8" else 1                             # u8: bytes, two per sample
    n = len(x) // u // 3
    for part in (x[:n * u], x[n * u:(2 * n + 7) * u], x[(2 * n + 7) * u:]):     # cut anywhere: the carry completes rows
        ref.feed(part)
    s = np.array([ref.sums(c) for c in range(len(freqs_hz))])
    return freq, s


@pytest.mark.parametrize("kind", list(K))
def test_per_channel_offsets(kind):
    freqs, fc = _planned(kind)
    shift = np.array([1700.0, -3200.0, 0.0])
    x = _render(kind, np.array(freqs) + shift, fc)
    freq, s = _measure(kind, x, freqs, fc)
    got = fr.offsets(s[:, 0], s[:, 1], K[kind])
    truth = np.array(freqs) + shift - freq               # freq_hz is the mixer's centre: within 4 Hz of the plan
    assert np.all(np.abs(got - truth) < OFF_TOL_HZ + OFF_TOL_REL * np.abs(truth)), (got, truth)
    assert np.all(np.sign(got[:2]) == np.sign(truth[:2]))
    assert np.all(np.hypot(s[:, 0], s[:, 1]) / s[:, 2] > 0.5)


@pytest.mark.parametrize("kind", list(K))
def test_stream_ppm(kind):
    freqs, fc = _planned(kind)
    ppm = 23.5
    x = _render(kind, np.array(freqs) * (1 + ppm * 1e-6), fc, seed=5)
    freq, s = _measure(kind, x, freqs, fc)
    truth = 1e6 * np.average((np.array(freqs) * (1 + ppm * 1e-6) - freq) / freq, weights=np.hypot(s[:, 0], s[:, 1]))
    got = fr.ppm(s[:, 0], s[:, 1], freq, K[kind])
    assert abs(got - ppm) < PPM_TOL, (got, truth)
    # the library's helper applies the same formulas
    t = np.zeros(len(freqs), api.CHAN_FREQ_DTYPE)
    t["pairs"], t["s_re"], t["s_im"], t["mag_sum"], t["freq_hz"] = 1, s[:, 0], s[:, 1], s[:, 2], freq
    e = api.freq_error(t, K[kind])
    assert np.allclose(e["offset_hz"][0], fr.offsets(s[:, 0], s[:, 1], K[kind]), rtol=1e-12, atol=1e-9)
    assert np.allclose(e["coherence"][0], np.hypot(s[:, 0], s[:, 1]) / s[:, 2], rtol=1e-12)
    assert abs(e["ppm"][0] - got) < 1e-9


@pytest.mark.parametrize("kind", list(K))
def test_noise_only_chains_are_incoherent(kind):
    freqs, fc = _planned(kind)
    x = _render(kind, freqs, fc, seed=9, drop=(1,))
    _, s = _measure(kind, x, freqs, fc)
    coh = np.hypot(s[:, 0], s[:, 1]) / s[:, 2]
    assert coh[1] < 0.1 and coh[0] > 0.5 and coh[2] > 0.5, coh


@pytest.mark.parametrize("kind", ["u8", "real"])
def test_offsets_past_half_the_lag_rate_alias(kind):
    """unambiguous within +-rate / (2h) = 12.5 kHz: a carrier 14 kHz high reads 14 - 25 = -11 kHz"""
    freqs, fc = _planned(kind)
    x = _render(kind, np.array(freqs) + np.array([14000.0, 0.0, 0.0]), fc, seed=4, drop=(1, 2))
    freq, s = _measure(kind, x, freqs, fc)
    got = fr.offsets(s[0, 0], s[0, 1], K[kind])
    truth = freqs[0] + 14000.0 - freq[0] - 25000.0
    assert abs(got - truth) < OFF_TOL_HZ + 0.05 * abs(truth), got


def test_dtype_matches_the_c_struct():
    assert api.CHAN_FREQ_DTYPE.itemsize == 56
    assert api.FLAG_FREQ_STATS == 1024
