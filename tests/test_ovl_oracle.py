"""CPU checks of the overlapping-window channelizer (taps > K): its restatement (tests/host/ovl_oracle.c, the
definition) against the reference's arithmetic at taps == K, its locality, the prototype filter and the planners'
tables against float64 restatements, and the point of the feature — a weak channel next to a strong neighbour —
on the CPU oracle."""
import numpy as np
import pytest

import ovl_refs
import refs
from acarsdec_b200 import api, synth
from common import bits_equal

FM = synth.DEFAULT_FREQS_MHZ[:5]


@pytest.fixture(scope="module")
def lib():
    from acarsdec_b200 import build
    build.build()
    return api.load()


def _cs16_folded(oracle, variant, K, fm):
    fd, _, fc = oracle.plan(K, fm)
    return fd, fc, api.build_wf_cs16(variant, K, fd, fc)


def test_taps_eq_k_is_the_reference_arithmetic(lib, oracle):
    """At taps == K the restatement is orc_channelize / orc_channelize_real / the folded CS16 form, bit for bit."""
    rng = np.random.default_rng(1)
    for K in (160, 200):
        wf = oracle.wf(K, FM)
        iq = rng.integers(0, 256, size=2 * 40 * K, dtype=np.uint8)
        assert bits_equal(ovl_refs.channelize_ovl(iq, K, wf), oracle.channelize(iq, K, wf))
        x = rng.standard_normal(40 * K).astype(np.float32) * 300
        wfa = oracle.air_wf(K * 12500, FM)
        assert bits_equal(ovl_refs.channelize_ovl_real(x, K, wfa), oracle.channelize_real(x, K, wfa))
        for variant in (0, 1):
            _, _, wfc = _cs16_folded(oracle, variant, K, FM)
            c16 = rng.integers(-32768, 32768, size=(40 * K, 2), dtype=np.int16)
            assert bits_equal(ovl_refs.channelize_ovl_cs16(c16, K, wfc), oracle.channelize_cs16(2, c16, K, wfc))


@pytest.mark.parametrize("K,taps", [(160, 168), (160, 317), (192, 4 * 192 - 3), (44, 130)])
def test_pieces_with_history_equal_whole_stream(K, taps):
    """A stream cut into pieces, each preceded by enough whole rows of history, gives the whole stream's rows."""
    rng = np.random.default_rng(taps)
    nrow = 60
    lead = -(-(taps - K) // K)                            # rows whose window reaches before their piece
    w = rng.standard_normal((3, 2 * taps)).astype(np.float32) * 1e-3
    iq = rng.integers(0, 256, size=2 * nrow * K, dtype=np.uint8)
    x = rng.standard_normal(nrow * K).astype(np.float32)
    c16 = rng.integers(-32768, 32768, size=(nrow * K, 2), dtype=np.int16)
    whole = (ovl_refs.channelize_ovl(iq, K, w), ovl_refs.channelize_ovl_real(x, K, w), ovl_refs.channelize_ovl_cs16(c16, K, w))
    for r0, r1 in ((0, 7), (7, 31), (31, 60)):
        s0 = max(0, r0 - lead)
        got = (ovl_refs.channelize_ovl(iq[2 * s0 * K:2 * r1 * K], K, w), ovl_refs.channelize_ovl_real(x[s0 * K:r1 * K], K, w),
               ovl_refs.channelize_ovl_cs16(c16[s0 * K:r1 * K], K, w))
        for g, wh in zip(got, whole):
            assert bits_equal(g[:, r0 - s0:], wh[:, r0:r1]), (r0, r1)
    # the first rows really omit the terms before the stream start: zero-padding the u8 bytes would not
    padded = np.concatenate([np.zeros(2 * lead * K, np.uint8), iq])
    assert not bits_equal(ovl_refs.channelize_ovl(padded, K, w)[:, lead:lead + 1], whole[0][:, :1])


@pytest.mark.parametrize("K", [160, 192, 200, 1600])
def test_lowpass_matches_float64_restatement(lib, K):
    for taps in (K + 1, 2 * K, 4 * K - 3, 8 * K, 16 * K):
        h = api.build_lowpass(K, taps)
        ref = ovl_refs.lowpass_f64(K, taps)
        ulp = np.spacing(np.abs(ref).astype(np.float32))
        assert np.all(np.abs(h.astype(np.float64) - ref) <= 4 * ulp + 1e-12 * np.abs(ref).max()), taps
        assert abs(float(np.sum(h.astype(np.float64))) - 1.0) < 1e-5
    with pytest.raises(api.AcbError):
        api.build_lowpass(K, 16 * K + 1)


def _response_db(w_complex: np.ndarray, rate: int):
    """Response of a table to a tone at f (relative to the tuner centre) on a dense grid: sum_i w[i] e^{+j2pi f i/rate}."""
    n = 1 << int(np.ceil(np.log2(len(w_complex) * 32)))
    r = np.fft.ifft(w_complex.astype(np.complex128), n) * n
    f = np.fft.fftfreq(n, 1.0 / rate)
    return f, 20 * np.log10(np.maximum(np.abs(r), 1e-300))


@pytest.mark.parametrize("K", [160, 192, 200, 1600])
def test_planner_tables_isolate_the_channel(lib, K):
    """From the float tables themselves: <= -60 dB at >= 21.4 kHz from the channel for taps >= 2K; <= -40 dB on
    8.9-21.4 kHz (what folds onto the audio band) and <= 0.2 dB passband loss to 3.6 kHz for taps >= 8K."""
    rate = K * 12500
    fm = (131.525, 131.550, 131.725) if K < 1600 else (130.025, 131.550, 135.000)
    fd, fr, fc = api.plan(K, fm)
    for taps in (2 * K, 8 * K, 16 * K):
        tabs = {"u8": api.build_wf_lp(K, taps, fm),
                "cs16": api.build_wf_cs16_lp(0, K, taps, fd, fc)}
        for kind, wf in tabs.items():
            for ch in range(len(fm)):
                w = wf[ch, 0::2].astype(np.float64) + 1j * wf[ch, 1::2]
                f, db = _response_db(w, rate)
                off = float(np.float32(fr[ch] if kind == "u8" else fd[ch]) - np.float32(fc))
                d = np.abs(((f - off) + rate / 2) % rate - rate / 2)
                db0 = db[np.argmin(d)]
                scale = 127.5 if kind == "u8" else 32768.0
                assert abs(db0 + 20 * np.log10(scale)) < 0.01, (kind, taps)           # reference level at the centre
                rel = db - db0
                assert rel[d >= 21400].max() <= -60, (kind, taps, ch, rel[d >= 21400].max())
                if taps >= 8 * K:
                    assert rel[(d >= 8900) & (d < 21400)].max() <= -40, (kind, taps, ch)
                    assert rel[d <= 3600].min() >= -0.2, (kind, taps, ch)
    # real input: the mixer is air.c's IF at rate/4
    wfa = api.build_wf_air_lp(rate, 8 * K, fm)
    fda, fca, _ = api.air_plan(rate, fm)
    w = wfa[0, 0::2].astype(np.float64) + 1j * wfa[0, 1::2]
    f, db = _response_db(w, rate)
    f_if = fca - fda[0] + rate // 4
    d = np.abs(((f - f_if) + rate / 2) % rate - rate / 2)
    assert abs(db[np.argmin(d)]) < 0.01 and (db[d >= 21400] - db[np.argmin(d)]).max() <= -60


def weak_strong_scenario(K: int = 160, nblk: int = 12, weak: float = 3.0, strong: float = 60.0, noise: float = 0.5, seed: int = 3):
    """u8 IQ of a weak channel (131.525 MHz) carrying frames and a strong AM voice carrier on its 25 kHz neighbour
    (131.550 MHz) with a +1 kHz carrier offset: returns (iq, planned channel freqs in MHz, the frames sent).  The
    neighbour peaks at strong * 1.8 = 108 LSB: no clipping."""
    fm = (131.525, 131.550)
    fd, _, fc = api.plan(K, fm)
    plan = synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, seed=seed, noise_sigma=noise)
    rng = np.random.default_rng(seed)
    t, sent = 0.05, []
    while t < nblk * 1024 / 12500 - 0.2:
        fr = synth.frame_bytes(synth.random_text(rng, 30))
        plan.bursts.append(synth.Burst(chan=0, t0=t, frame=fr, amp=weak, phase=float(rng.uniform(0, 2 * np.pi))))
        sent.append(fr)
        t += len(fr) * 8 / 2400 + 0.03
    fs, ns = K * 12500, nblk * 1024 * K
    tt = np.arange(ns, dtype=np.float64) / fs
    audio = 0.5 * np.sin(2 * np.pi * 400 * tt) + 0.3 * np.sin(2 * np.pi * 1100 * tt + 1) + 0.2 * np.sin(2 * np.pi * 2300 * tt + 2)
    x = strong * (1 + 0.8 * audio) * np.exp(2j * np.pi * (fd[1] + 1000 - fc) * tt)
    for b in plan.bursts:
        lo, hi, v = synth.burst_samples(plan, b, 0, ns)
        x[lo:hi] += v
    iq = np.empty(2 * ns)
    iq[0::2], iq[1::2] = x.real, x.imag
    iq += np.random.default_rng([seed, 9]).standard_normal(2 * ns) * noise
    return np.clip(np.floor(iq + 128.0), 0, 255).astype(np.uint8), fm, sent


def decode_oracle(oracle, dm_row):
    sink = refs.Sink()
    ch = oracle.new_chan(0)
    oracle.demod(ch, dm_row, sink)
    fixed = [oracle.fec(m) for m in sink.msgs()]
    return [f for f in fixed if f is not None]


def test_weak_channel_next_to_strong_neighbour(lib, oracle):
    """The reference's boxcar lets the neighbour through and the weak channel's frames are lost; the 8K-tap low-pass
    decodes every one of them without a parity error."""
    K = 160
    iq, fm, sent = weak_strong_scenario(K)
    box = decode_oracle(oracle, ovl_refs.channelize_ovl(iq, K, api.build_wf(K, fm)[:1])[0])
    ovl = decode_oracle(oracle, ovl_refs.channelize_ovl(iq, K, api.build_wf_lp(K, 8 * K, fm)[:1])[0])
    assert len(sent) >= 3
    assert len([m for m in box if m.err == 0]) == 0
    assert len(ovl) == len(sent) and all(m.err == 0 for m in ovl)
