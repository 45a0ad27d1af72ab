"""CPU checks of the polyphase fast form of the overlapping-window channelizer (ACB_FLAG_FAST_FILTER, taps > K): its
restatement (tests/host/ovl_fast_oracle.c: orc_channelize_ovl_fast{,_cs16}) against the exact definition
(orc_channelize_ovl{,_cs16}) and against the definition evaluated in float64, per output row relative to
S = sum |x| * |w|, and the frames the oracle demodulator decodes from each envelope."""
import numpy as np
import pytest

import ovl_fast_refs
import ovl_refs
from acarsdec_b200 import api, synth
from test_ovl_oracle import decode_oracle, weak_strong_scenario

TABLE_EPS = 1e-5          # (a) fast vs exact form
IDEAL_EPS = 1e-6          # (b) fast vs the float64 definition
NROWS = 160


@pytest.fixture(scope="module")
def lib():
    from acarsdec_b200 import build
    build.build()
    return api.load()


def fast_plan(kind, variant, K, freqs_hz, fc):
    """(kbin, tw (nch, K/4, 2) float32) of acb_fast_plan / acb_fast_plan_cs16; the frequencies must be on the raster."""
    L = api.load()
    f = np.asarray(freqs_hz, dtype=np.uint32)
    k = np.zeros(len(f), dtype=np.int32)
    tw = np.zeros((len(f), K // 4, 2), dtype=np.float32)
    if kind == "u8":
        ok = L.acb_fast_plan(f.ctypes.data, len(f), K, fc, k.ctypes.data, tw.ctypes.data)
    else:
        ok = L.acb_fast_plan_cs16(variant, f.ctypes.data, len(f), K, fc, k.ctypes.data, tw.ctypes.data)
    assert ok == 1
    return k, tw


def setup(kind, variant, K, taps, fm=synth.DEFAULT_FREQS_MHZ):
    """(exact table, prototype h, kbin, tw, f64 weights (nch, taps)) of the planners for the channels fm."""
    fd, fr, fc = api.plan(K, fm)
    h = api.build_lowpass(K, taps)
    k, tw = fast_plan(kind, variant, K, fd, fc)
    if kind == "u8":
        wf, scale = api.build_wf_lp(K, taps, fm), 1 / 127.5
    else:
        wf, scale = api.build_wf_cs16_lp(variant, K, taps, fd, fc), (1 / 32768 if variant == 0 else 0.25)
    i = np.arange(taps) - (taps - K)
    w64 = h.astype(np.float64)[None, :] * np.exp(-2j * np.pi * np.outer(k, i) / K) * scale
    return wf, h, k, tw, w64


def f64_rows(xc: np.ndarray, K: int, w64: np.ndarray):
    """|D| and S = sum |x||w| of the definition in float64: xc the converted samples (complex128), (nch, nout) each."""
    taps = w64.shape[1]
    H = taps - K
    nout = len(xc) // K
    xp = np.concatenate([np.zeros(H, np.complex128), xc])
    win = np.lib.stride_tricks.sliding_window_view(xp, taps)[::K][:nout]
    return np.abs(win @ w64.T).T, (np.abs(win) @ np.abs(w64).T).T


def u8_inputs(K, rng):
    n = NROWS * K
    fm = synth.DEFAULT_FREQS_MHZ
    plan = synth.make_plan(K, fm, api.plan(K, fm)[2], seconds=1024 / 12500, seed=K, msgs_per_chan_per_sec=20.0)
    t = np.arange(n)
    sq = np.empty(2 * n, np.uint8)
    sq[0::2] = np.where((t // 7) % 2, 255, 0)
    sq[1::2] = np.where((t // 3) % 2, 0, 255)
    return {"frames": synth.render_blocks(plan, 0, 1).reshape(-1)[:2 * n],
            "uniform": rng.integers(0, 256, 2 * n, dtype=np.uint8),
            "zeros": np.zeros(2 * n, np.uint8), "ones255": np.full(2 * n, 255, np.uint8), "square": sq}


def cs16_inputs(K, rng):
    n = NROWS * K
    sat = rng.choice(np.array([-32768, 32767], np.int16), size=(n, 2))
    dc = np.empty((n, 2), np.int16)
    dc[:, 0], dc[:, 1] = 16384, -16384
    return {"saturation": sat, "dc": dc, "uniform": rng.integers(-32768, 32768, size=(n, 2), dtype=np.int16)}


MEASURED = {}


def check(name, got, exact, ideal, S):
    ea = np.abs(got.astype(np.float64) - exact) / np.maximum(S, 1e-300)
    eb = np.abs(got.astype(np.float64) - ideal) / np.maximum(S, 1e-300)
    ee = np.abs(exact.astype(np.float64) - ideal) / np.maximum(S, 1e-300)
    for key, v in (("fast_vs_exact", ea), ("fast_vs_f64", eb), ("exact_vs_f64", ee)):
        MEASURED[key] = max(MEASURED.get(key, 0.0), float(v.max()))
    assert np.all(np.abs(got.astype(np.float64) - exact) <= TABLE_EPS * S), (name, float(ea.max()))
    assert np.all(np.abs(got.astype(np.float64) - ideal) <= IDEAL_EPS * S), (name, float(eb.max()))


TAPS = ("K+8", "2K+3", "4K", "8K", "16K")


def taps_of(K, t):
    return {"K+8": K + 8, "2K+3": 2 * K + 3, "4K": 4 * K, "8K": 8 * K, "16K": 16 * K}[t]


@pytest.mark.parametrize("K", [160, 192])
@pytest.mark.parametrize("t", TAPS)
def test_fast_u8_within_bars(lib, K, t):
    taps = taps_of(K, t)
    wf, h, k, tw, w64 = setup("u8", None, K, taps)
    for name, iq in u8_inputs(K, np.random.default_rng(K + taps)).items():
        got = ovl_fast_refs.channelize_ovl_fast(iq, K, h, k, tw)
        exact = ovl_refs.channelize_ovl(iq, K, wf)
        xc = (iq[0::2].astype(np.float32) - np.float32(127.37)).astype(np.float64) + 1j * (iq[1::2].astype(np.float32) - np.float32(127.37))
        ideal, S = f64_rows(xc, K, w64)
        check((name, K, taps), got, exact, ideal, S)


@pytest.mark.parametrize("K", [160, 192])
@pytest.mark.parametrize("t", TAPS)
@pytest.mark.parametrize("variant", [0, 1])
def test_fast_cs16_within_bars(lib, K, t, variant):
    taps = taps_of(K, t)
    wf, h, k, tw, w64 = setup("cs16", variant, K, taps)
    for name, x in cs16_inputs(K, np.random.default_rng(K + taps + variant)).items():
        got = ovl_fast_refs.channelize_ovl_fast_cs16(x, K, h, k, tw)
        exact = ovl_refs.channelize_ovl_cs16(x, K, wf)
        ideal, S = f64_rows(x[:, 0].astype(np.float64) + 1j * x[:, 1], K, w64)
        check((name, K, taps, variant), got, exact, ideal, S)


def test_report_measured_maxima():
    """The worst ratios |error| / S over the two tests above (DESIGN.md §4 quotes them)."""
    if not MEASURED:
        pytest.skip("the tolerance tests did not run in this session")
    print("\npolyphase fast form, max |error|/S:", {k: f"{v:.3g}" for k, v in sorted(MEASURED.items())})
    assert MEASURED["fast_vs_exact"] <= TABLE_EPS and MEASURED["fast_vs_f64"] <= IDEAL_EPS


def _frames(oracle, dm_row):
    """(chn, len, err, txt, crc) of the frames the oracle decodes, in decoding (time) order"""
    return [m.as_tuple() for m in decode_oracle(oracle, dm_row)]


def test_weak_channel_frames_identical(lib, oracle):
    """The weak-channel fixture at 8K taps: the fast envelope decodes exactly the exact one's frames, all with err = 0."""
    K = 160
    iq, fm, sent = weak_strong_scenario(K)
    wf, h, k, tw, _ = setup("u8", None, K, 8 * K, fm)
    exact = _frames(oracle, ovl_refs.channelize_ovl(iq, K, wf[:1])[0])
    fast = _frames(oracle, ovl_fast_refs.channelize_ovl_fast(iq, K, h, k[:1], tw[:1])[0])
    assert fast == exact and len(fast) == len(sent) and all(m[2] == 0 for m in fast)


def test_eight_channel_frames_identical(lib, oracle):
    """An 8-channel synthetic stream at 8K taps: every channel decodes the same frames from both envelopes."""
    K, nblk = 160, 8
    fm = synth.DEFAULT_FREQS_MHZ
    plan = synth.make_plan(K, fm, api.plan(K, fm)[2], seconds=nblk * 1024 / 12500, seed=17, msgs_per_chan_per_sec=6.0,
                           text_len=(5, 30), amp=(4.0, 12.0))
    iq = synth.render_blocks(plan, 0, nblk).reshape(-1)
    wf, h, k, tw, _ = setup("u8", None, K, 8 * K, fm)
    exact = ovl_refs.channelize_ovl(iq, K, wf)
    fast = ovl_fast_refs.channelize_ovl_fast(iq, K, h, k, tw)
    total = 0
    for c in range(len(fm)):
        want = _frames(oracle, exact[c])
        assert _frames(oracle, fast[c]) == want, c
        total += len(want)
    assert total >= 10
