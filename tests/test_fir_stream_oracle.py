"""CPU checks of the short channel filter's definition for the streaming front-ends (tests/host/fir_stream_oracle.c,
taps <= K on float32 real and CS16 input): at taps == K it is the reference's arithmetic bit for bit, and at every
taps it is the exact sum over the FIRST `taps` samples of each row to within a bound derived from its operation count,
across the whole float32 exponent range and at full-scale int16."""
import numpy as np
import pytest

import fir_stream_refs as fsr
import ovl_refs
from acarsdec_b200 import api, synth
from common import bits_equal

FM = synth.DEFAULT_FREQS_MHZ[:5]
U = 2.0 ** -24                      # unit roundoff of float32, round to nearest


@pytest.fixture(scope="module")
def lib():
    from acarsdec_b200 import build
    build.build()
    return api.load()


def bound(taps: int, S: np.ndarray) -> np.ndarray:
    """Worst-case |fl(|D|) - |D|| for the definition's operations.  Per component (re or im) a term is one rounded
    product (real input) or two rounded products and a rounded difference (CS16): its error is at most 2u times
    |a c| + |b d| <= |x| |w|.  Recursive summation of `taps` terms adds at most (taps - 1) u times the partial sums'
    magnitudes, each <= S = sum_i |x_i| |w_i|.  So each component is off by at most (taps + 1) u S (first order), the
    complex sum by sqrt(2) times that, and hypotf adds one rounding of |D| <= S.  A 1 % margin covers the second-order
    terms (n u << 1 here)."""
    return 1.01 * (np.sqrt(2.0) * (taps + 1) + 1) * U * S


def test_taps_eq_k_is_the_reference_arithmetic(lib, oracle):
    """At taps == K: orc_channelize_real on air.c's tables, orc_channelize_ovl_cs16 (the folded form) on both CS16
    variants' tables and on random ones, bit for bit."""
    rng = np.random.default_rng(3)
    for K in (160, 200, 42):
        x = (rng.standard_normal(37 * K) * 300).astype(np.float32)
        wfa = oracle.air_wf(K * 12500, FM) if K % 4 == 0 else (rng.standard_normal((5, 2 * K)) / K).astype(np.float32)
        assert bits_equal(fsr.channelize_fir_real(x, K, wfa), oracle.channelize_real(x, K, wfa)), K
        c16 = rng.integers(-32768, 32768, size=(37 * K, 2), dtype=np.int16)
        tables = [(rng.standard_normal((3, 2 * K)) / K).astype(np.float32)]
        if K % 4 == 0:
            fd, _, fc = oracle.plan(K, FM)
            tables += [api.build_wf_cs16(v, K, fd, fc) for v in (0, 1)]
        for wfc in tables:
            assert bits_equal(fsr.channelize_fir_cs16(c16, K, wfc), ovl_refs.channelize_ovl_cs16(c16, K, wfc)), K


def test_first_taps_of_the_row(oracle):
    """taps < K weights the first `taps` samples of a row: the rest of the row changes nothing, and the result equals
    the taps == K sum with the table padded by zeros behind (bit for bit: +0 terms leave a float sum unchanged)."""
    rng = np.random.default_rng(4)
    K, taps = 44, 13
    w = (rng.standard_normal((4, 2 * taps)) / taps).astype(np.float32)
    wk = np.zeros((4, 2 * K), np.float32)
    wk[:, :2 * taps] = w
    x = (rng.standard_normal(25 * K) * 10).astype(np.float32)
    c16 = rng.integers(-32768, 32768, size=(25 * K, 2), dtype=np.int16)
    assert bits_equal(fsr.channelize_fir_real(x, K, w), oracle.channelize_real(x, K, wk))
    assert bits_equal(fsr.channelize_fir_cs16(c16, K, w), ovl_refs.channelize_ovl_cs16(c16, K, wk))
    x2, c2 = x.reshape(25, K).copy(), c16.reshape(25, K, 2).copy()
    x2[:, taps:] = rng.standard_normal((25, K - taps)).astype(np.float32) * 1e6
    c2[:, taps:] = rng.integers(-32768, 32768, size=(25, K - taps, 2), dtype=np.int16)
    assert bits_equal(fsr.channelize_fir_real(x2, K, w), fsr.channelize_fir_real(x, K, w))
    assert bits_equal(fsr.channelize_fir_cs16(c2, K, w), fsr.channelize_fir_cs16(c16, K, w))
    # not the last `taps` samples (what ovl_oracle.c's H = taps - K < 0 would give)
    assert not bits_equal(fsr.channelize_fir_real(x, K, w), ovl_refs.channelize_ovl_real(x, K, w))


@pytest.mark.parametrize("K", [64, 42])
@pytest.mark.parametrize("taps", [1, 3, 4, 21, "K-1"])
def test_within_float64_bound(K, taps):
    taps = K - 1 if taps == "K-1" else taps
    rng = np.random.default_rng(K * 100 + taps)
    nch, nrow = 6, 300
    w = (rng.standard_normal((nch, 2 * taps)) / np.sqrt(taps)).astype(np.float32)
    cases = [(rng.standard_normal(nrow * K) * 100).astype(np.float32),
             rng.integers(-32768, 32768, size=(nrow * K, 2), dtype=np.int16)]
    for x in cases:
        got = fsr.channelize_fir_real(x, K, w) if x.dtype == np.float32 else fsr.channelize_fir_cs16(x, K, w)
        ref, S = fsr.fir_f64(x, K, w)
        err = np.abs(got.astype(np.float64) - ref)
        assert np.all(err <= bound(taps, S)), (x.dtype, float((err / np.maximum(S, 1e-300)).max()))
        # the bound is not vacuous: the definition is not exact either
        assert err.max() > 0


@pytest.mark.parametrize("e", [-70, -40, 0, 40, 70])
def test_real_input_across_the_exponent_range(e):
    """float32 real input scaled by 2^e (products stay normal: |w| ~ 2^-3, |x| up to ~2^(e+3)): the bound holds with
    the same relative size at every scale, and a power-of-two scale of the input scales the output exactly."""
    K, taps, nch = 64, 21, 4
    rng = np.random.default_rng(70 + e)
    w = (rng.standard_normal((nch, 2 * taps)) / np.sqrt(taps)).astype(np.float32)
    x0 = rng.standard_normal(200 * K).astype(np.float32)
    x = (x0 * np.float32(2.0 ** e)).astype(np.float32)
    got = fsr.channelize_fir_real(x, K, w)
    ref, S = fsr.fir_f64(x, K, w)
    assert np.all(np.isfinite(got)) and np.all(S > 0)
    assert np.all(np.abs(got.astype(np.float64) - ref) <= bound(taps, S))
    assert bits_equal(got, (fsr.channelize_fir_real(x0, K, w) * np.float32(2.0 ** e)).astype(np.float32))


def test_full_scale_int16():
    """CS16 at full scale: -32768 and 32767 in both components, alternating signs (the largest |D| a table allows),
    and a row of -32768 only (the one value whose negation is not an int16)."""
    K, taps, nch = 48, 37, 3
    rng = np.random.default_rng(16)
    w = (rng.standard_normal((nch, 2 * taps)) / np.sqrt(taps)).astype(np.float32)
    nrow = 64
    iq = rng.choice(np.array([-32768, 32767], np.int16), size=(nrow * K, 2))
    iq[:K] = -32768
    iq[K:2 * K, 0], iq[K:2 * K, 1] = 32767, -32768
    got = fsr.channelize_fir_cs16(iq, K, w)
    ref, S = fsr.fir_f64(iq, K, w)
    assert np.all(np.abs(got.astype(np.float64) - ref) <= bound(taps, S))
    # row 0: every sample is -32768 - 32768j, so |D| = 32768 sqrt(2) |sum w|, independently of fir_f64
    d0 = 32768.0 * np.sqrt(2.0) * np.abs((w[:, 0:2 * taps:2].astype(np.float64) + 1j * w[:, 1:2 * taps:2]).sum(axis=1))
    assert np.all(np.abs(got[:, 0] - d0) <= bound(taps, S[:, 0]))
