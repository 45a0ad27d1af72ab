"""The scalable level definition (tests/level_stats_wide_refs.py) against the term-by-term one (tests/level_stats_refs.py):
on that module's hand-worked cases and on random ragged schedules with resets, counts, windows and peaks equal and sums
within 1e-13."""
import math

import numpy as np
import pytest

import level_stats_refs as lr
import level_stats_wide_refs as wr


def _same_input(w: wr.InputLevels, n: lr.InputLevels):
    ws, wc, wp, wk = w.row()
    ns, nc, np_, nk = n.row()
    assert (ws, wc, wk) == (ns, nc, nk)
    assert math.isclose(wp, np_, rel_tol=1e-13, abs_tol=0.0 if np_ else 1e-300), (wp, np_)
    assert (w.carry is None or not len(w.carry)) == (n.carry is None or not len(n.carry))
    if n.carry is not None and len(n.carry):
        assert np.array_equal(w.carry, n.carry)


def _same_chans(w: wr.ChanLevels, ns: list[lr.ChanLevels]):
    for c, n in enumerate(ns):
        rows, p, peak, windows, floor = n.row()
        assert (w.rows, w.windows, float(w.peak[c])) == (rows, windows, peak), c
        assert w.open_rows == n.open_rows
        assert math.isclose(w.power_sum()[c], p, rel_tol=1e-13, abs_tol=0.0 if p else 1e-300), (c, w.power_sum()[c], p)
        assert math.isclose(w.floor[c], floor, rel_tol=1e-13, abs_tol=0.0 if floor else 1e-300), (c, w.floor[c], floor)


def test_window_split_over_three_submits():
    w = wr.ChanLevels(1)
    for x in (np.full(500, 1.0), np.full(400, 2.0)):
        w.feed(x[:, None])
    assert (w.rows, w.windows) == (900, 0) and w.floor[0] == 0.0
    w.feed(np.full((300, 1), 3.0))
    assert (w.rows, w.windows, w.open_rows) == (1200, 1, 176)
    assert w.floor[0] == (500 * 1 + 400 * 4 + 124 * 9) / 1024
    assert w.power_sum()[0] == 500 * 1 + 400 * 4 + 300 * 9 and w.peak[0] == 3.0
    w.clear()                                          # reset != 0 keeps the open window
    w.feed(np.full((848, 1), 0.5))
    assert (w.rows, w.windows) == (848, 1)
    assert w.floor[0] == (176 * 9 + 848 * 0.25) / 1024


def test_streaming_carry_completes_a_row_in_the_next_submit():
    inp = wr.InputLevels("real", 4)
    x = np.array([0.5, -0.25, 0.125, 0.0, 1.0, -1.0, 0.75, 0.5], np.float32)
    assert inp.feed(x[:6]) == 1
    assert (inp.samples, inp.clipped) == (4, 0)
    assert inp.power_sum() == 0.25 + 0.0625 + 0.015625
    assert inp.feed(x[6:]) == 1
    assert (inp.samples, inp.clipped) == (8, 2)
    assert inp.power_sum() == 0.25 + 0.0625 + 0.015625 + 1 + 1 + 0.5625 + 0.25
    assert inp.peak == 1.0


def test_full_scale_codes():
    inp = wr.InputLevels("u8", 1)
    inp.feed(np.array([0, 255, 127, 128], np.uint8))
    assert (inp.samples, inp.clipped) == (2, 1)
    assert inp.peak == np.float32(255) - np.float32(127.37)
    v = [np.float64(np.float32(b) - np.float32(127.37)) for b in (0, 255, 127, 128)]
    assert inp.power_sum() == math.fsum(t * t for t in v)
    cs = wr.InputLevels("cs16", 2)
    cs.feed(np.array([[-32768, -32768], [32767, 0], [5, -5], [0, 0]], np.int16))
    assert (cs.samples, cs.clipped, cs.peak) == (4, 2, 32768.0)
    assert cs.power_sum() == 2 * 32768 ** 2 + 32767 ** 2 + 50


@pytest.mark.parametrize("kind,K", [("u8", 1), ("u8", 3), ("cs16", 7), ("cs16", 4), ("real", 5), ("real", 8)])
def test_random_ragged_schedules(kind, K):
    """both definitions fed the same submits, some empty or shorter than a row, with clears and stream resets between"""
    rng = np.random.default_rng([K, len(kind)])
    nch = 5
    w_in, n_in = wr.InputLevels(kind, K), lr.InputLevels(kind, K)
    w_ch, n_ch = wr.ChanLevels(nch), [lr.ChanLevels() for _ in range(nch)]
    for i in range(60):
        n = int(rng.choice([0, rng.integers(1, K + 1), rng.integers(K, 40 * K), rng.integers(300 * K, 2600 * K)]))
        if kind == "u8":
            x = rng.choice(np.array([0, 1, 127, 128, 254, 255], np.uint8), size=2 * n) if i % 7 == 3 else \
                rng.integers(0, 256, size=2 * n, dtype=np.uint8)
        elif kind == "cs16":
            x = rng.integers(-32768, 32768, size=(n, 2), dtype=np.int16)
            x[rng.random(n) < 0.01] = -32768
        else:
            x = (rng.standard_normal(n) * rng.choice([1e-3, 0.3, 2.0])).astype(np.float32)
        rows = w_in.feed(x)
        assert n_in.feed(x) == rows
        dm = (rng.random((int(rng.integers(0, 2600)), nch)) * rng.choice([1e-20, 1.0, 1e20])).astype(np.float32)
        w_ch.feed(dm)
        for c in range(nch):
            n_ch[c].feed(dm[:, c])
        if i % 11 == 5:
            w_in.clear(), n_in.clear(), w_ch.clear()
            for c in n_ch:
                c.clear()
        if i % 23 == 17:
            w_in, n_in = wr.InputLevels(kind, K), lr.InputLevels(kind, K)
            w_ch, n_ch = wr.ChanLevels(nch), [lr.ChanLevels() for _ in range(nch)]
        _same_input(w_in, n_in)
        _same_chans(w_ch, n_ch)
    assert w_ch.windows > 0 and w_in.samples > 0


def test_table_checks_see_a_wrong_entry():
    """check_inputs / check_chans fail on a count off by one, a peak's last bit, and a sum 1e-9 off"""
    import acarsdec_b200.api as api
    rng = np.random.default_rng(3)
    inp, ch = wr.InputLevels("cs16", 3), wr.ChanLevels(4)
    inp.feed(rng.integers(-9, 9, size=(3000, 2), dtype=np.int16))
    ch.feed(rng.random((3000, 4)).astype(np.float32))
    gi = np.zeros(1, api.INPUT_LEVEL_DTYPE)
    gi[0] = (inp.samples, inp.clipped, inp.power_sum(), inp.peak, 0)
    gc = np.zeros((1, 4), api.CHAN_LEVEL_DTYPE)
    for c in range(4):
        gc[0, c] = (ch.rows, ch.power_sum()[c], ch.peak[c], 0, ch.windows, ch.floor[c])
    wr.check_inputs(gi, [inp])
    wr.check_chans(gc, [ch])
    for f, bump in (("samples", lambda v: v + 1), ("power_sum", lambda v: v * (1 + 1e-9))):
        bad = gi.copy()
        bad[0][f] = bump(bad[0][f])
        with pytest.raises(AssertionError):
            wr.check_inputs(bad, [inp])
    for f, bump in (("windows", lambda v: v + 1), ("peak", lambda v: np.nextafter(v, np.float32(9))),
                    ("floor", lambda v: v * (1 + 1e-9))):
        bad = gc.copy()
        bad[0, 3][f] = bump(bad[0, 3][f])
        with pytest.raises(AssertionError):
            wr.check_chans(bad, [ch])
