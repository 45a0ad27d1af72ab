"""The level tables' float64 definition (tests/level_stats_refs.py) on hand-worked cases, and the ctypes dtypes against
the C structs (include/acars_b200.h) through a small C probe."""
import math
import shutil
import subprocess

import numpy as np
import pytest

import level_stats_refs as lr
from acarsdec_b200 import api
from common import ROOT


def test_window_split_over_three_submits():
    ch = lr.ChanLevels()
    parts = [np.full(500, 1.0), np.full(400, 2.0), np.full(300, 3.0)]
    ch.feed(parts[0])
    ch.feed(parts[1])
    assert (ch.rows, ch.windows) == (900, 0) and ch.floor == 0.0
    ch.feed(parts[2])
    # rows 0..1023: 500 ones, 400 twos, 124 threes; the last 176 threes stay open
    assert (ch.rows, ch.windows, ch.open_rows) == (1200, 1, 176)
    assert ch.floor == (500 * 1 + 400 * 4 + 124 * 9) / 1024
    assert ch.power_sum() == 500 * 1 + 400 * 4 + 300 * 9
    assert ch.peak == 3.0
    ch.clear()                                         # reset != 0 keeps the open window
    ch.feed(np.full(848, 0.5))
    assert (ch.rows, ch.windows) == (848, 1)
    assert ch.floor == (176 * 9 + 848 * 0.25) / 1024


def test_streaming_carry_completes_a_row_in_the_next_submit():
    inp = lr.InputLevels("real", 4)
    x = np.array([0.5, -0.25, 0.125, 0.0, 1.0, -1.0, 0.75, 0.5], np.float32)
    assert inp.feed(x[:6]) == 1                        # one row: x[0:4]; x[4:6] carried
    assert (inp.samples, inp.clipped) == (4, 0)
    assert inp.power_sum() == 0.25 + 0.0625 + 0.015625
    assert inp.feed(x[6:]) == 1                        # the carried pair completes row 1 with the new pair
    assert (inp.samples, inp.clipped) == (8, 2)        # 1.0 and -1.0 are full scale
    assert inp.power_sum() == 0.25 + 0.0625 + 0.015625 + 1 + 1 + 0.5625 + 0.25
    assert inp.peak == 1.0


def test_taps_history_is_not_counted_twice():
    K, taps, rows = 8, 20, 6
    spans = lr.row_spans(rows, K, taps)
    seen = np.zeros(rows * K, np.int64)
    for a, b in spans:
        seen[a:b] += 1
    assert (seen == 1).all()                           # each sample once, though each window reads taps - K before it
    windows = [(max(0, (m + 1) * K - taps), (m + 1) * K) for m in range(rows)]
    assert sum(b - a for a, b in windows) > rows * K


def test_full_scale_codes():
    u8 = np.array([[0, 128], [255, 128], [1, 254], [128, 0], [127, 127]], np.uint8)
    assert lr.clipped("u8", u8).tolist() == [True, True, False, True, False]
    cs = np.array([[-32768, 0], [0, 32767], [-32767, 32766], [5, -5]], np.int16)
    assert lr.clipped("cs16", cs).tolist() == [True, True, False, False]
    re = np.array([-1.0, -1.5, -2047 / 2048, 2047 / 2048, 2046 / 2048, 1.0, 0.0], np.float32)
    assert lr.clipped("real", re).tolist() == [True, True, False, True, False, True, False]
    # the converted extremes and the full-scale amplitudes the header states
    assert float(lr.convert("u8", np.array([0], np.uint8))[0]) == float(np.float32(0) - np.float32(127.37))
    assert lr.FULL_SCALE == api.FULL_SCALE == {"u8": 127.5, "cs16": 32768.0, "real": 1.0}
    inp = lr.InputLevels("u8", 1)
    inp.feed(np.array([0, 255, 127, 128], np.uint8))
    assert (inp.samples, inp.clipped) == (2, 1)
    assert inp.peak == np.float32(255) - np.float32(127.37)      # |255 - 127.37f| is larger than |0 - 127.37f|
    v = [np.float64(np.float32(b) - np.float32(127.37)) for b in (0, 255, 127, 128)]
    assert inp.power_sum() == math.fsum(t * t for t in v)


PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "acars_b200.h"
#define F(T, f) printf(#T " " #f " %zu %zu\n", offsetof(T, f), sizeof(((T *)0)->f))
int main(void)
{
	printf("acb_input_level_t size %zu\n", sizeof(acb_input_level_t));
	printf("acb_chan_level_t size %zu\n", sizeof(acb_chan_level_t));
	F(acb_input_level_t, samples); F(acb_input_level_t, clipped); F(acb_input_level_t, power_sum);
	F(acb_input_level_t, peak); F(acb_input_level_t, pad);
	F(acb_chan_level_t, rows); F(acb_chan_level_t, power_sum); F(acb_chan_level_t, peak); F(acb_chan_level_t, pad);
	F(acb_chan_level_t, windows); F(acb_chan_level_t, floor);
	printf("flag %d\n", ACB_FLAG_LEVEL_STATS);
	return 0;
}
"""


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no C compiler")
def test_dtypes_match_the_c_structs(tmp_path):
    src = tmp_path / "probe.c"
    src.write_text(PROBE)
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-std=c11", "-I", str(ROOT / "include"), "-o", str(exe), str(src)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    dtypes = {"acb_input_level_t": api.INPUT_LEVEL_DTYPE, "acb_chan_level_t": api.CHAN_LEVEL_DTYPE}
    for line in filter(None, out):
        w = line.split()
        if w[0] == "flag":
            assert int(w[1]) == api.FLAG_LEVEL_STATS
        elif w[1] == "size":
            assert int(w[2]) == dtypes[w[0]].itemsize, line
        else:
            dt = dtypes[w[0]]
            assert (dt.fields[w[1]][1], dt.fields[w[1]][0].itemsize) == (int(w[2]), int(w[3])), line
