"""The float64 definition of the level tables (tests/level_stats_refs.py) in a form that scales to wide shapes: 10^8
samples per stream, hundreds of channels, thousands of rows per submit.

The semantics are level_stats_refs.py's: rows [m*K, (m+1)*K), a streaming kind's samples waiting in the carry until
their row completes, windows of 1024 rows counted from the stream's own start, clear() (reset != 0) keeping the carry
and the open window, and a new object for acb_reset_stream.  Only the sums are made differently, so that nothing keeps
every squared term:
  u8       a byte histogram per stream (exact counts); the power is math.fsum over the 256 terms count[b] * v(b)^2,
           v = float32(b) - 127.37f;
  CS16     I^2 + Q^2 summed in int64 (exact);
  real     a float64 np.sum per submit, then math.fsum over those partial sums;
  envelope a float64 np.sum per submit and per window (all channels at once), then math.fsum over the partial sums.
Clipped counts, sample and row counts, windows and peaks are exact."""
from __future__ import annotations

import math

import numpy as np

from level_stats_refs import OUTBLK, clipped, convert

U8_V = (np.arange(256, dtype=np.float32) - np.float32(127.37)).astype(np.float64)      # v(b), exact in float64


class InputLevels:
    """acb_input_level_t of one stream.  feed() takes a submit's new samples (u8: bytes or (n, 2); CS16: (n, 2); real:
    (n,)) and returns the rows they complete."""

    def __init__(self, kind: str, K: int):
        self.kind, self.K = kind, K
        self.carry = None
        self.clear()

    def clear(self):
        self.samples = self.clipped = 0
        self.hist = np.zeros(256, np.int64)          # u8: how often each byte value occurred (I and Q alike)
        self.sq = 0                                  # CS16: sum of I^2 + Q^2, a Python int
        self.parts: list[float] = []                 # real: one float64 partial sum per submit
        self.peak = np.float32(0.0)

    def feed(self, x) -> int:
        x = np.asarray(x)
        if self.kind == "u8":
            x = x.reshape(-1, 2)
        x = x if self.carry is None or not len(self.carry) else np.concatenate([self.carry, x])
        rows = len(x) // self.K
        done, self.carry = x[:rows * self.K], x[rows * self.K:]
        if not rows:
            return 0
        self.samples += len(done)
        self.clipped += int(clipped(self.kind, done).sum())
        if self.kind == "u8":
            h = np.bincount(done.reshape(-1), minlength=256)
            self.hist += h
            seen = np.nonzero(h)[0]
            self.peak = max(self.peak, np.float32(np.abs(U8_V[seen]).max()))
        elif self.kind == "cs16":
            v = done.astype(np.int64)
            self.sq += int((v * v).sum())
            self.peak = max(self.peak, np.float32(np.abs(v).max()))
        else:
            v = done.astype(np.float64)
            self.parts.append(float(np.sum(v * v)))
            self.peak = max(self.peak, np.float32(np.abs(done).max()))
        return rows

    def power_sum(self) -> float:
        if self.kind == "u8":
            return math.fsum((self.hist.astype(np.float64) * U8_V * U8_V).tolist())
        if self.kind == "cs16":
            return float(self.sq)
        return math.fsum(self.parts)

    def row(self) -> tuple:
        return (self.samples, self.clipped, self.power_sum(), float(self.peak))


class ChanLevels:
    """acb_chan_level_t of every chain of one stream at once.  feed() takes a submit's envelope rows (n, nch)."""

    def __init__(self, nch: int):
        self.nch = nch
        self.open: list[np.ndarray] = []            # per-channel partial sums of the window not yet complete
        self.open_rows = 0
        self.clear()

    def clear(self):
        """reset != 0: the counts restart, the open window stays"""
        self.parts: list[np.ndarray] = []
        self.rows = self.windows = 0
        self.peak = np.zeros(self.nch, np.float32)
        self.floor = np.zeros(self.nch, np.float64)

    def feed(self, dm):
        dm = np.asarray(dm, dtype=np.float32).reshape(-1, self.nch)
        if not len(dm):
            return
        sq = dm.astype(np.float64) ** 2
        self.parts.append(sq.sum(axis=0))
        self.rows += len(dm)
        self.peak = np.maximum(self.peak, dm.max(axis=0))
        i = 0
        while i < len(sq):
            take = min(OUTBLK - self.open_rows, len(sq) - i)
            self.open.append(sq[i:i + take].sum(axis=0))
            self.open_rows += take
            i += take
            if self.open_rows == OUTBLK:
                mean = _fsum_rows(self.open) / OUTBLK
                self.floor = mean if self.windows == 0 else np.minimum(self.floor, mean)
                self.windows += 1
                self.open, self.open_rows = [], 0

    def power_sum(self) -> np.ndarray:
        return _fsum_rows(self.parts) if self.parts else np.zeros(self.nch)


def _fsum_rows(parts: list[np.ndarray]) -> np.ndarray:
    """math.fsum over a list of per-channel arrays, channel by channel"""
    a = np.stack(parts)
    return np.array([math.fsum(a[:, c].tolist()) for c in range(a.shape[1])])


def _close(got: np.ndarray, want: np.ndarray, rel: float) -> np.ndarray:
    """elementwise |got - want| <= rel * |want| (exact where want is 0)"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return np.abs(got - want) <= rel * np.abs(want)


def check_inputs(got: np.ndarray, refs: list[InputLevels], rel: float = 1e-10, streams=None):
    """an acb_input_level_t table against the definition: counts and peak exact, power within `rel`"""
    for s in range(len(refs)) if streams is None else streams:
        samples, clip, p, peak = refs[s].row()
        g = got[s]
        assert (int(g["samples"]), int(g["clipped"]), float(g["peak"])) == (samples, clip, peak), (s, g, refs[s].row())
        assert _close(g["power_sum"], p, rel), (s, g, refs[s].row())


def check_chans(got: np.ndarray, refs: list[ChanLevels], rel: float = 1e-10, streams=None):
    """an (nstreams, nch) acb_chan_level_t table against the definition: rows, windows and peak exact, power and floor
    within `rel`"""
    for s in range(len(refs)) if streams is None else streams:
        r, g = refs[s], got[s]
        assert (g["rows"] == r.rows).all() and (g["windows"] == r.windows).all(), (s, g["rows"], r.rows, g["windows"], r.windows)
        bad = np.nonzero(g["peak"] != r.peak)[0]
        assert not len(bad), (s, "peak", bad[:8], g["peak"][bad[:8]], r.peak[bad[:8]])
        for f, want in (("power_sum", r.power_sum()), ("floor", r.floor)):
            bad = np.nonzero(~_close(g[f], want, rel))[0]
            assert not len(bad), (s, f, bad[:8], g[f][bad[:8]], want[bad[:8]])
