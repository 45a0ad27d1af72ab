"""The float64 definition of the level tables (ACB_FLAG_LEVEL_STATS, include/acars_b200.h: acb_input_level_t,
acb_chan_level_t), one stream at a time, fed submit by submit.

Input: every sample of the K-sample span [m*K, (m+1)*K) of each output row m counts once; a streaming kind's samples
wait in the carry until their row completes.  Components are converted as the channelizer converts them (float32), and
sums are math.fsum over the exact float64 squares.  Envelope: windows of 1024 rows from the stream's own start, a window
counting when the submit that completes it is made."""
from __future__ import annotations

import math

import numpy as np

OUTBLK = 1024
FULL_SCALE = {"u8": 127.5, "cs16": 32768.0, "real": 1.0}


def convert(kind: str, x: np.ndarray) -> np.ndarray:
    """Components as float32, as K1 converts them: u8 (float)b - 127.37f, CS16 (float)int16, real the float itself."""
    if kind == "u8":
        return x.astype(np.float32) - np.float32(127.37)
    return x.astype(np.float32)


def clipped(kind: str, x: np.ndarray) -> np.ndarray:
    """Per sample (x: u8 / CS16 (n, 2) components, real (n,)): a component at full scale."""
    if kind == "u8":
        return ((x == 0) | (x == 255)).any(axis=-1)
    if kind == "cs16":
        return ((x == -32768) | (x == 32767)).any(axis=-1)
    return (x <= np.float32(-1.0)) | (x >= np.float32(2047.0 / 2048.0))


def row_spans(rows: int, K: int, taps: int) -> list[tuple[int, int]]:
    """The samples each row counts, [m*K, (m+1)*K), whatever the window K1 reads for it ([(m+1)*K - taps, (m+1)*K))."""
    del taps                                        # the window's history belongs to the rows before: not counted again
    return [(m * K, (m + 1) * K) for m in range(rows)]


class InputLevels:
    """acb_input_level_t of one stream.  feed() takes a submit's new samples (u8 / CS16: (n, 2); real: (n,))."""

    def __init__(self, kind: str, K: int):
        self.kind, self.K = kind, K
        self.carry = None
        self.terms: list[np.ndarray] = []
        self.samples = self.clipped = 0
        self.peak = np.float32(0.0)

    def feed(self, x: np.ndarray) -> int:
        x = np.asarray(x)
        if self.kind == "u8":
            x = x.reshape(-1, 2)
        x = x if self.carry is None else np.concatenate([self.carry, x])
        rows = len(x) // self.K
        done, self.carry = x[:rows * self.K], x[rows * self.K:]
        if rows:
            v = convert(self.kind, done).astype(np.float64)
            self.terms.append((v * v).reshape(-1))          # every component's exact square: I^2 and Q^2, or x^2
            self.samples += len(done)
            self.clipped += int(clipped(self.kind, done).sum())
            self.peak = max(self.peak, np.float32(np.abs(convert(self.kind, done)).max()))
        return rows

    def clear(self):
        """reset != 0: the counts restart, the carried samples stay (they belong to a row not yet produced)"""
        self.terms, self.samples, self.clipped, self.peak = [], 0, 0, np.float32(0.0)

    def power_sum(self) -> float:
        return math.fsum(np.concatenate(self.terms).tolist()) if self.terms else 0.0

    def row(self) -> tuple:
        return (self.samples, self.clipped, self.power_sum(), float(self.peak))


class ChanLevels:
    """acb_chan_level_t of one chain.  feed() takes a submit's envelope rows of the chain (float32)."""

    def __init__(self):
        self.open: list[np.ndarray] = []            # the window not yet complete
        self.open_rows = 0
        self.clear()

    def clear(self):
        """reset != 0: the counts restart, the open window stays"""
        self.terms: list[np.ndarray] = []
        self.rows = self.windows = 0
        self.peak = np.float32(0.0)
        self.floor = 0.0

    def feed(self, dm: np.ndarray):
        dm = np.asarray(dm, dtype=np.float32)
        if not len(dm):
            return
        sq = dm.astype(np.float64) ** 2
        self.terms.append(sq)
        self.rows += len(dm)
        self.peak = max(self.peak, np.float32(dm.max()))
        i = 0
        while i < len(sq):
            take = min(OUTBLK - self.open_rows, len(sq) - i)
            self.open.append(sq[i:i + take])
            self.open_rows += take
            i += take
            if self.open_rows == OUTBLK:
                mean = math.fsum(np.concatenate(self.open).tolist()) / OUTBLK
                self.floor = mean if self.windows == 0 else min(self.floor, mean)
                self.windows += 1
                self.open, self.open_rows = [], 0

    def power_sum(self) -> float:
        return math.fsum(np.concatenate(self.terms).tolist()) if self.terms else 0.0

    def row(self) -> tuple:
        return (self.rows, self.power_sum(), float(self.peak), self.windows, self.floor)


def check_input(got, ref: InputLevels, rel: float = 1e-10):
    """one acb_input_level_t against the definition: counts and peak exact, power within `rel`"""
    samples, clip, p, peak = ref.row()
    assert int(got["samples"]) == samples and int(got["clipped"]) == clip, (got, ref.row())
    assert float(got["peak"]) == peak, (got, ref.row())
    assert math.isclose(float(got["power_sum"]), p, rel_tol=rel, abs_tol=0.0 if p else 1e-300), (got, ref.row())


def check_chan(got, ref: ChanLevels, rel: float = 1e-10):
    """one acb_chan_level_t against the definition: rows, windows and peak exact, power and floor within `rel`"""
    rows, p, peak, windows, floor = ref.row()
    assert int(got["rows"]) == rows and int(got["windows"]) == windows, (got, ref.row())
    assert float(got["peak"]) == peak, (got, ref.row())
    assert math.isclose(float(got["power_sum"]), p, rel_tol=rel, abs_tol=0.0 if p else 1e-300), (got, ref.row())
    assert math.isclose(float(got["floor"]), floor, rel_tol=rel, abs_tol=0.0 if floor else 1e-300), (got, ref.row())
