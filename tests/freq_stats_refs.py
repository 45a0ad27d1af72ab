"""The float64 definition of the frequency-error table (ACB_FLAG_FREQ_STATS, include/acars_b200.h: acb_chan_freq_t), one
stream at a time, fed submit by submit, and the planners' record of each chain (freq_hz, step) restated from the header.

Each output row m of a stream has its own K input samples [m*K, (m+1)*K), converted as the channelizer converts them.
With h = K // 2, a_m = sum_{n<h} x[mK+n] w[n] and b_m = sum_{n<h} x[mK+h+n] w[h+n], w[n] = (float)cos(step n) -
j (float)sin(step n).  Per chain: pairs, sum b conj(a), sum |a||b|, sum |a|^2 + |b|^2."""
from __future__ import annotations

import math

import numpy as np

INTRATE = 12500


def nco(step: float, K: int) -> np.ndarray:
    """The chain's table as the device holds it: float32 components, evaluated in double"""
    ph = step * np.arange(K, dtype=np.float64)
    return np.cos(ph).astype(np.float32).astype(np.float64) - 1j * np.sin(ph).astype(np.float32).astype(np.float64)


def convert(kind: str, x: np.ndarray) -> np.ndarray:
    """Samples as the channelizer converts them: u8 / CS16 (n, 2) components to complex, real (n,) as they are"""
    if kind == "u8":
        v = np.asarray(x).reshape(-1, 2).astype(np.float32) - np.float32(127.37)
    elif kind == "cs16":
        v = np.asarray(x).reshape(-1, 2).astype(np.float32)
    else:
        return np.asarray(x, dtype=np.float32).astype(np.float64)
    return v[:, 0].astype(np.float64) + 1j * v[:, 1].astype(np.float64)


def plan_record(kind: str, K: int, freqs_hz, fc: int) -> tuple[np.ndarray, np.ndarray]:
    """(freq_hz, step) per chain as the planners record them (u8: acb_set_plan*, cs16: acb_set_plan_cs16, real:
    acb_set_plan_air*): the mixer's offset from the tuner centre, and for real input the mirror image of air.c's IF."""
    rate = K * INTRATE
    f32 = np.float32
    if kind == "u8":
        off = [float(f32(f32(int(f32(f)))) - f32(fc)) for f in freqs_hz]      # acb_stored_fr: (int)(float)Fr
        f0 = float(fc)
    elif kind == "cs16":
        off = [float(f32(f) - f32(fc)) for f in freqs_hz]
        f0 = float(fc)
    else:
        off = [-float((int(fc) - int(f) + rate // 4) & 0xFFFFFFFF) for f in freqs_hz]
        f0 = float(fc) + rate // 4
    off = np.array(off)
    return f0 + off, 2 * np.pi * off / rate


class ChainFreq:
    """acb_chan_freq_t sums of one stream's chains.  feed() takes a submit's new samples (u8 / CS16: (n, 2); real: (n,))."""

    def __init__(self, kind: str, K: int, steps):
        self.kind, self.K = kind, K
        self.w = [nco(float(st), K) for st in steps]
        self.carry = None
        self.clear()

    def replan(self, steps):
        """a re-plan: the rows after it are measured with the new tables"""
        self.w = [nco(float(st), self.K) for st in steps]

    def clear(self):
        """reset != 0: the sums restart, the carried samples stay"""
        n = len(self.w)
        self.pairs = 0
        self.terms = [[] for _ in range(n)]

    def feed(self, x: np.ndarray) -> int:
        x = np.asarray(x)
        if self.kind != "real":
            x = x.reshape(-1, 2)
        x = x if self.carry is None else np.concatenate([self.carry, x])
        rows = len(x) // self.K
        done, self.carry = x[:rows * self.K], x[rows * self.K:]
        if rows:
            v = convert(self.kind, done).reshape(rows, self.K)
            h = self.K // 2
            W = np.stack(self.w, axis=1)                     # (K, nch)
            a, b = v[:, :h] @ W[:h], v[:, h:2 * h] @ W[h:2 * h]
            p = b * np.conj(a)
            t = np.stack([p.real, p.imag, np.abs(a) * np.abs(b), np.abs(a) ** 2 + np.abs(b) ** 2])     # (4, rows, nch)
            for c in range(len(self.w)):
                self.terms[c].append(t[:, :, c])
            self.pairs += rows
        return rows

    def sums(self, c: int) -> tuple[float, float, float, float]:
        if not self.terms[c]:
            return 0.0, 0.0, 0.0, 0.0
        t = np.concatenate(self.terms[c], axis=1)
        return tuple(math.fsum(t[i].tolist()) for i in range(4))


def offsets(s_re, s_im, K: int) -> np.ndarray:
    """rate * atan2(s_im, s_re) / (2 pi h): the carrier's offset from freq_hz, in Hz"""
    return K * INTRATE * np.arctan2(s_im, s_re) / (2 * np.pi * (K // 2))


def ppm(s_re, s_im, freq_hz, K: int) -> float:
    w = np.hypot(s_re, s_im)
    return float(1e6 * np.sum(w * offsets(s_re, s_im, K) / freq_hz) / np.sum(w))


def check_chain(got, ref: ChainFreq, c: int, rel: float = 1e-5):
    """one acb_chan_freq_t against the definition: pairs exact; s, mag_sum within rel * mag_sum, power_sum within
    rel * power_sum"""
    re, im, mag, pw = ref.sums(c)
    assert int(got["pairs"]) == ref.pairs, (got, ref.pairs)
    for name, v, scale in (("s_re", re, mag), ("s_im", im, mag), ("mag_sum", mag, mag), ("power_sum", pw, pw)):
        assert abs(float(got[name]) - v) <= rel * scale + 1e-300, (name, float(got[name]), v, scale)
