"""ctypes front-end for tests/host/ovl_oracle.c, the CPU restatement (the definition) of the overlapping-window
channelizer (taps > K), plus the numpy restatement of its prototype filter (TEST INFRASTRUCTURE).

The library is compiled once per process into a temporary directory, so the tree may stay read-only."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
SRC = ROOT / "tests" / "host" / "ovl_oracle.c"

_lib = None


def load():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="acb_ovl_oracle_")
        so = Path(d) / "libovl_oracle.so"
        subprocess.run([os.environ.get("CC", "gcc"), "-O2", "-std=gnu11", "-ffp-contract=off", "-fPIC", "-shared",
                        "-o", str(so), str(SRC), "-lm"], check=True)
        lib = C.CDLL(str(so))
        shutil.rmtree(d, ignore_errors=True)          # the mapping stays valid
        for name in ("orc_channelize_ovl", "orc_channelize_ovl_cs16", "orc_channelize_ovl_real"):
            fn = getattr(lib, name)
            fn.restype = None
            fn.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        _lib = lib
    return _lib


def _run(fn, x, nsamp: int, K: int, wf: np.ndarray) -> np.ndarray:
    wf = np.ascontiguousarray(wf, dtype=np.float32)
    nch, taps = wf.shape[0], wf.shape[1] // 2
    nout = nsamp // K
    dm = np.empty((nch, nout), dtype=np.float32)
    fn(x.ctypes.data, nsamp, K, taps, nch, wf.ctypes.data, dm.ctypes.data)
    return dm


def channelize_ovl(iq: np.ndarray, K: int, wf: np.ndarray) -> np.ndarray:
    """u8 IQ stream (interleaved I,Q bytes) -> (nch, nout) envelope; wf (nch, 2*taps)."""
    iq = np.ascontiguousarray(iq, dtype=np.uint8).reshape(-1)
    return _run(load().orc_channelize_ovl, iq, iq.size // 2, K, wf)


def channelize_ovl_cs16(iq: np.ndarray, K: int, wf: np.ndarray) -> np.ndarray:
    """int16 IQ stream (n, 2) or interleaved -> (nch, nout); wf carries the front-end's folded scale."""
    iq = np.ascontiguousarray(iq, dtype=np.int16).reshape(-1)
    return _run(load().orc_channelize_ovl_cs16, iq, iq.size // 2, K, wf)


def channelize_ovl_real(x: np.ndarray, K: int, wf: np.ndarray) -> np.ndarray:
    x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1)
    return _run(load().orc_channelize_ovl_real, x, x.size, K, wf)


def lowpass_f64(K: int, taps: int) -> np.ndarray:
    """acb_build_lowpass restated in float64: ideal low-pass at 1/(2K) cycles/sample centred at (taps-1)/2, Kaiser
    window beta = 6, normalised to sum 1 (before the float rounding)."""
    n = np.arange(taps, dtype=np.float64)
    fc = 0.5 / K
    h = 2 * fc * np.sinc(2 * fc * (n - (taps - 1) / 2)) * np.kaiser(taps, 6.0)
    return h / h.sum()


def response_db(w: np.ndarray, freqs_hz, rate: float) -> np.ndarray:
    """|sum_i w[i] exp(-j 2 pi f i / rate)| in dB (float64) for a complex or real table w."""
    w = np.asarray(w, dtype=np.complex128)
    i = np.arange(len(w))
    f = np.asarray(freqs_hz, dtype=np.float64)
    resp = np.exp(-2j * np.pi * np.outer(f, i) / rate) @ w
    return 20 * np.log10(np.maximum(np.abs(resp), 1e-300))
