"""ctypes front-end for tests/host/fir_stream_oracle.c, the CPU restatement (the definition) of the short channel filter
(taps <= K) on the streaming front-ends' 4-byte input (TEST INFRASTRUCTURE).

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
SRC = ROOT / "tests" / "host" / "fir_stream_oracle.c"

_lib = None


def load():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="acb_fir_stream_oracle_")
        so = Path(d) / "libfir_stream_oracle.so"
        subprocess.run([os.environ.get("CC", "gcc"), "-O2", "-std=gnu11", "-ffp-contract=off", "-fPIC", "-shared",
                        "-o", str(so), str(SRC), "-lm"], check=True)
        lib = C.CDLL(str(so))
        shutil.rmtree(d, ignore_errors=True)          # the mapping stays valid
        for name in ("orc_channelize_fir_real", "orc_channelize_fir_cs16"):
            fn = getattr(lib, name)
            fn.restype = None
            fn.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        _lib = lib
    return _lib


def _run(fn, x, nsamp: int, K: int, wf: np.ndarray) -> np.ndarray:
    wf = np.ascontiguousarray(wf, dtype=np.float32)
    nch, taps = wf.shape[0], wf.shape[1] // 2
    assert 1 <= taps <= K
    nout = nsamp // K
    dm = np.empty((nch, nout), dtype=np.float32)
    fn(x.ctypes.data, nsamp, K, taps, nch, wf.ctypes.data, dm.ctypes.data)
    return dm


def channelize_fir_real(x: np.ndarray, K: int, wf: np.ndarray) -> np.ndarray:
    """float32 real stream -> (nch, nout) envelope; wf (nch, 2*taps), taps <= K."""
    x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1)
    return _run(load().orc_channelize_fir_real, x, x.size, K, wf)


def channelize_fir_cs16(iq: np.ndarray, K: int, wf: np.ndarray) -> np.ndarray:
    """int16 IQ stream (n, 2) or interleaved -> (nch, nout); wf carries the front-end's folded scale."""
    iq = np.ascontiguousarray(iq, dtype=np.int16).reshape(-1)
    return _run(load().orc_channelize_fir_cs16, iq, iq.size // 2, K, wf)


def fir_f64(x: np.ndarray, K: int, wf: np.ndarray):
    """The same sum in float64 (complex128), exact products of the float32 operands: ((nch, nout) |D|, (nch, nout)
    S = sum_i |x[mK+i]| * |w[i]|, the scale of the rounding error)."""
    wf = np.asarray(wf, dtype=np.float64)
    taps = wf.shape[1] // 2
    w = wf[:, 0::2] + 1j * wf[:, 1::2]                                    # (nch, taps)
    if np.asarray(x).dtype == np.int16:
        x = np.asarray(x, dtype=np.float64).reshape(-1, 2)
        x = x[:, 0] + 1j * x[:, 1]
    else:
        x = np.asarray(x, dtype=np.float64).reshape(-1)
    nout = x.size // K
    rows = x[:nout * K].reshape(nout, K)[:, :taps]                        # (nout, taps)
    d = rows @ w.T                                                        # (nout, nch)
    s = np.abs(rows) @ np.abs(w).T
    return np.abs(d).T, s.T
