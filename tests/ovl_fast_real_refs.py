"""ctypes front-end for tests/host/ovl_fast_real_oracle.c, the CPU restatement of the pre-sum of the polyphase fast form
of the overlapping-window channelizer for real input (ACB_FLAG_FAST_FILTER_REAL, taps > K) (TEST INFRASTRUCTURE).

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
SRC = ROOT / "tests" / "host" / "ovl_fast_real_oracle.c"

_lib = None


def load():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="acb_ovl_fast_real_oracle_")
        so = Path(d) / "libovl_fast_real_oracle.so"
        subprocess.run([os.environ.get("CC", "gcc"), "-O2", "-std=gnu11", "-ffp-contract=off", "-fPIC", "-shared",
                        "-o", str(so), str(SRC), "-lm"], check=True)
        lib = C.CDLL(str(so))
        shutil.rmtree(d, ignore_errors=True)          # the mapping stays valid
        lib.orc_ovl_presum_real.restype = None
        lib.orc_ovl_presum_real.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        _lib = lib
    return _lib


def ovl_presum_real(x: np.ndarray, K: int, h: np.ndarray) -> np.ndarray:
    """The real-input pre-sum rows of a float32 stream -> (nout, K) float32; h the float prototype (acb_build_lowpass,
    taps entries)."""
    x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1)
    h = np.ascontiguousarray(h, dtype=np.float32)
    nout = x.size // K
    z = np.empty((nout, K), dtype=np.float32)
    load().orc_ovl_presum_real(x.ctypes.data, x.size, K, len(h), h.ctypes.data, z.ctypes.data)
    return z


def channelize_ovl_rdft(oracle, x: np.ndarray, K: int, h: np.ndarray, kbin: np.ndarray, tw: np.ndarray) -> np.ndarray:
    """Polyphase fast form of a float32 real stream -> (nch, nout): orc_channelize_rdft (the `oracle` library,
    refs.OracleLib) of the pre-sum rows; kbin / tw the fast plan of acb_fast_plan_air."""
    z = ovl_presum_real(x, K, h)
    return oracle.channelize_rdft(z.reshape(-1), K, kbin, tw)
