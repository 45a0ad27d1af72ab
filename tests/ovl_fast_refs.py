"""ctypes front-end for tests/host/ovl_fast_oracle.c, the CPU restatement of the polyphase fast form of the
overlapping-window channelizer (ACB_FLAG_FAST_FILTER, taps > K) (TEST INFRASTRUCTURE).

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
SRC = ROOT / "tests" / "host" / "ovl_fast_oracle.c"

_lib = None


def load():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="acb_ovl_fast_oracle_")
        so = Path(d) / "libovl_fast_oracle.so"
        subprocess.run([os.environ.get("CC", "gcc"), "-O2", "-std=gnu11", "-ffp-contract=off", "-fPIC", "-shared",
                        "-o", str(so), str(SRC), "-lm"], check=True)
        lib = C.CDLL(str(so))
        shutil.rmtree(d, ignore_errors=True)          # the mapping stays valid
        for name in ("orc_channelize_ovl_fast", "orc_channelize_ovl_fast_cs16"):
            fn = getattr(lib, name)
            fn.restype = None
            fn.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = lib
    return _lib


def _run(fn, x, nsamp: int, K: int, h: np.ndarray, kbin: np.ndarray, tw: np.ndarray) -> np.ndarray:
    h = np.ascontiguousarray(h, dtype=np.float32)
    kbin = np.ascontiguousarray(kbin, dtype=np.int32)
    tw = np.ascontiguousarray(tw, dtype=np.float32)             # (nch, K/4, 2)
    nch, nout = len(kbin), nsamp // K
    dm = np.empty((nch, nout), dtype=np.float32)
    fn(x.ctypes.data, nsamp, K, len(h), nch, h.ctypes.data, kbin.ctypes.data, tw.ctypes.data, dm.ctypes.data)
    return dm


def channelize_ovl_fast(iq: np.ndarray, K: int, h: np.ndarray, kbin: np.ndarray, tw: np.ndarray) -> np.ndarray:
    """Polyphase fast form of a u8 IQ stream -> (nch, nout); h the float prototype (acb_build_lowpass, taps entries),
    kbin / tw the fast plan (acb_fast_plan: tw (nch, K/4, 2) float32)."""
    iq = np.ascontiguousarray(iq, dtype=np.uint8).reshape(-1)
    return _run(load().orc_channelize_ovl_fast, iq, iq.size // 2, K, h, kbin, tw)


def channelize_ovl_fast_cs16(iq: np.ndarray, K: int, h: np.ndarray, kbin: np.ndarray, tw: np.ndarray) -> np.ndarray:
    """The same for CS16 input; tw from acb_fast_plan_cs16 carries the variant's scale."""
    iq = np.ascontiguousarray(iq, dtype=np.int16).reshape(-1)
    return _run(load().orc_channelize_ovl_fast_cs16, iq, iq.size // 2, K, h, kbin, tw)
