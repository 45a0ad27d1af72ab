"""Restatement side of the decode statistics (ACB_FLAG_DECODE_STATS): tests/host/decode_stats_oracle.c (the counts,
on top of the pinned restatement oracle/libacars_oracle.so) and tests/host/demod_emul_counted.cpp (the device loop's
counting accessor on the host) through ctypes, and the reading of the reference's -v lines into the same counts."""
from __future__ import annotations

import ctypes as C
import re
from collections import Counter

import numpy as np

import refs
from acarsdec_b200 import api
from common import HOST, LIBDIR, _build_host_lib

FIELDS = api.DECODE_STATS_FIELDS
K2_FIELDS = ("preamble", "started", "txt_parity", "txt_long", "txt_missed_end", "emitted", "fec_short")


class OrcCounts(C.Structure):
    _fields_ = [(f, C.c_uint64) for f in FIELDS]

    def as_dict(self):
        return {f: int(getattr(self, f)) for f in FIELDS}


class SyncState(C.Structure):
    """dso_sync_t: the replayed frame synchroniser's state"""
    _fields_ = [("state", C.c_int), ("nbits", C.c_int), ("blk_len", C.c_int), ("blk_err", C.c_int), ("outbits", C.c_uint)]


_lib = None


def lib():
    """tests/host/decode_stats_oracle.c built by gcc against oracle/libacars_oracle.so"""
    global _lib
    if _lib is None:
        refs.ensure_built()
        src = HOST / "decode_stats_oracle.c"
        path = _build_host_lib(HOST / "libdecode_stats_oracle.so", src, lambda out: [
            "gcc", "-O2", "-std=gnu11", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-o", out, src,
            "-L", refs.ORACLE_DIR, "-lacars_oracle", "-Wl,-rpath," + str(refs.ORACLE_DIR), "-lm"])
        L = C.CDLL(str(path))
        L.dso_sync_init.argtypes = [C.POINTER(SyncState)]
        L.dso_demod.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.POINTER(SyncState), C.POINTER(OrcCounts)]
        L.dso_demod.restype = C.c_long
        L.dso_block_fec.argtypes = [C.POINTER(refs.Msg), C.POINTER(OrcCounts)]
        L.dso_block_fec.restype = C.c_int
        _lib = L
    return _lib


def emul_counted_lib():
    """tests/host/demod_emul_counted.cpp built by g++ (demod_emul.cpp with the counting accessor)"""
    src = HOST / "demod_emul_counted.cpp"
    return _build_host_lib(HOST / "libdemod_emul_counted.so", src, lambda out: [
        "g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", out, src,
        "-L", LIBDIR, "-lacars_b200", "-Wl,-rpath," + str(LIBDIR), "-lm"])


def new_sync() -> SyncState:
    s = SyncState()
    lib().dso_sync_init(C.byref(s))
    return s


def demod_counted(oracle: refs.OracleLib, chan: refs.OrcChan, sync: SyncState, dm: np.ndarray, sink: refs.Sink,
                  k: OrcCounts) -> None:
    """orc_demod over dm with the frame synchroniser's events counted; the replay must end where orc_demod did"""
    dm = np.ascontiguousarray(dm, dtype=np.float32)
    assert lib().dso_demod(C.byref(chan), oracle._h.ctypes.data, dm.ctypes.data, len(dm), C.byref(sink.c), C.byref(sync),
                           C.byref(k)) >= 0
    assert (sync.state, sync.nbits, sync.outbits & 0xFF) == (chan.state, chan.nbits, chan.outbits)


def fec_counted(oracle: refs.OracleLib, m: refs.Msg, k: OrcCounts):
    """blk_thread on a copy of m with its verdict added to k; returns the repaired copy or None, and holds both to the
    pinned orc_block_fec"""
    out = refs.Msg()
    C.memmove(C.byref(out), C.byref(m), C.sizeof(refs.Msg))
    keep = lib().dso_block_fec(C.byref(out), C.byref(k))
    want = oracle.fec(m)
    assert bool(keep) == (want is not None)
    if keep:
        assert (out.err, bytes(out.txt[:out.len])) == (want.err, bytes(want.txt[:want.len]))
    return out if keep else None


def restate_chain(oracle: refs.OracleLib, dm: np.ndarray, chunks=None, chan: refs.OrcChan | None = None):
    """One chain's envelope through the restatement, cut into `chunks` (default: whole): (counts dict, delivered
    messages, the channel state).  The state is returned so a caller can tell whether a block is still open."""
    k = OrcCounts()
    chan = chan if chan is not None else oracle.new_chan(0)
    sync = new_sync()
    sink = refs.Sink()
    pos = 0
    for n in (chunks if chunks is not None else [len(dm)]):
        if pos >= len(dm):
            break
        demod_counted(oracle, chan, sync, dm[pos:pos + n], sink, k)
        pos += n
    out = [m for m in (fec_counted(oracle, m, k) for m in sink.msgs()) if m is not None]
    return k.as_dict(), out, chan


def open_block(state: int) -> int:
    return int(state in (3, 4, 5))             # TXT, CRC1, CRC2 (acarsdec.h:88)


def check_invariants(d: dict, state: int) -> None:
    assert d["emitted"] == (d["fec_short"] + d["fec_parity_excess"] + d["fec_unfixable"] + d["fec_parity_problem"]
                            + d["delivered"] + d["lost"]), d
    assert d["started"] == d["emitted"] + d["txt_parity"] + d["txt_long"] + open_block(state), (d, state)


# the reference's -v lines (acars.c:101-206, 311-354) -> (field, channel index); None: a line no counter stands for
_LINES = [
    (re.compile(r"^#(\d+) too many parity errors$"), "txt_parity"),
    (re.compile(r"^#(\d+) miss txt end$"), "txt_missed_end"),
    (re.compile(r"^#(\d+) too long$"), "txt_long"),
    (re.compile(r"^put message #(\d+)$"), "emitted"),
    (re.compile(r"^#(\d+) too short$"), "fec_short"),
    (re.compile(r"^#(\d+) too many parity errors: \d+$"), "fec_parity_excess"),
    (re.compile(r"^#(\d+) parity error\(s\): \d+$"), "fec_parity"),
    (re.compile(r"^#(\d+) crc error$"), "fec_crc"),
    (re.compile(r"^#(\d+) errors fixed$"), "fec_fixed"),
    (re.compile(r"^#(\d+) not able to fix errors$"), "fec_unfixable"),
    (re.compile(r"^#(\d+) parity check problem$"), "fec_parity_problem"),
    (re.compile(r"^get message #(\d+)$"), None),
    (re.compile(r"^blk_starting$"), None),
]


def count_lines(text: str, skip_chn=()) -> dict:
    """{channel index: Counter(field)} of the reference's stderr; every line must be one of the known kinds."""
    out: dict[int, Counter] = {}
    for line in text.splitlines():
        for rx, field in _LINES:
            m = rx.match(line)
            if m:
                break
        else:
            raise AssertionError(f"unknown -v line: {line!r}")
        if field is None:
            continue
        chn = int(m.group(1)) - 1
        if chn in skip_chn:
            continue
        out.setdefault(chn, Counter())[field] += 1
    return out
