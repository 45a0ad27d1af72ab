"""ctypes binding of the C ABI in include/acars_b200.h.

This is host-side convenience for the tests and bench.py; the product is the shared library.
There is no CPU fallback: importing works anywhere (so the symbol tests can run on a CPU-only
box), but creating a Context without an H100 raises, and a missing libacars_b200.so raises at
import of this module.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

PKG = Path(__file__).resolve().parent
LIB_PATH = PKG / "libacars_b200.so"

OUTBLK = 1024
TXTMAX = 250
FLAG_FAST_WIDEBAND = 64          # ACB_FLAG_FAST_WIDEBAND: the fast forms for any K % 8 == 0 and any channel count
FLAG_FAST_WIDEBAND_REAL = 128    # ACB_FLAG_FAST_WIDEBAND_REAL: the same for real input (air.c)
FLAG_DECODE_STATS = 256          # ACB_FLAG_DECODE_STATS: per-chain decode statistics (Context.decode_stats)
FLAG_LEVEL_STATS = 512           # ACB_FLAG_LEVEL_STATS: input and envelope levels (Context.level_stats)
FLAG_FREQ_STATS = 1024           # ACB_FLAG_FREQ_STATS: per-chain carrier offsets (Context.freq_stats, freq_error)


class Config(C.Structure):
    _fields_ = [("device", C.c_int), ("K", C.c_int), ("nstreams", C.c_int), ("nch", C.c_int),
                ("max_blocks", C.c_int), ("flags", C.c_int), ("taps", C.c_int)]


class Msg(C.Structure):
    _fields_ = [("stream", C.c_int), ("chn", C.c_int), ("len", C.c_int), ("err", C.c_int), ("lvl", C.c_float),
                ("block", C.c_uint64), ("pos", C.c_uint64), ("soh_pos", C.c_uint64),
                ("txt", C.c_ubyte * TXTMAX), ("crc", C.c_ubyte * 2)]

    def as_tuple(self):
        """(chn, len, err, txt, crc) — the fields the reference's msgblk_t carries."""
        return (self.chn, self.len, self.err, bytes(self.txt[:self.len]), bytes(self.crc))

    def key(self):
        return self.as_tuple() + (np.float32(self.lvl).tobytes(),)


# acb_msg_t as a numpy record (same layout as the ctypes Msg above; checked at import)
MSG_DTYPE = np.dtype([("stream", "<i4"), ("chn", "<i4"), ("len", "<i4"), ("err", "<i4"), ("lvl", "<f4"),
                      ("block", "<u8"), ("pos", "<u8"), ("soh_pos", "<u8"), ("txt", "u1", (TXTMAX,)), ("crc", "u1", (2,))],
                     align=True)
assert MSG_DTYPE.itemsize == C.sizeof(Msg)


class Fields(C.Structure):
    """acb_fields_t: outputmsg's field split + label.c's OOOI fields (include/acars_b200.h)."""
    _fields_ = [("mode", C.c_char), ("ack", C.c_char), ("bid", C.c_char), ("bs", C.c_char), ("be", C.c_char),
                ("addr", C.c_char * 8), ("label", C.c_char * 3), ("no", C.c_char * 5), ("fid", C.c_char * 7),
                ("downlink", C.c_int), ("txt_off", C.c_int), ("txt_len", C.c_int), ("has_oooi", C.c_int),
                ("da", C.c_char * 5), ("sa", C.c_char * 5), ("eta", C.c_char * 5), ("gout", C.c_char * 5),
                ("gin", C.c_char * 5), ("woff", C.c_char * 5), ("won", C.c_char * 5)]


class FmtOpts(C.Structure):
    """acb_fmt_opts_t"""
    _fields_ = [("tv_sec", C.c_int64), ("tv_usec", C.c_int64), ("freq_hz", C.c_uint), ("inmode", C.c_int),
                ("airflt", C.c_int), ("emptymsg", C.c_int), ("labels", C.c_char_p), ("station_id", C.c_char_p)]


FMT_ONELINE, FMT_FULL, FMT_JSON, FMT_NET_PP, FMT_NET_NATIVE, FMT_NET_JSON = 1, 2, 4, 11, 12, 13


class ChanState(C.Structure):
    _fields_ = [("MskPhi", C.c_double), ("MskDf", C.c_double), ("MskLvlSum", C.c_double), ("MskClk", C.c_float),
                ("MskBitCount", C.c_int), ("MskS", C.c_uint), ("idx", C.c_uint), ("nbits", C.c_int),
                ("Acarsstate", C.c_int), ("outbits", C.c_uint), ("blk_len", C.c_int), ("blk_err", C.c_int),
                ("pos", C.c_uint64), ("soh_pos", C.c_uint64), ("inb_re", C.c_float * 11), ("inb_im", C.c_float * 11),
                ("blk_crc", C.c_ubyte * 2), ("blk_txt", C.c_ubyte * TXTMAX)]

    def vec(self):
        """Same tuple shape as tests/refs.py RefState.vec() / OrcChan.vec()."""
        inb = []
        for i in range(11):
            inb += [self.inb_re[i], self.inb_im[i]]
        return (self.MskPhi, self.MskDf, self.MskLvlSum, self.MskClk, self.MskBitCount, self.MskS, self.idx,
                self.nbits, self.Acarsstate, self.outbits & 0xFF, tuple(inb))


class Stats(C.Structure):
    _fields_ = [("submits", C.c_uint64), ("kernel_launches", C.c_uint64), ("blocks", C.c_uint64),
                ("raw_frames", C.c_uint64), ("fec_dropped", C.c_uint64), ("chan_ms", C.c_double),
                ("demod_ms", C.c_double), ("chan_launches", C.c_uint64), ("demod_launches", C.c_uint64),
                ("fast_chan_launches", C.c_uint64), ("frames_lost", C.c_uint64), ("host_ms", C.c_double)]


# acb_decode_stats_t, field for field (include/acars_b200.h names the reference event each one counts)
DECODE_STATS_FIELDS = ("preamble", "started", "txt_parity", "txt_long", "txt_missed_end", "emitted",
                       "fec_short", "fec_parity_excess", "fec_parity", "fec_crc", "fec_fixed", "fec_unfixable",
                       "fec_parity_problem", "delivered", "lost")
DECODE_STATS_DTYPE = np.dtype([(f, "<u8") for f in DECODE_STATS_FIELDS])

# acb_input_level_t and acb_chan_level_t (include/acars_b200.h defines each field)
INPUT_LEVEL_DTYPE = np.dtype([("samples", "<u8"), ("clipped", "<u8"), ("power_sum", "<f8"), ("peak", "<f4"), ("pad", "<f4")])
CHAN_LEVEL_DTYPE = np.dtype([("rows", "<u8"), ("power_sum", "<f8"), ("peak", "<f4"), ("pad", "<f4"), ("windows", "<u8"),
                             ("floor", "<f8")])
# full-scale amplitude of each input kind's converted components: the mean input power in dBFS is
# 10*log10(power_sum / samples / fs**2)
FULL_SCALE = {"u8": 127.5, "cs16": 32768.0, "real": 1.0}
# acb_chan_freq_t: one chain's half-row rotation sums, its planned RF frequency and its NCO step
CHAN_FREQ_DTYPE = np.dtype([("pairs", "<u8"), ("s_re", "<f8"), ("s_im", "<f8"), ("mag_sum", "<f8"), ("power_sum", "<f8"),
                            ("freq_hz", "<f8"), ("step", "<f8")])


class BlobInfo(C.Structure):
    """acb_streams_blob_info_t: the fingerprint of a stream blob (Context.save_streams)."""
    _fields_ = [("in_kind", C.c_int), ("K", C.c_int), ("taps", C.c_int), ("nch", C.c_int), ("form", C.c_int), ("flags", C.c_int),
                ("group_unit", C.c_int), ("group_period", C.c_uint64), ("count", C.c_int), ("record_bytes", C.c_uint64)]


# every symbol include/acars_b200.h declares: (name, restype, argtypes)
ABI = [
    ("acb_round_freq", C.c_int, [C.c_double]),
    ("acb_stored_fr", C.c_int, [C.c_uint]),
    ("acb_choose_fc", C.c_uint, [C.c_void_p, C.c_int, C.c_int]),
    ("acb_plan_bands", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]),
    ("acb_build_wf", None, [C.c_int, C.c_uint, C.c_int, C.c_void_p]),
    ("acb_air_choose_fc", C.c_uint, [C.c_uint, C.c_uint]),
    ("acb_air_build_wf", None, [C.c_int, C.c_int, C.c_uint, C.c_void_p]),
    ("acb_cs16_build_wf", None, [C.c_int, C.c_uint, C.c_uint, C.c_int, C.c_void_p]),
    ("acb_fast_plan", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_uint, C.c_void_p, C.c_void_p]),
    ("acb_fast_plan_cs16", C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_uint, C.c_void_p, C.c_void_p]),
    ("acb_fast_plan_air", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_uint, C.c_void_p, C.c_void_p]),
    ("acb_build_h", None, [C.c_void_p]),
    ("acb_build_lowpass", C.c_int, [C.c_int, C.c_int, C.c_void_p]),
    ("acb_build_wf_lp", None, [C.c_int, C.c_uint, C.c_int, C.c_int, C.c_void_p]),
    ("acb_cs16_build_wf_lp", None, [C.c_int, C.c_uint, C.c_uint, C.c_int, C.c_int, C.c_void_p]),
    ("acb_air_build_wf_lp", None, [C.c_int, C.c_int, C.c_uint, C.c_int, C.c_void_p]),
    ("acb_create", C.c_int, [C.POINTER(Config), C.POINTER(C.c_void_p)]),
    ("acb_destroy", None, [C.c_void_p]),
    ("acb_last_error", C.c_char_p, []),
    ("acb_version", C.c_char_p, []),
    ("acb_set_plan", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_uint)]),
    ("acb_set_plan_air", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_uint)]),
    ("acb_set_plan_air_at", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_uint]),
    ("acb_set_plan_cs16", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_uint, C.POINTER(C.c_uint)]),
    ("acb_set_plan_at", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_uint]),
    ("acb_set_wf", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int]),
    ("acb_reset", C.c_int, [C.c_void_p]),
    ("acb_reset_stream", C.c_int, [C.c_void_p, C.c_int]),
    ("acb_submit_host_ragged", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("acb_submit_device_ragged", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("acb_submit_real_host_ragged", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("acb_submit_cs16_host_ragged", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("acb_submit_cs16_planar_host_ragged", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("acb_submit_real_device_ragged", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("acb_submit_cs16_device_ragged", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("acb_submit_cs16_planar_device_ragged", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("acb_submit_host", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    ("acb_submit_device", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    ("acb_submit_real_host", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    ("acb_submit_cs16_host", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    ("acb_submit_cs16_planar_host", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    ("acb_submit_real_device", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    ("acb_submit_cs16_device", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    ("acb_submit_cs16_planar_device", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    ("acb_set_emission_groups", C.c_int, [C.c_void_p, C.c_int, C.c_uint64]),
    ("acb_submit_dm_host", C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    ("acb_sync", C.c_int, [C.c_void_p]),
    ("acb_collect", C.c_int, [C.c_void_p]),
    ("acb_wait_event", C.c_int, [C.c_void_p, C.c_void_p]),
    ("acb_multi_create", C.c_int, [C.POINTER(Config), C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    ("acb_multi_destroy", None, [C.c_void_p]),
    ("acb_multi_parts", C.c_int, [C.c_void_p]),
    ("acb_multi_part", C.c_void_p, [C.c_void_p, C.c_int]),
    ("acb_multi_set_plan", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_uint)]),
    ("acb_multi_set_wf", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int]),
    ("acb_multi_reset", C.c_int, [C.c_void_p]),
    ("acb_multi_submit_host", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    ("acb_multi_set_plan_air", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_uint)]),
    ("acb_multi_set_plan_cs16", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_uint, C.POINTER(C.c_uint)]),
    ("acb_multi_submit_real_host", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    ("acb_multi_submit_cs16_host", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    ("acb_multi_submit_cs16_planar_host", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t]),
    ("acb_multi_set_emission_groups", C.c_int, [C.c_void_p, C.c_int, C.c_uint64]),
    ("acb_multi_submit_host_ragged", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("acb_multi_submit_real_host_ragged", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("acb_multi_submit_cs16_host_ragged", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("acb_multi_submit_cs16_planar_host_ragged", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("acb_multi_reset_stream", C.c_int, [C.c_void_p, C.c_int]),
    ("acb_multi_collect", C.c_int, [C.c_void_p]),
    ("acb_multi_sync", C.c_int, [C.c_void_p]),
    ("acb_multi_drain", C.c_int, [C.c_void_p, C.POINTER(Msg), C.c_int]),
    ("acb_multi_get_state", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(ChanState)]),
    ("acb_multi_set_state", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(ChanState)]),
    ("acb_mark", C.c_int, [C.c_void_p, C.c_int]),
    ("acb_elapsed_ms", C.c_int, [C.c_void_p, C.POINTER(C.c_float)]),
    ("acb_msg_fields", C.c_int, [C.POINTER(Msg), C.POINTER(Fields)]),
    ("acb_format_msg", C.c_int, [C.POINTER(Msg), C.c_int, C.POINTER(FmtOpts), C.c_char_p, C.c_size_t]),
    ("acb_flights_new", C.c_void_p, [C.c_int]),
    ("acb_flights_free", None, [C.c_void_p]),
    ("acb_flights_route_json", C.c_int, [C.c_void_p, C.POINTER(Msg), C.POINTER(FmtOpts), C.c_char_p, C.c_size_t]),
    ("acb_flights_monitor", C.c_int, [C.c_void_p, C.POINTER(Msg), C.c_int, C.POINTER(FmtOpts), C.c_char_p, C.c_size_t]),
    ("acb_drain", C.c_int, [C.c_void_p, C.POINTER(Msg), C.c_int]),
    ("acb_pending", C.c_int, [C.c_void_p]),
    ("acb_host_alloc", C.c_void_p, [C.c_size_t]),
    ("acb_host_free", None, [C.c_void_p]),
    ("acb_device_alloc", C.c_void_p, [C.c_void_p, C.c_size_t]),
    ("acb_device_free", None, [C.c_void_p, C.c_void_p]),
    ("acb_copy_to_device", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    ("acb_read_dm", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    ("acb_get_state", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(ChanState)]),
    ("acb_set_state", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(ChanState)]),
    ("acb_get_stats", C.c_int, [C.c_void_p, C.POINTER(Stats), C.c_int]),
    ("acb_get_decode_stats", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    ("acb_multi_get_decode_stats", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    ("acb_get_level_stats", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]),
    ("acb_multi_get_level_stats", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]),
    ("acb_get_freq_stats", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    ("acb_multi_get_freq_stats", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    ("acb_freq_error", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("acb_streams_blob_bytes", C.c_size_t, [C.c_void_p, C.c_int]),
    ("acb_save_streams", C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    ("acb_load_streams", C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    ("acb_streams_blob_check", C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(BlobInfo)]),
    ("acb_multi_streams_blob_bytes", C.c_size_t, [C.c_void_p, C.c_int]),
    ("acb_multi_save_streams", C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    ("acb_multi_load_streams", C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    ("acb_block_fec", C.c_int, [C.POINTER(Msg)]),
    ("acb_block_fec_batch", C.c_int, [C.c_void_p, C.POINTER(Msg), C.c_int, C.POINTER(C.c_int)]),
    ("acb_crc_update", C.c_uint16, [C.c_uint16, C.c_uint8]),
    ("acb_syndrome", C.c_uint16, [C.c_int]),
    ("acb_frame_byte", None, [C.c_void_p, C.c_ubyte]),
]

_lib = None


def load():
    """Load libacars_b200.so (built in-tree by acarsdec_b200.build); raises if it is missing."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise ImportError(f"{LIB_PATH} is missing: run `python -m acarsdec_b200.build` (needs nvcc). "
                              "There is no CPU fallback.")
        lib = C.CDLL(str(LIB_PATH))
        for name, res, args in ABI:
            fn = getattr(lib, name)     # AttributeError if the library does not export it
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


class AcbError(RuntimeError):
    pass


def _check(lib, rc: int) -> int:
    if rc < 0:
        raise AcbError(f"acars_b200 error {rc}: {lib.acb_last_error().decode()}")
    return rc


def freq_error(table: np.ndarray, K: int) -> dict:
    """A freq_stats table (CHAN_FREQ_DTYPE, shape (nstreams, nch)) of a context with this K, through acb_freq_error:
    offset_hz and coherence of shape (nstreams, nch), and each stream's ppm of shape (nstreams,).  A positive offset is
    a carrier above its planned frequency, for every input kind."""
    lib = load()
    t = np.ascontiguousarray(table, dtype=CHAN_FREQ_DTYPE)
    t = t.reshape(1, -1) if t.ndim == 1 else t
    ns, nch = t.shape
    off, coh, ppm = np.zeros((ns, nch)), np.zeros((ns, nch)), np.zeros(ns)
    for s in range(ns):
        _check(lib, lib.acb_freq_error(t[s].ctypes.data, nch, K, off[s].ctypes.data, coh[s].ctypes.data, ppm[s:].ctypes.data))
    return {"offset_hz": off, "coherence": coh, "ppm": ppm}


# ---- front-end planning (host; same results as initRtl) ----

def plan(K: int, freqs_mhz):
    """(freqs_hz, stored Fr, Fc) as initRtl derives them (rtl.c:243-268)."""
    lib = load()
    fd = np.array([lib.acb_round_freq(float(f)) for f in freqs_mhz], dtype=np.uint32)
    fc = lib.acb_choose_fc(fd.ctypes.data, len(fd), K)
    return [int(f) for f in fd], [lib.acb_stored_fr(int(f)) for f in fd], int(fc)


def plan_bands(K: int, freqs_hz, max_groups: int = 64):
    """Fewest receiver bands covering `freqs_hz` (any span): (band index per channel, centre per band)."""
    lib = load()
    f = np.asarray(freqs_hz, dtype=np.uint32)
    grp = np.zeros(len(f), dtype=np.int32)
    fc = np.zeros(max_groups, dtype=np.uint32)
    n = lib.acb_plan_bands(f.ctypes.data, len(f), K, grp.ctypes.data, fc.ctypes.data, max_groups)
    if n < 0:
        raise AcbError(f"acb_plan_bands failed ({n})")
    return grp, fc[:n]


def build_wf(K: int, freqs_mhz) -> np.ndarray:
    lib = load()
    _, fr, fc = plan(K, freqs_mhz)
    out = np.empty((len(fr), 2 * K), dtype=np.float32)
    for i, f in enumerate(fr):
        lib.acb_build_wf(f, fc, K, out[i].ctypes.data)
    return out


def fast_plan(K: int, freqs_hz, fc: int):
    """Planning step of the fast channelizer: (k per channel, twiddles (nch, K/4) complex64), or None when
    some channel is off the 12.5 kHz raster around Fc (the exact kernel runs then)."""
    lib = load()
    f = np.asarray(freqs_hz, dtype=np.uint32)
    k = np.zeros(len(f), dtype=np.int32)
    tw = np.zeros((len(f), K // 4, 2), dtype=np.float32)
    if lib.acb_fast_plan(f.ctypes.data, len(f), K, fc, k.ctypes.data, tw.ctypes.data) != 1:
        return None
    return k, tw[..., 0] + 1j * tw[..., 1]


def blob_info(blob: bytes) -> BlobInfo:
    """acb_streams_blob_check: the fingerprint of a stream blob; AcbError when it is not a valid one (magic, version,
    size, CRC).  Host only."""
    lib = load()
    info = BlobInfo()
    _check(lib, lib.acb_streams_blob_check(blob, len(blob), C.byref(info)))
    return info


def _save_streams(lib, bytes_fn, save_fn, h, streams) -> bytes:
    s = np.ascontiguousarray(streams, dtype=np.int32).reshape(-1)
    n = bytes_fn(h, len(s))
    if n == 0:
        raise AcbError("no stream blob for this context / stream count")
    buf = C.create_string_buffer(n)
    _check(lib, save_fn(h, s.ctypes.data, len(s), buf, n))
    return buf.raw


def _load_streams(lib, load_fn, h, streams, blob: bytes) -> None:
    s = np.ascontiguousarray(streams, dtype=np.int32).reshape(-1)
    _check(lib, load_fn(h, s.ctypes.data, len(s), bytes(blob), len(blob)))


def msg_fields(m: Msg) -> Fields | None:
    f = Fields()
    return f if load().acb_msg_fields(C.byref(m), C.byref(f)) == 1 else None


def format_msg(m: Msg, fmt: int, *, tv_sec: int = 0, tv_usec: int = 0, freq_hz: int = 0, inmode: int = 0, airflt: bool = False,
               emptymsg: bool = False, labels: str | None = None, station_id: str | None = None) -> bytes | None:
    """One decoded block in one of the reference's wire formats (FMT_*), byte for byte; None when a filter drops it."""
    o = FmtOpts(tv_sec, tv_usec, freq_hz, inmode, int(airflt), int(emptymsg),
                labels.encode() if labels else None, station_id.encode() if station_id else None)
    buf = C.create_string_buffer(8192)
    n = load().acb_format_msg(C.byref(m), fmt, C.byref(o), buf, len(buf))
    if n < 0:
        raise AcbError(f"acb_format_msg: error {n} (bad block, unknown format or buffer too small)")
    return buf.raw[:n] if n else None


class Flights:
    """The flight table behind acarsdec's route JSON (-o 5) and monitor screen (-o 3): feed every block in emission order."""

    def __init__(self, mdly_seconds: int = 600):
        self.lib = load()
        self.h = C.c_void_p(self.lib.acb_flights_new(mdly_seconds))
        if not self.h:
            raise AcbError("acb_flights_new failed")

    @staticmethod
    def _opts(kw):
        lab, sta = kw.get("labels"), kw.get("station_id")
        return FmtOpts(kw.get("tv_sec", 0), kw.get("tv_usec", 0), kw.get("freq_hz", 0), kw.get("inmode", 0), int(kw.get("airflt", False)),
                       int(kw.get("emptymsg", False)), lab.encode() if lab else None, sta.encode() if sta else None)

    def _call(self, fn, *args):
        buf = C.create_string_buffer(16384)
        n = fn(*args, buf, len(buf))
        if n < 0:
            raise AcbError(f"flight table: error {n}")
        return buf.raw[:n] if n else None

    def route_json(self, m: Msg, **kw) -> bytes | None:
        o = self._opts(kw)
        return self._call(self.lib.acb_flights_route_json, self.h, C.byref(m), C.byref(o))

    def monitor(self, m: Msg, nbch: int, **kw) -> bytes | None:
        o = self._opts(kw)
        return self._call(self.lib.acb_flights_monitor, self.h, C.byref(m), nbch, C.byref(o))

    def close(self):
        if self.h:
            self.lib.acb_flights_free(self.h)
            self.h = None

    def __del__(self):
        self.close()


def air_plan(rate: int, freqs_mhz):
    """(freqs_hz, Fc, K) as initAirspy derives them (air.c:165-242, no-filter rates)."""
    lib = load()
    fd = [lib.acb_round_freq(float(f)) for f in freqs_mhz]
    return fd, int(lib.acb_air_choose_fc(min(fd), max(fd))), rate // 12500


def build_wf_air(rate: int, freqs_mhz) -> np.ndarray:
    lib = load()
    fd, fc, K = air_plan(rate, freqs_mhz)
    out = np.empty((len(fd), 2 * K), dtype=np.float32)
    for i, f in enumerate(fd):
        lib.acb_air_build_wf(f, fc, rate, out[i].ctypes.data)
    return out


def build_wf_cs16(variant: int, K: int, freqs_hz, fc_hz: int) -> np.ndarray:
    lib = load()
    out = np.empty((len(freqs_hz), 2 * K), dtype=np.float32)
    for i, f in enumerate(freqs_hz):
        lib.acb_cs16_build_wf(variant, int(f), int(fc_hz), K, out[i].ctypes.data)
    return out


def build_h() -> np.ndarray:
    h = np.empty(133, dtype=np.float32)
    load().acb_build_h(h.ctypes.data)
    return h


MAXTAPS_PER_K = 16


def build_lowpass(K: int, taps: int) -> np.ndarray:
    """The channel-filter prototype of an overlapping-window context (taps > K): Kaiser-windowed (beta 6) ideal
    low-pass at 6.25 kHz, sum 1, float32 (acb_build_lowpass)."""
    h = np.empty(taps, dtype=np.float32)
    _check(load(), load().acb_build_lowpass(K, taps, h.ctypes.data))
    return h


def build_wf_lp(K: int, taps: int, freqs_mhz) -> np.ndarray:
    """(nch, 2*taps) tables acb_set_plan builds for a u8 context with taps > K (acb_build_wf_lp)."""
    lib = load()
    _, fr, fc = plan(K, freqs_mhz)
    out = np.empty((len(fr), 2 * taps), dtype=np.float32)
    for i, f in enumerate(fr):
        lib.acb_build_wf_lp(f, fc, K, taps, out[i].ctypes.data)
    return out


def build_wf_cs16_lp(variant: int, K: int, taps: int, freqs_hz, fc_hz: int) -> np.ndarray:
    lib = load()
    out = np.empty((len(freqs_hz), 2 * taps), dtype=np.float32)
    for i, f in enumerate(freqs_hz):
        lib.acb_cs16_build_wf_lp(variant, int(f), int(fc_hz), K, taps, out[i].ctypes.data)
    return out


def build_wf_air_lp(rate: int, taps: int, freqs_mhz) -> np.ndarray:
    lib = load()
    fd, fc, _ = air_plan(rate, freqs_mhz)
    out = np.empty((len(fd), 2 * taps), dtype=np.float32)
    for i, f in enumerate(fd):
        lib.acb_air_build_wf_lp(f, fc, rate, taps, out[i].ctypes.data)
    return out


def block_fec(msg: Msg):
    out = Msg()
    C.memmove(C.byref(out), C.byref(msg), C.sizeof(Msg))
    return out if load().acb_block_fec(C.byref(out)) else None


class PinnedBuffer:
    """uint8 numpy view over cudaHostAlloc memory (acb_host_alloc)."""

    def __init__(self, nbytes: int):
        self.lib = load()
        self.ptr = self.lib.acb_host_alloc(nbytes)
        if not self.ptr:
            raise AcbError(self.lib.acb_last_error().decode())
        self.nbytes = nbytes
        self.array = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(self.ptr))

    def close(self):
        if self.ptr:
            self.lib.acb_host_free(self.ptr)
            self.ptr = None

    def __del__(self):
        self.close()


class Context:
    """N streams x C channels on one GPU (acb_ctx_t)."""

    def __init__(self, K: int, nstreams: int, nch: int, max_blocks: int, device: int = 0, flags: int = 0, taps: int = 0):
        self.lib = load()
        self.K, self.nstreams, self.nch, self.max_blocks = K, nstreams, nch, max_blocks
        self.device = device
        self.block_bytes = OUTBLK * K * 2
        cfg = Config(device, K, nstreams, nch, max_blocks, flags, taps)
        h = C.c_void_p()
        rc = self.lib.acb_create(C.byref(cfg), C.byref(h))
        if rc < 0:
            msg = self.lib.acb_last_error().decode()
            if h:
                self.lib.acb_destroy(h)
            raise AcbError(f"acb_create failed ({rc}): {msg}")
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.lib.acb_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def set_plan(self, stream: int, freqs_hz) -> int:
        f = np.asarray(freqs_hz, dtype=np.uint32)
        fc = C.c_uint()
        _check(self.lib, self.lib.acb_set_plan(self.h, stream, f.ctypes.data, len(f), C.byref(fc)))
        return fc.value

    def set_wf(self, stream: int, wf: np.ndarray) -> None:
        wf = np.ascontiguousarray(wf, dtype=np.float32)
        _check(self.lib, self.lib.acb_set_wf(self.h, stream, wf.ctypes.data, wf.shape[0]))

    def reset(self) -> None:
        _check(self.lib, self.lib.acb_reset(self.h))

    def reset_stream(self, stream: int) -> None:
        """Restart one stream (acb_reset_stream): its chains, carried remainder, history, position and decode counts."""
        _check(self.lib, self.lib.acb_reset_stream(self.h, stream))

    def _counts(self, counts, dtype):
        """A per-stream count array for the ragged calls."""
        c = np.ascontiguousarray(counts, dtype=dtype)
        assert c.shape == (self.nstreams,), f"counts: one entry per stream ({self.nstreams})"
        return c

    def _ragged(self, fn, *args, counts) -> np.ndarray:
        """A ragged streaming call: returns each stream's new envelope rows."""
        c = self._counts(counts, np.uint64)
        nout = np.zeros(self.nstreams, dtype=np.uint64)
        _check(self.lib, fn(self.h, *args, c.ctypes.data, nout.ctypes.data))
        return nout.astype(np.int64)

    def submit_host(self, iq, nblk: int = 0, stream_stride: int | None = None, counts=None) -> None:
        """iq: uint8 array (nstreams, nblk*block_bytes) or a raw pointer + stride.  counts: blocks per stream (the
        ragged call; nblk is then ignored and the array's row pitch is the default stride)."""
        if counts is not None:
            c = self._counts(counts, np.int32)
            nblk = int(c.max())
        if isinstance(iq, np.ndarray):
            assert iq.dtype == np.uint8 and iq.flags.c_contiguous
            ptr = iq.ctypes.data
            if stream_stride is None:
                stream_stride = iq.strides[0] if iq.ndim == 2 else nblk * self.block_bytes
        else:
            ptr = iq
        if counts is not None:
            _check(self.lib, self.lib.acb_submit_host_ragged(self.h, ptr, stream_stride, c.ctypes.data))
        else:
            _check(self.lib, self.lib.acb_submit_host(self.h, ptr, stream_stride, nblk))

    def submit_device(self, dev_ptr: int, nblk: int, stream_stride: int, counts=None) -> None:
        """counts: blocks per stream (the ragged call; nblk is then ignored)."""
        if counts is not None:
            c = self._counts(counts, np.int32)
            _check(self.lib, self.lib.acb_submit_device_ragged(self.h, dev_ptr, stream_stride, c.ctypes.data))
        else:
            _check(self.lib, self.lib.acb_submit_device(self.h, dev_ptr, stream_stride, nblk))

    def set_plan_air(self, stream: int, freqs_hz) -> int:
        f = np.asarray(freqs_hz, dtype=np.uint32)
        fc = C.c_uint()
        _check(self.lib, self.lib.acb_set_plan_air(self.h, stream, f.ctypes.data, len(f), C.byref(fc)))
        return fc.value

    def set_plan_air_at(self, stream: int, freqs_hz, fc_hz: int) -> None:
        """set_plan_air around a given tuner centre (a context serving some of a receiver's channels)."""
        f = np.asarray(freqs_hz, dtype=np.uint32)
        _check(self.lib, self.lib.acb_set_plan_air_at(self.h, stream, f.ctypes.data, len(f), int(fc_hz)))

    @staticmethod
    def _stream_stride(a: np.ndarray, sample_bytes: int, stream_stride: int | None) -> int:
        """Stream stride in samples: the array's row pitch (a view into wider rows keeps its pitch), which an explicit
        `stream_stride` must agree with when there is more than one stream."""
        # numpy may give a length-1 axis any stride: only the strides of axes longer than 1 say where the data is
        assert a.shape[1] <= 1 or a.strides[1] == sample_bytes
        assert a.shape[0] <= 1 or a.strides[0] % sample_bytes == 0
        pitch = a.strides[0] // sample_bytes if a.shape[0] > 1 else a.shape[1]
        if stream_stride is None:
            return pitch
        assert stream_stride >= a.shape[1] and (a.shape[0] == 1 or stream_stride == pitch)
        return stream_stride

    def submit_real(self, x: np.ndarray, stream_stride: int | None = None, counts=None):
        """x: float32 (nstreams, nsamples) real samples, rows contiguous; stream s starts stream_stride samples after
        stream s-1 (default: the array's row pitch).  Returns envelope samples produced per channel.  counts: samples
        per stream (the ragged call, each <= the row length); returns each stream's new rows."""
        assert x.dtype == np.float32 and x.ndim == 2 and x.shape[0] == self.nstreams
        stride = self._stream_stride(x, 4, stream_stride)
        if counts is not None:
            return self._ragged(self.lib.acb_submit_real_host_ragged, x.ctypes.data, stride, counts=counts)
        return _check(self.lib, self.lib.acb_submit_real_host(self.h, x.ctypes.data, stride, x.shape[1]))

    def set_plan_cs16(self, stream: int, freqs_hz, variant: int, fc_hz: int = 0) -> int:
        f = np.asarray(freqs_hz, dtype=np.uint32)
        fc = C.c_uint()
        _check(self.lib, self.lib.acb_set_plan_cs16(self.h, stream, f.ctypes.data, len(f), variant, fc_hz, C.byref(fc)))
        return fc.value

    def submit_cs16(self, iq: np.ndarray, stream_stride: int | None = None, counts=None):
        """iq: int16 (nstreams, nsamples, 2) interleaved I,Q, rows contiguous; stream_stride in complex samples
        (default: the array's row pitch).  counts: as submit_real's."""
        assert iq.dtype == np.int16 and iq.ndim == 3 and iq.shape[0] == self.nstreams and iq.shape[2] == 2 and iq.strides[2] == 2
        stride = self._stream_stride(iq, 4, stream_stride)
        if counts is not None:
            return self._ragged(self.lib.acb_submit_cs16_host_ragged, iq.ctypes.data, stride, counts=counts)
        return _check(self.lib, self.lib.acb_submit_cs16_host(self.h, iq.ctypes.data, stride, iq.shape[1]))

    def submit_cs16_planar(self, xi: np.ndarray, xq: np.ndarray, stream_stride: int | None = None, counts=None):
        """xi, xq: int16 (nstreams, nsamples) separate I and Q planes (the SDRplay callback's layout), rows contiguous and
        both planes with the same stream_stride (default: their row pitch).  counts: as submit_real's."""
        assert xi.dtype == np.int16 and xq.dtype == np.int16 and xi.shape == xq.shape and xi.shape[0] == self.nstreams
        stride = self._stream_stride(xi, 2, stream_stride)
        assert self._stream_stride(xq, 2, stream_stride) == stride
        if counts is not None:
            return self._ragged(self.lib.acb_submit_cs16_planar_host_ragged, xi.ctypes.data, xq.ctypes.data, stride, counts=counts)
        return _check(self.lib, self.lib.acb_submit_cs16_planar_host(self.h, xi.ctypes.data, xq.ctypes.data, stride, xi.shape[1]))

    # the streaming submits with the input in device memory: pointers, `nsamples` and the stream stride in samples, as the
    # C calls take them; each returns the envelope samples produced per channel, or with `counts` (samples per stream,
    # nsamples ignored) each stream's new rows
    def submit_real_device(self, x_dev: int, nsamples: int, stream_stride: int, counts=None):
        if counts is not None:
            return self._ragged(self.lib.acb_submit_real_device_ragged, x_dev, stream_stride, counts=counts)
        return _check(self.lib, self.lib.acb_submit_real_device(self.h, x_dev, stream_stride, nsamples))

    def submit_cs16_device(self, iq_dev: int, nsamples: int, stream_stride: int, counts=None):
        if counts is not None:
            return self._ragged(self.lib.acb_submit_cs16_device_ragged, iq_dev, stream_stride, counts=counts)
        return _check(self.lib, self.lib.acb_submit_cs16_device(self.h, iq_dev, stream_stride, nsamples))

    def submit_cs16_planar_device(self, xi_dev: int, xq_dev: int, nsamples: int, stream_stride: int, counts=None):
        if counts is not None:
            return self._ragged(self.lib.acb_submit_cs16_planar_device_ragged, xi_dev, xq_dev, stream_stride, counts=counts)
        return _check(self.lib, self.lib.acb_submit_cs16_planar_device(self.h, xi_dev, xq_dev, stream_stride, nsamples))

    def submit_tensor(self, x, xq=None, counts=None):
        """The device submits from torch CUDA tensors: float32 (nstreams, n) for a real-input context, int16
        (nstreams, n, 2) interleaved or two int16 (nstreams, n) planes (x = I, xq = Q) for a CS16 context.  Rows may be
        views into wider rows (their pitch is the stream stride); samples within a row are contiguous."""
        import torch
        for t in (x,) if xq is None else (x, xq):
            if not (isinstance(t, torch.Tensor) and t.is_cuda and t.device.index == self.device):
                raise TypeError(f"torch tensors on cuda:{self.device} expected; host arrays go to submit_real / submit_cs16")
        if xq is not None:
            ok = x.dtype == xq.dtype == torch.int16 and x.dim() == 2 and x.shape == xq.shape and x.stride() == xq.stride()
            layout = "two int16 (nstreams, n) planes of one shape and stride"
        elif x.dtype == torch.float32:
            ok, layout = x.dim() == 2, "float32 (nstreams, n)"
        else:
            ok = x.dtype == torch.int16 and x.dim() == 3 and x.shape[2] == 2 and x.stride(2) == 1
            layout = "float32 (nstreams, n) or int16 (nstreams, n, 2)"
        per = 2 if x.dim() == 3 else 1                       # tensor elements per sample: CS16 interleaved carries I and Q
        n = x.shape[1]
        ok = ok and x.shape[0] == self.nstreams and (n <= 1 or x.stride(1) == per) and x.stride(0) % per == 0
        if not ok:
            raise ValueError(f"expected {layout}, {self.nstreams} streams, samples contiguous within a row")
        stride = x.stride(0) // per if x.shape[0] > 1 else n
        if counts is not None:           # the ragged calls: samples per stream, each <= n
            assert int(np.max(counts)) <= n
        if xq is not None:
            return self.submit_cs16_planar_device(x.data_ptr(), xq.data_ptr(), n, stride, counts=counts)
        if x.dtype == torch.float32:
            return self.submit_real_device(x.data_ptr(), n, stride, counts=counts)
        return self.submit_cs16_device(x.data_ptr(), n, stride, counts=counts)

    def set_emission_groups(self, unit: int, period: int = 0) -> None:
        """unit: 0 per submit, 1 every `period` envelope samples, 2 per transfer of `period` input samples."""
        _check(self.lib, self.lib.acb_set_emission_groups(self.h, unit, period))

    def submit_dm(self, dm: np.ndarray) -> None:
        """dm: float32 (nstreams, nsamp, nch)."""
        dm = np.ascontiguousarray(dm, dtype=np.float32)
        assert dm.shape[0] == self.nstreams and dm.shape[2] == self.nch
        _check(self.lib, self.lib.acb_submit_dm_host(self.h, dm.ctypes.data, dm.shape[1]))

    def sync(self) -> int:
        return _check(self.lib, self.lib.acb_sync(self.h))

    def collect(self) -> int:
        return _check(self.lib, self.lib.acb_collect(self.h))

    def mark(self, which: int) -> None:
        _check(self.lib, self.lib.acb_mark(self.h, which))

    def elapsed_ms(self) -> float:
        ms = C.c_float()
        _check(self.lib, self.lib.acb_elapsed_ms(self.h, C.byref(ms)))
        return ms.value

    def drain(self):
        out = []
        buf = (Msg * 256)()
        while True:
            n = self.lib.acb_drain(self.h, buf, 256)
            for i in range(n):
                m = Msg()
                C.memmove(C.byref(m), C.byref(buf[i]), C.sizeof(Msg))
                out.append(m)
            if n < 256:
                return out

    def pending(self) -> int:
        return self.lib.acb_pending(self.h)

    def drain_records(self) -> np.ndarray:
        """All queued messages as one numpy record array (MSG_DTYPE), one C call."""
        n = self.lib.acb_pending(self.h)
        buf = np.empty(n, dtype=MSG_DTYPE)
        if n:
            got = self.lib.acb_drain(self.h, buf.ctypes.data_as(C.POINTER(Msg)), n)
            buf = buf[:got]
        return buf

    def block_fec_batch(self, msgs):
        """Device block FEC over a list of raw Msg (parity-bearing txt): returns [fixed Msg or None]."""
        n = len(msgs)
        arr = (Msg * n)()
        for i, m in enumerate(msgs):
            C.memmove(C.byref(arr[i]), C.byref(m), C.sizeof(Msg))
        keep = (C.c_int * n)()
        _check(self.lib, self.lib.acb_block_fec_batch(self.h, arr, n, keep))
        out = []
        for i in range(n):
            if keep[i]:
                m = Msg()
                C.memmove(C.byref(m), C.byref(arr[i]), C.sizeof(Msg))
                out.append(m)
            else:
                out.append(None)
        return out

    def read_dm(self, nsamp: int) -> np.ndarray:
        out = np.empty((self.nstreams, nsamp, self.nch), dtype=np.float32)
        _check(self.lib, self.lib.acb_read_dm(self.h, out.ctypes.data, out.size))
        return out

    def get_state(self, stream: int, chn: int) -> ChanState:
        s = ChanState()
        _check(self.lib, self.lib.acb_get_state(self.h, stream, chn, C.byref(s)))
        return s

    def set_state(self, stream: int, chn: int, s: ChanState) -> None:
        _check(self.lib, self.lib.acb_set_state(self.h, stream, chn, C.byref(s)))

    def stats(self, reset: bool = False) -> Stats:
        s = Stats()
        _check(self.lib, self.lib.acb_get_stats(self.h, C.byref(s), int(reset)))
        return s

    def decode_stats(self, reset: bool = False) -> np.ndarray:
        """Per-chain decode statistics (FLAG_DECODE_STATS): a DECODE_STATS_DTYPE array of shape (nstreams, nch)."""
        out = np.zeros((self.nstreams, self.nch), dtype=DECODE_STATS_DTYPE)
        _check(self.lib, self.lib.acb_get_decode_stats(self.h, out.ctypes.data, out.size, int(reset)))
        return out

    def level_stats(self, reset: bool = False) -> tuple[np.ndarray, np.ndarray]:
        """Input and envelope levels (FLAG_LEVEL_STATS): an INPUT_LEVEL_DTYPE array of shape (nstreams,) and a
        CHAN_LEVEL_DTYPE array of shape (nstreams, nch)."""
        inp = np.zeros(self.nstreams, dtype=INPUT_LEVEL_DTYPE)
        ch = np.zeros((self.nstreams, self.nch), dtype=CHAN_LEVEL_DTYPE)
        _check(self.lib, self.lib.acb_get_level_stats(self.h, inp.ctypes.data, inp.size, ch.ctypes.data, ch.size, int(reset)))
        return inp, ch

    def freq_stats(self, reset: bool = False) -> np.ndarray:
        """Per-chain carrier rotation sums (FLAG_FREQ_STATS): a CHAN_FREQ_DTYPE array of shape (nstreams, nch); freq_error
        turns it into offsets and ppm."""
        out = np.zeros((self.nstreams, self.nch), dtype=CHAN_FREQ_DTYPE)
        _check(self.lib, self.lib.acb_get_freq_stats(self.h, out.ctypes.data, out.size, int(reset)))
        return out

    def device_alloc(self, nbytes: int) -> int:
        p = self.lib.acb_device_alloc(self.h, nbytes)
        if not p:
            raise AcbError(self.lib.acb_last_error().decode())
        return p

    def device_free(self, p: int) -> None:
        self.lib.acb_device_free(self.h, p)

    def copy_to_device(self, dst: int, src: np.ndarray) -> None:
        src = np.ascontiguousarray(src)
        _check(self.lib, self.lib.acb_copy_to_device(self.h, dst, src.ctypes.data, src.nbytes))

    def set_plan_at(self, stream: int, freqs_hz, fc_hz: int) -> None:
        f = np.asarray(freqs_hz, dtype=np.uint32)
        _check(self.lib, self.lib.acb_set_plan_at(self.h, stream, f.ctypes.data, len(f), int(fc_hz)))

    def wait_event(self, cuda_event: int) -> None:
        """Order the next submit_device (and the next streaming device submit's read of its input) behind a cudaEvent_t of
        another stream (torch.cuda.Event.cuda_event)."""
        _check(self.lib, self.lib.acb_wait_event(self.h, cuda_event))

    def save_streams(self, streams) -> bytes:
        """acb_save_streams: the whole decoding state of these streams (record i = streams[i]) after every submit made so
        far; the submits in flight are collected first, the context is otherwise unchanged."""
        return _save_streams(self.lib, self.lib.acb_streams_blob_bytes, self.lib.acb_save_streams, self.h, streams)

    def load_streams(self, streams, blob: bytes) -> None:
        """acb_load_streams: record i of blob into stream streams[i], queued behind the work in flight."""
        _load_streams(self.lib, self.lib.acb_load_streams, self.h, streams, blob)


class MultiContext:
    """acb_multi_t: one process, several GPUs; streams (mode 0) or channels (mode 1) split among them."""

    def __init__(self, K: int, nstreams: int, nch: int, max_blocks: int, devices, mode: int = 0, flags: int = 0, taps: int = 0):
        self.lib = load()
        self.K, self.nstreams, self.nch = K, nstreams, nch
        cfg = Config(0, K, nstreams, nch, max_blocks, flags, taps)
        dev = np.asarray(list(devices), dtype=np.int32)
        h = C.c_void_p()
        rc = self.lib.acb_multi_create(C.byref(cfg), dev.ctypes.data, len(dev), mode, C.byref(h))
        if rc < 0:
            msg = self.lib.acb_last_error().decode()
            if h:
                self.lib.acb_multi_destroy(h)
            raise AcbError(f"acb_multi_create failed ({rc}): {msg}")
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.lib.acb_multi_destroy(self.h)
            self.h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def parts(self) -> int:
        return self.lib.acb_multi_parts(self.h)

    def set_plan(self, stream: int, freqs_hz) -> int:
        f = np.asarray(freqs_hz, dtype=np.uint32)
        fc = C.c_uint()
        _check(self.lib, self.lib.acb_multi_set_plan(self.h, stream, f.ctypes.data, len(f), C.byref(fc)))
        return fc.value

    def set_wf(self, stream: int, wf: np.ndarray) -> None:
        wf = np.ascontiguousarray(wf, dtype=np.float32)
        _check(self.lib, self.lib.acb_multi_set_wf(self.h, stream, wf.ctypes.data, wf.shape[0]))

    def submit_host(self, iq: np.ndarray, nblk: int = 0, counts=None) -> None:
        """counts: blocks per stream (the ragged call; nblk is then ignored)."""
        assert iq.dtype == np.uint8 and iq.flags.c_contiguous
        if counts is not None:
            c = np.ascontiguousarray(counts, dtype=np.int32)
            assert c.shape == (self.nstreams,)
            nblk = int(c.max())
        stride = iq.strides[0] if iq.ndim == 2 else nblk * OUTBLK * self.K * 2
        if counts is not None:
            _check(self.lib, self.lib.acb_multi_submit_host_ragged(self.h, iq.ctypes.data, stride, c.ctypes.data))
        else:
            _check(self.lib, self.lib.acb_multi_submit_host(self.h, iq.ctypes.data, stride, nblk))

    def reset_stream(self, stream: int) -> None:
        """acb_multi_reset_stream: collects the submits in flight, then restarts one stream on the parts serving it."""
        _check(self.lib, self.lib.acb_multi_reset_stream(self.h, stream))

    def _ragged(self, fn, *args, counts) -> np.ndarray:
        c = np.ascontiguousarray(counts, dtype=np.uint64)
        assert c.shape == (self.nstreams,), f"counts: one entry per stream ({self.nstreams})"
        nout = np.zeros(self.nstreams, dtype=np.uint64)
        _check(self.lib, fn(self.h, *args, c.ctypes.data, nout.ctypes.data))
        return nout.astype(np.int64)

    def set_plan_air(self, stream: int, freqs_hz) -> int:
        """Real input: Fc chosen once over all channels (acb_air_choose_fc), every part planned around it."""
        f = np.asarray(freqs_hz, dtype=np.uint32)
        fc = C.c_uint()
        _check(self.lib, self.lib.acb_multi_set_plan_air(self.h, stream, f.ctypes.data, len(f), C.byref(fc)))
        return fc.value

    def set_plan_cs16(self, stream: int, freqs_hz, variant: int, fc_hz: int = 0) -> int:
        f = np.asarray(freqs_hz, dtype=np.uint32)
        fc = C.c_uint()
        _check(self.lib, self.lib.acb_multi_set_plan_cs16(self.h, stream, f.ctypes.data, len(f), variant, fc_hz, C.byref(fc)))
        return fc.value

    # the streaming submits take what Context's take, with the same stride rules (counts: the ragged calls, as Context's)
    def submit_real(self, x: np.ndarray, stream_stride: int | None = None, counts=None):
        assert x.dtype == np.float32 and x.ndim == 2 and x.shape[0] == self.nstreams
        stride = Context._stream_stride(x, 4, stream_stride)
        if counts is not None:
            return self._ragged(self.lib.acb_multi_submit_real_host_ragged, x.ctypes.data, stride, counts=counts)
        return _check(self.lib, self.lib.acb_multi_submit_real_host(self.h, x.ctypes.data, stride, x.shape[1]))

    def submit_cs16(self, iq: np.ndarray, stream_stride: int | None = None, counts=None):
        assert iq.dtype == np.int16 and iq.ndim == 3 and iq.shape[0] == self.nstreams and iq.shape[2] == 2 and iq.strides[2] == 2
        stride = Context._stream_stride(iq, 4, stream_stride)
        if counts is not None:
            return self._ragged(self.lib.acb_multi_submit_cs16_host_ragged, iq.ctypes.data, stride, counts=counts)
        return _check(self.lib, self.lib.acb_multi_submit_cs16_host(self.h, iq.ctypes.data, stride, iq.shape[1]))

    def submit_cs16_planar(self, xi: np.ndarray, xq: np.ndarray, stream_stride: int | None = None, counts=None):
        assert xi.dtype == np.int16 and xq.dtype == np.int16 and xi.shape == xq.shape and xi.shape[0] == self.nstreams
        stride = Context._stream_stride(xi, 2, stream_stride)
        assert Context._stream_stride(xq, 2, stream_stride) == stride
        if counts is not None:
            return self._ragged(self.lib.acb_multi_submit_cs16_planar_host_ragged, xi.ctypes.data, xq.ctypes.data, stride, counts=counts)
        return _check(self.lib, self.lib.acb_multi_submit_cs16_planar_host(self.h, xi.ctypes.data, xq.ctypes.data, stride, xi.shape[1]))

    def set_emission_groups(self, unit: int, period: int = 0) -> None:
        """As Context.set_emission_groups; the merged order follows these groups."""
        _check(self.lib, self.lib.acb_multi_set_emission_groups(self.h, unit, period))

    def reset(self) -> None:
        _check(self.lib, self.lib.acb_multi_reset(self.h))

    def part_stats(self, i: int, reset: bool = False) -> Stats:
        """acb_get_stats of the i-th per-device context."""
        s = Stats()
        _check(self.lib, self.lib.acb_get_stats(self.lib.acb_multi_part(self.h, i), C.byref(s), int(reset)))
        return s

    def decode_stats(self, reset: bool = False) -> np.ndarray:
        """As Context.decode_stats, indexed by global stream and channel."""
        out = np.zeros((self.nstreams, self.nch), dtype=DECODE_STATS_DTYPE)
        _check(self.lib, self.lib.acb_multi_get_decode_stats(self.h, out.ctypes.data, out.size, int(reset)))
        return out

    def level_stats(self, reset: bool = False) -> tuple[np.ndarray, np.ndarray]:
        """As Context.level_stats, indexed by global stream and channel (a channel split's input levels are part 0's)."""
        inp = np.zeros(self.nstreams, dtype=INPUT_LEVEL_DTYPE)
        ch = np.zeros((self.nstreams, self.nch), dtype=CHAN_LEVEL_DTYPE)
        _check(self.lib, self.lib.acb_multi_get_level_stats(self.h, inp.ctypes.data, inp.size, ch.ctypes.data, ch.size, int(reset)))
        return inp, ch

    def freq_stats(self, reset: bool = False) -> np.ndarray:
        """As Context.freq_stats, indexed by global stream and channel."""
        out = np.zeros((self.nstreams, self.nch), dtype=CHAN_FREQ_DTYPE)
        _check(self.lib, self.lib.acb_multi_get_freq_stats(self.h, out.ctypes.data, out.size, int(reset)))
        return out

    def part_input_levels(self, i: int) -> np.ndarray:
        """The input table of the i-th per-device context: its streams first (in a channel split, every stream)."""
        inp = np.zeros(self.nstreams, dtype=INPUT_LEVEL_DTYPE)
        _check(self.lib, self.lib.acb_get_level_stats(self.lib.acb_multi_part(self.h, i), inp.ctypes.data, inp.size, None, 0, 0))
        return inp

    def sync(self) -> int:
        return _check(self.lib, self.lib.acb_multi_sync(self.h))

    def collect(self) -> int:
        return _check(self.lib, self.lib.acb_multi_collect(self.h))

    def drain(self):
        out = []
        buf = (Msg * 256)()
        while True:
            n = self.lib.acb_multi_drain(self.h, buf, 256)
            for i in range(n):
                m = Msg()
                C.memmove(C.byref(m), C.byref(buf[i]), C.sizeof(Msg))
                out.append(m)
            if n < 256:
                return out

    def get_state(self, stream: int, chn: int) -> ChanState:
        s = ChanState()
        _check(self.lib, self.lib.acb_multi_get_state(self.h, stream, chn, C.byref(s)))
        return s

    def save_streams(self, streams) -> bytes:
        """acb_multi_save_streams (stream split): the blob a single context would give."""
        return _save_streams(self.lib, self.lib.acb_multi_streams_blob_bytes, self.lib.acb_multi_save_streams, self.h, streams)

    def load_streams(self, streams, blob: bytes) -> None:
        """acb_multi_load_streams (stream split): collects the submits in flight, then loads each record on its part."""
        _load_streams(self.lib, self.lib.acb_multi_load_streams, self.h, streams, blob)
