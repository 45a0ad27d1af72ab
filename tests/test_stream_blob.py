"""Stream blobs (acb_save_streams / acb_load_streams) on the host: acb_streams_blob_check on blobs written here by the
documented layout (include/acars_b200.h, DESIGN.md §4 "Moving streams"), its refusals, and the ctypes fingerprint
struct against the C struct through a compiled C probe.  No device."""
import ctypes as C
import shutil
import struct
import subprocess
import zlib
from pathlib import Path

import numpy as np
import pytest

from acarsdec_b200 import api

ROOT = Path(__file__).resolve().parents[1]
ERR_ARG = -1
MAGIC, VERSION = b"ACBSTRM\0", 1
U8, REAL, CS16 = 0, 1, 2
EXACT, GENERIC, DFT, RDFT, OVL_FAST, OVL_RDFT, WB, WB_REAL = range(8)
DECODE, LEVEL = 256, 512


def r16(x):
    return (x + 15) // 16 * 16


def record_bytes(kind, K, taps, nch, form, flags):
    """The record size, restated from the layout: host part, device regions at 16-byte offsets, then the statistics"""
    unit = 8 if kind == U8 else 4
    if taps > K:
        hpad = -(-(taps - K) // unit) * unit
        taps_pad = K + hpad
    else:
        hpad = 0
        taps_pad = taps if form == GENERIC else min(K, -(-taps // unit) * unit)
    ngrp, nct = -(-nch // 8), -(-nch // 256)
    regions = [nch * 432]                                   # chain states (sizeof ChainState)
    if kind != U8:
        regions.append(r16((hpad + K) * 4))                  # history + carry
    elif hpad:
        regions.append(hpad * 2)                             # u8 history
    regions.append(ngrp * taps_pad * 8 * 2 * 4)              # exact tables
    if form in (DFT, RDFT, OVL_FAST, OVL_RDFT):
        regions += [ngrp * 8 * (K // 4) * 2 * 4, ngrp * 4]   # twiddles, residues
    if form in (WB, WB_REAL):
        regions.append(nct * (2 + 2 * (256 + 12 + 4)) * 4)   # wideband plan
    if flags & LEVEL:
        regions.append(nch * 16)                             # open windows
    off = 32 + sum(r16(r) for r in regions)
    if flags & DECODE:
        off += nch * 120
    if flags & LEVEL:
        off += 32 + nch * 40
    return r16(off)


def make_blob(kind=U8, K=160, taps=160, nch=4, form=EXACT, flags=0, unit=0, period=0, count=2, seed=0, version=VERSION,
              magic=MAGIC, rec=None):
    rec = record_bytes(kind, K, taps, nch, form, flags) if rec is None else rec
    payload = np.random.default_rng(seed).integers(0, 256, size=count * rec, dtype=np.uint8).tobytes()
    body = struct.pack("<8iQQ", kind, K, taps, nch, form, flags, unit, count, period, rec) + payload
    return magic + struct.pack("<II", version, zlib.crc32(body)) + body


def check(blob, n=None):
    lib = api.load()
    info = api.BlobInfo()
    return lib.acb_streams_blob_check(blob, len(blob) if n is None else n, C.byref(info)), info


CONFIGS = [
    (U8, 160, 160, 4, EXACT, 0), (U8, 164, 2 * 164 + 40, 4, GENERIC, DECODE), (U8, 160, 2 * 160 + 48, 8, OVL_FAST, LEVEL),
    (U8, 160, 160, 8, DFT, DECODE | LEVEL), (CS16, 160, 2 * 160 + 48, 4, WB, 0), (CS16, 160, 160, 300, WB, LEVEL),
    (REAL, 200, 200, 4, RDFT, 0), (REAL, 200, 2 * 200 + 40, 4, OVL_RDFT, DECODE), (REAL, 200, 200, 9, WB_REAL, LEVEL),
    (REAL, 200, 2 * 200 + 40, 4, EXACT, 0),
]


@pytest.mark.parametrize("cfg", CONFIGS)
def test_valid_blob_is_accepted_with_its_fingerprint(cfg):
    kind, K, taps, nch, form, flags = cfg
    unit, period = (2, 4096) if kind != U8 else (0, 0)
    blob = make_blob(kind, K, taps, nch, form, flags, unit, period, count=3)
    rc, info = check(blob)
    assert rc == 0, api.load().acb_last_error().decode()
    assert (info.in_kind, info.K, info.taps, info.nch, info.form, info.flags) == cfg
    assert (info.group_unit, info.group_period, info.count) == (unit, period, 3)
    assert info.record_bytes == record_bytes(*cfg)
    assert api.blob_info(blob).count == 3


def test_refusals():
    blob = make_blob(count=2)
    assert check(blob)[0] == 0
    for i in (16, 64, 64 + 100, len(blob) - 1):                  # a flipped byte anywhere the CRC covers
        bad = bytearray(blob)
        bad[i] ^= 0x01
        assert check(bytes(bad))[0] == ERR_ARG, i
    assert check(blob[:-1])[0] == ERR_ARG                        # truncated
    assert check(blob[:-record_bytes(U8, 160, 160, 4, EXACT, 0)])[0] == ERR_ARG   # a whole record short
    assert check(blob[:40])[0] == ERR_ARG                        # shorter than the header
    assert check(blob + b"\0" * 16)[0] == ERR_ARG                # trailing bytes
    assert check(make_blob(magic=b"ACBSTRX\0"))[0] == ERR_ARG
    assert check(make_blob(version=VERSION + 1))[0] == ERR_ARG
    assert check(make_blob(rec=record_bytes(U8, 160, 160, 4, EXACT, 0) + 16))[0] == ERR_ARG   # not this layout's size
    assert check(make_blob(flags=1))[0] == ERR_ARG               # a flag the blob never carries
    assert check(make_blob(count=0))[0] == ERR_ARG
    with pytest.raises(api.AcbError):
        api.blob_info(blob[:-1])


PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "acars_b200.h"
#define F(f) printf(#f " %zu %zu\n", offsetof(acb_streams_blob_info_t, f), sizeof(((acb_streams_blob_info_t *)0)->f))
int main(void)
{
	printf("size %zu\n", sizeof(acb_streams_blob_info_t));
	F(in_kind); F(K); F(taps); F(nch); F(form); F(flags); F(group_unit); F(group_period); F(count); F(record_bytes);
	return 0;
}
"""


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no C compiler")
def test_info_struct_matches_the_c_struct(tmp_path):
    src = tmp_path / "probe.c"
    src.write_text(PROBE)
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-std=c11", "-I", str(ROOT / "include"), "-o", str(exe), str(src)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    fields = {name: (getattr(api.BlobInfo, name).offset, getattr(api.BlobInfo, name).size) for name, _ in api.BlobInfo._fields_}
    seen = set()
    for line in filter(None, out):
        w = line.split()
        if w[0] == "size":
            assert int(w[1]) == C.sizeof(api.BlobInfo)
        else:
            assert fields[w[0]] == (int(w[1]), int(w[2])), line
            seen.add(w[0])
    assert seen == set(fields)
