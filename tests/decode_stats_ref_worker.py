"""Runs the reference with -v in a process of its own (its state is process-global and its lines go to stderr):

    python decode_stats_ref_worker.py audio ENVELOPE.npy CHUNK    decodeAcars + blk_thread on an (nch, nsamp) envelope,
                                                                   fed like soundfile.c (chunks, channel by channel)
    python decode_stats_ref_worker.py blocks FRAMES.npz           blk_thread alone on pre-FEC blocks, block i as chn i

stdout: one JSON object, the messages outputmsg() received per channel; stderr: the reference's -v lines.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
import refs  # noqa: E402


def main() -> None:
    ref = refs.RefLib("verbose")
    ref.lib.ref_set_verbose.argtypes = [C.c_int]
    mode = sys.argv[1]
    if mode == "audio":
        dm = np.load(sys.argv[2])
        chunk = int(sys.argv[3])
        ref.open_audio(dm.shape[0])
        ref.lib.ref_set_verbose(1)
        for p in range(0, dm.shape[1], chunk):
            for c in range(dm.shape[0]):
                seg = np.ascontiguousarray(dm[c, p:p + chunk], dtype=np.float32)
                ref.lib.ref_audio_chunk(c, seg.ctypes.data, len(seg))
    else:
        z = np.load(sys.argv[2])
        ref.open_audio(1)                   # initAcars of channel 0 starts blk_thread (acars.c:220-228)
        ref.lib.ref_set_verbose(1)
        for i, (n, txt, crc) in enumerate(zip(z["len"], z["txt"], z["crc"])):
            ref.push_block(i, bytes(txt[:n]), bytes(crc))
    msgs = ref.msgs()                       # flushes: every queued block went through blk_thread
    per = {}
    for m in msgs:
        per[m.chn] = per.get(m.chn, 0) + 1
    sys.stderr.flush()
    sys.stdout.write(json.dumps({str(k): v for k, v in per.items()}))
    sys.stdout.flush()
    os._exit(0)                             # blk_thread is still waiting on its queue


if __name__ == "__main__":
    main()
