"""The one-sample definition of message positions and framing exits (tests/frame_pos_refs.py) held to itself and to the
host build of the device's demodulator loop (tests/host/demod_emul.cpp), and the fixture's proof of coverage.  The GPU
side of the same definition is tests/test_gpu_frame_sync.py."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import frame_pos_refs as F
from test_demod_core import EmulFrame, emul, fresh_state  # noqa: F401  (emul is a fixture)


def test_fixture_reaches_every_exit(oracle):
    """Every exit kind at least twice, on at least two channels; blocks of 13, 240 and 241 bytes and frames under 13
    bytes reach the sink; at least one frame is dropped by the FEC and most are delivered."""
    trs = F.traces()
    cov = F.coverage(trs)
    for k in F.EXITS:
        n, chans = cov.get(k, (0, set()))
        assert n >= 2 and len(chans) >= 2, (k, n, chans)
    lens = [f.msg.len for tr in trs for f in tr.frames]
    assert {13, 240, 241} <= set(lens) and min(lens) < 13
    kept = [oracle.fec(f.msg) is not None for tr in trs for f in tr.frames]
    assert 0 < kept.count(False) < kept.count(True)
    for tr in trs:          # positions increase along a channel; an SOH precedes its frame
        pos = [f.pos for f in tr.frames]
        assert pos == sorted(pos) and len(set(pos)) == len(pos)
        assert all(0 < f.pos - f.soh_pos < 8 * 6 * 256 for f in tr.frames)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_positions_do_not_depend_on_chunking(oracle, seed):
    """The same channels in ragged orc_demod calls (1 to 3000 samples, and a few single samples): every call emits
    exactly the frames whose one-sample position falls inside it, in order, and the state after every call equals the
    one-sample run's at that sample."""
    fx = F.fixture()
    rng = np.random.default_rng(seed)
    chans = rng.choice(F.NCH, size=4, replace=False)
    cuts = [int(v) for v in rng.integers(1, 3000, size=40)] + [1] * 5 + [int(v) for v in rng.integers(1, 300, size=100)]
    bounds = [int(b) for b in np.cumsum(cuts) if b < fx.env.shape[1]]
    one = F.traces(tuple(bounds + [fx.env.shape[1]]))
    for c in chans:
        calls, snaps = F.run_chunked(oracle, fx.env[c], cuts)
        frames = one[c].frames
        i = 0
        for keys, (a, b) in calls:
            inside = [f for f in frames[i:] if a <= f.pos < b]
            assert keys == [f.msg.key() for f in inside], (c, a, b)
            i += len(inside)
            vec, fr = one[c].snaps[b]
            assert snaps[b] == (vec, fr[:-1]), (c, b)
        assert i == len(frames)


def test_emulation_positions_and_framing_state(emul, oracle):
    """demod_emul (demod_core.h + frame_sm.h on the host, one lane) over the whole fixture in 4096-sample calls: its
    frame records (pos and soh_pos included) and its whole acb_chan_state_t after every call — blk_len, blk_err, the
    text, crc[0] in F_CRC2, pos and soh_pos — equal the one-sample run's."""
    fx = F.fixture()
    n = fx.env.shape[1]
    bounds = list(range(4096, n, 4096)) + [n]
    one = F.traces(tuple(bounds))
    frames = (EmulFrame * 64)()
    for c in range(F.NCH):
        x = np.ascontiguousarray(fx.env[c])
        st = fresh_state()
        got, a = [], 0
        for b in bounds:
            k = emul.demod_emul(C.byref(st), x[a:].ctypes.data, b - a, 1, 0, frames, 64)
            assert k <= 64
            got += [(f.len, f.err, bytes(f.txt[:f.len]), bytes(f.crc), int(f.pos), int(f.soh_pos)) for f in frames[:k]]
            vec, fr = one[c].snaps[b]
            assert st.vec() == vec and F.device_framing(st) == fr and st.pos == b, (c, b)
            a = b
        want = [(f.msg.len, f.msg.err, bytes(f.msg.txt[:f.msg.len]), bytes(f.msg.crc), f.pos, f.soh_pos)
                for f in one[c].frames]
        assert got == want, c
