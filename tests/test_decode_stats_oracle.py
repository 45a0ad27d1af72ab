"""Decode statistics (ACB_FLAG_DECODE_STATS) off the GPU.

1. The restatement's counts (tests/host/decode_stats_oracle.c on the pinned oracle/acars_oracle.c) equal the number of
   lines of each kind the unmodified reference prints with -v (acars.c compiled in place, oracle/_ref/
   libacarsref_verbose.so), per channel, on the synthetic fixtures (tests/decode_stats_fixtures.py) and test.wav.
   Counting is order-free, so the reference's thread interleaving does not matter.
2. The demodulator loop the device runs (demod_core.h, built for the host with the counting accessor by
   tests/host/demod_emul_counted.cpp) counts what the restatement counts, under ragged chunkings.
3. The block FEC's verdicts: the restatement's classification equals the reference's lines frame by frame on the
   6000-frame fuzz of test_oracle_vs_reference.
"""
from __future__ import annotations

import ctypes as C
import json
import subprocess
import sys
from collections import Counter
from pathlib import Path

import numpy as np
import pytest

import decode_stats_fixtures as fx
import decode_stats_refs as dsr
import refs
from acarsdec_b200 import synth
from common import load_testwav

HERE = Path(__file__).resolve().parent
K = 160
FM = synth.DEFAULT_FREQS_MHZ


def fixture_envelope(oracle) -> np.ndarray:
    """(8, nsamp) float32: a noisy stream of every fixture kind, 3000 samples of silence, a noise-free one."""
    parts = []
    for seed, sigma in ((31, 1.5), (32, 0.0)):
        plan, _ = fx.plan_stream(K, 2.4, seed, noise_sigma=sigma)
        iq = synth.render_blocks(plan, 0, synth.blocks_for_seconds(K, 2.4)).reshape(-1)
        parts.append(oracle.channelize(iq, K, oracle.wf(K, FM)))
        parts.append(np.zeros((len(FM), 3000), np.float32))
    return np.ascontiguousarray(np.concatenate(parts, axis=1))


@pytest.fixture(scope="module")
def envelope(oracle):
    return fixture_envelope(oracle)


def run_reference(args) -> tuple[dict, str]:
    r = subprocess.run([sys.executable, str(HERE / "decode_stats_ref_worker.py"), *map(str, args)], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return {int(k): v for k, v in json.loads(r.stdout).items()}, r.stderr


needs_ref = pytest.mark.skipif(not refs.ref_available("verbose"), reason="oracle/_ref not built (needs the reference tree)")


def test_fixtures_reach_every_counter(oracle, envelope):
    total = Counter()
    for c in range(envelope.shape[0]):
        d, _, st = dsr.restate_chain(oracle, envelope[c])
        dsr.check_invariants(d, st.state)
        total.update(d)
    for f in dsr.FIELDS:
        if f in ("lost", "fec_parity_problem"):       # no ring here; no input reaches the second (fixture docstring)
            assert total[f] == 0, f
        else:
            assert total[f] > 0, (f, dict(total))


@needs_ref
@pytest.mark.parametrize("source", ["fixtures", "testwav"])
def test_restatement_counts_equal_reference_lines(oracle, envelope, tmp_path, source):
    if source == "fixtures":
        dm, chunk = envelope, 4096
    else:
        x, _ = load_testwav()
        dm, chunk = np.ascontiguousarray(x.T), 4096        # soundfile.c's chunks
    np.save(tmp_path / "dm.npy", dm)
    delivered, err = run_reference(["audio", tmp_path / "dm.npy", chunk])
    lines = dsr.count_lines(err)
    assert set(lines) <= set(range(dm.shape[0]))
    for c in range(dm.shape[0]):
        d, _, _ = dsr.restate_chain(oracle, dm[c], [chunk] * (dm.shape[1] // chunk + 1))
        got = lines.get(c, Counter())
        for f, n in got.items():
            assert d[f] == n, (c, f, d[f], n)
        for f in dsr.FIELDS:
            if f not in ("preamble", "started", "delivered", "lost") and f not in got:
                assert d[f] == 0, (c, f)
        assert d["delivered"] == delivered.get(c, 0), c


@pytest.fixture(scope="module")
def emul(native):
    L = C.CDLL(str(dsr.emul_counted_lib()))
    from test_demod_core import EmulFrame
    from acarsdec_b200 import api
    L.demod_emul_counted.argtypes = [C.POINTER(api.ChanState), C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(EmulFrame),
                                     C.c_int, C.POINTER(C.c_uint64)]
    return L, EmulFrame


EV_FIELDS = ("preamble", "started", "txt_parity", "txt_long", "txt_missed_end", "emitted", "fec_short", "lost")


@pytest.mark.parametrize("f2f", [0, 1])
def test_device_loop_counts_equal_restatement_ragged(oracle, envelope, emul, f2f):
    from acarsdec_b200 import api
    L, EmulFrame = emul
    rng = np.random.default_rng(77 + f2f)
    frames = (EmulFrame * 64)()
    for c in range(envelope.shape[0]):
        x = envelope[c]
        chunks = [int(v) for v in rng.integers(1, 3000, size=len(x) // 700)]
        chunks.append(len(x))
        want, _, _ = dsr.restate_chain(oracle, x, chunks)
        st = api.ChanState()
        st.nbits = 8
        cnt = (C.c_uint64 * len(EV_FIELDS))()
        pos = 0
        for n in chunks:
            seg = np.ascontiguousarray(x[pos:pos + n])
            if len(seg) == 0:
                break
            assert L.demod_emul_counted(C.byref(st), seg.ctypes.data, len(seg), 1, f2f, frames, 64, cnt) <= 64
            pos += len(seg)
        got = dict(zip(EV_FIELDS, (int(v) for v in cnt)))
        assert got["lost"] == 0
        for f in dsr.K2_FIELDS:
            assert got[f] == want[f], (c, f, got[f], want[f])


@needs_ref
def test_fec_classification_equals_reference_on_fuzz(oracle, tmp_path):
    from test_oracle_vs_reference import _fec_cases
    rng = np.random.default_rng(4321)
    cases = _fec_cases(rng, 6000)
    lens = np.array([len(t) for _, t, _ in cases], np.int32)
    txt = np.zeros((len(cases), 250), np.uint8)
    crcs = np.zeros((len(cases), 2), np.uint8)
    mine = []
    for i, (_, t, crc) in enumerate(cases):
        txt[i, :len(t)] = np.frombuffer(bytes(t), np.uint8)[:250]
        crcs[i] = np.frombuffer(bytes(crc), np.uint8)
        m = refs.Msg()
        m.chn, m.len = i, len(t)
        m.txt[:min(len(t), 250)] = bytes(t)[:250]
        m.crc[:] = bytes(crc)
        k = dsr.OrcCounts()
        dsr.fec_counted(oracle, m, k)          # also holds the keep decision and the repair to orc_block_fec
        mine.append({f: v for f, v in k.as_dict().items() if v})
    np.savez(tmp_path / "frames.npz", len=lens, txt=txt, crc=crcs)
    delivered, err = run_reference(["blocks", tmp_path / "frames.npz"])
    lines = dsr.count_lines(err, skip_chn=(0x7FFE,))
    kinds = Counter()
    for i, want in enumerate(mine):
        got = dict(lines.get(i, Counter()))
        got.pop("emitted", None)
        if delivered.get(i):
            got["delivered"] = delivered[i]
        assert got == want, (i, got, want)
        kinds.update(want)
    for f in ("fec_parity_excess", "fec_parity", "fec_crc", "fec_fixed", "fec_unfixable", "delivered"):
        assert kinds[f] > 50, (f, dict(kinds))
    assert kinds["fec_short"] > 5
