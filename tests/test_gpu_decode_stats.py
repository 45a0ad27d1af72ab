"""Decode statistics on the device (ACB_FLAG_DECODE_STATS): k_demod2_stats and k_block_fec_stats against the
restatement's counts (tests/host/decode_stats_oracle.c, pinned to the reference's -v lines by
tests/test_decode_stats_oracle.py),
per chain, after every acb_collect and acb_sync."""
from __future__ import annotations

from collections import Counter

import numpy as np
import pytest

import decode_stats_fixtures as fx
import decode_stats_refs as dsr
import refs
from acarsdec_b200 import api, synth

pytestmark = pytest.mark.gpu

K = 160
FM = synth.DEFAULT_FREQS_MHZ
NCH = len(FM)
NBLK, NSUB = 4, 8                      # blocks per submit, submits: 2.6 s of every fixture kind
NPLAN = 4                              # distinct streams; stream s carries plan s % NPLAN


@pytest.fixture(scope="module")
def signal(oracle):
    """u8 IQ of NPLAN fixture streams and, per (plan, channel), the restatement's cumulative counts after each submit."""
    iq, snaps = [], []
    for p in range(NPLAN):
        plan, fd = fx.plan_stream(K, NBLK * NSUB * 1024 / 12500, 41 + p, noise_sigma=0.0 if p == NPLAN - 1 else 1.5)
        x = synth.render_blocks(plan, 0, NBLK * NSUB)
        iq.append(x.reshape(NSUB, -1))
        dm = oracle.channelize(x.reshape(-1), K, oracle.wf(K, FM))
        per_ch = []
        for c in range(NCH):
            chan, sync, k, sink, seq = oracle.new_chan(c), dsr.new_sync(), dsr.OrcCounts(), refs.Sink(), []
            for i in range(NSUB):
                dsr.demod_counted(oracle, chan, sync, dm[c, i * NBLK * 1024:(i + 1) * NBLK * 1024], sink, k)
                for m in sink.msgs():
                    dsr.fec_counted(oracle, m, k)
                sink.c.nmsg = 0
                d = k.as_dict()
                dsr.check_invariants(d, chan.state)
                seq.append(d)
            per_ch.append(seq)
        snaps.append(per_ch)
    return fd, np.stack(iq, axis=1), snaps          # iq: (NSUB, NPLAN, bytes per stream and submit)


def _expect(snaps, S, covered) -> np.ndarray:
    """(S, NCH) DECODE_STATS_DTYPE: stream s's chains as the restatement counts plan s % NPLAN after `covered` submits"""
    per_plan = np.array([[tuple(snaps[p][c][covered - 1][f] for f in dsr.FIELDS) for c in range(NCH)] for p in range(NPLAN)],
                        dtype=api.DECODE_STATS_DTYPE)
    return per_plan[np.arange(S) % NPLAN]


def _check(got: np.ndarray, want: np.ndarray, delivered: Counter):
    bad = np.argwhere(got != want)
    assert len(bad) == 0, [(tuple(i), got[tuple(i)], want[tuple(i)]) for i in bad[:3]]
    d = np.zeros(got.shape, np.uint64)
    for (s, c), v in delivered.items():
        d[s, c] = v
    assert np.array_equal(got["delivered"], d)


def _delivered(records) -> Counter:
    return Counter(zip(records["stream"].tolist(), records["chn"].tolist()))


def _run_u8(signal, S, flags=api.FLAG_DECODE_STATS, on_collect=None):
    """S streams (u8 IQ from device memory), one collect behind each submit; returns the context's final table and the
    messages.  on_collect(ctx, covered, table, delivered) runs after every collect and the final sync."""
    import torch
    fd, iq, snaps = signal
    dev = torch.from_numpy(iq).cuda()                 # (NSUB, NPLAN, n)
    idx = torch.arange(S, device="cuda") % NPLAN
    delivered, msgs = Counter(), []
    with api.Context(K, S, NCH, NBLK, flags=flags | 1) as ctx:       # NO_INPUT_STAGING: device submits only
        for s in range(S):
            ctx.set_plan(s, fd)
        keep = []
        for i in range(NSUB):
            x = dev[i].index_select(0, idx).contiguous()
            torch.cuda.synchronize()                  # the context's streams are not ordered behind torch's
            keep.append(x)
            ctx.submit_device(x.data_ptr(), NBLK, x.stride(0))
            if i >= 1:
                ctx.collect()
                r = ctx.drain_records()
                msgs.append(r)
                delivered.update(zip(r["stream"].tolist(), r["chn"].tolist()))
                if on_collect:
                    on_collect(ctx, i, delivered)
            if len(keep) > 2:
                keep.pop(0)
        ctx.sync()
        r = ctx.drain_records()
        msgs.append(r)
        delivered.update(zip(r["stream"].tolist(), r["chn"].tolist()))
        if on_collect:
            on_collect(ctx, NSUB, delivered)
        states = [ctx.get_state(s, c).vec() for s in range(min(S, 8)) for c in range(NCH)]
        return np.concatenate(msgs), states, ctx.read_dm(NBLK * 1024)


@pytest.mark.parametrize("S,lanes", [(4, 8), (528, 4), (1056, 2), (2112, 1), (4224, 1)])
def test_counts_equal_restatement_after_every_collect(native, signal, S, lanes):
    """Stream counts at which the context picks each width (one lane at 2112 and 4224 streams: the two register budgets)."""
    dev_sms = __import__("torch").cuda.get_device_properties(0).multi_processor_count
    if dev_sms != 132:
        pytest.skip("stream counts chosen for a 132-SM H100")
    _, _, snaps = signal
    seen = []

    def on_collect(ctx, covered, delivered):
        _check(ctx.decode_stats(), _expect(snaps, S, covered), delivered)
        seen.append(covered)
    _run_u8(signal, S, on_collect=on_collect)
    assert seen == list(range(1, NSUB + 1))


def test_flag_changes_nothing_else(native, signal):
    a, sa, da = _run_u8(signal, 4)
    b, sb, db = _run_u8(signal, 4, flags=0)
    assert len(a) == len(b) > 0 and bool((a == b).all())           # field by field (the records' padding is not data)
    assert sa == sb
    assert da.tobytes() == db.tobytes()
    with api.Context(K, 1, NCH, 1) as ctx:
        with pytest.raises(api.AcbError):
            ctx.decode_stats()


def test_reset_and_acb_reset(native, signal):
    fd, iq, snaps = signal
    with api.Context(K, NPLAN, NCH, NBLK, flags=api.FLAG_DECODE_STATS) as ctx:
        for s in range(NPLAN):
            ctx.set_plan(s, fd)
        ctx.submit_host(np.ascontiguousarray(iq[0]), NBLK)
        ctx.submit_host(np.ascontiguousarray(iq[1]), NBLK)
        ctx.sync()
        r = ctx.drain_records()
        first = ctx.decode_stats(reset=True)
        _check(first, _expect(snaps, NPLAN, 2), _delivered(r))
        assert int(ctx.decode_stats()["started"].sum()) == 0           # read and cleared
        # submits in flight when acb_reset comes are abandoned: they count nothing, and the counts restart
        ctx.submit_host(np.ascontiguousarray(iq[2]), NBLK)
        ctx.reset()
        assert all(int(ctx.decode_stats()[f].sum()) == 0 for f in dsr.FIELDS)
        ctx.submit_host(np.ascontiguousarray(iq[0]), NBLK)
        ctx.sync()
        _check(ctx.decode_stats(), _expect(snaps, NPLAN, 1), _delivered(ctx.drain_records()))


@pytest.mark.parametrize("mode", [0, 1])
def test_multi_equals_one_context(native, signal, mode):
    import torch
    fd, iq, snaps = signal
    ndev = torch.cuda.device_count()
    S = 6
    x = np.ascontiguousarray(np.stack([iq[:, s % NPLAN] for s in range(S)], axis=1))   # (NSUB, S, n)
    devices = [i % ndev for i in range(2)]
    with api.MultiContext(K, S, NCH, NBLK, devices, mode=mode, flags=api.FLAG_DECODE_STATS) as m:
        for s in range(S):
            m.set_plan(s, fd)
        delivered = Counter()
        for i in range(NSUB):
            m.submit_host(x[i], NBLK)
            if i >= 1:
                m.collect()
                delivered.update((g.stream, g.chn) for g in m.drain())
                _check(m.decode_stats(), _expect(snaps, S, i), delivered)
        m.sync()
        delivered.update((g.stream, g.chn) for g in m.drain())
        _check(m.decode_stats(), _expect(snaps, S, NSUB), delivered)


# ----------------------------------------------------------------------------- the streaming kinds


STREAM_CASES = [("real", 0, 0, "host"), ("cs16", 0, 0, "device"), ("planar", 0, 0, "host"),
                ("real", 2 * 200 + 40, 32, "device"), ("cs16", 160 + 96, 16, "host"), ("planar", 0, 64, "device"),
                ("real", 0, 8, "host")]


@pytest.mark.parametrize("kind,taps,fast,where", STREAM_CASES)
def test_streaming_counts_follow_the_envelope(native, oracle, kind, taps, fast, where):
    """Real and CS16 input (interleaved and planar, host and device submits, taps = K and > K, exact and fast forms):
    the counts are the restatement's over the context's own envelope, and the same for two different cuts."""
    import test_gpu_stream_device as sd
    Kk = sd._kind_K(kind)
    n = 3 * sd.MAXBLK * 1024 * Kk
    fd, fc, x = sd._signal(kind, 5, n)
    results = []
    ragged = sd._counts(Kk)[:5]
    ragged += [1024 * Kk] * ((n - sum(ragged)) // (1024 * Kk)) + [(n - sum(ragged)) % (1024 * Kk)]
    for cuts in (ragged, [n // 3, n // 3, n - 2 * (n // 3)]):
        ctx = sd._make(kind, fast | api.FLAG_DECODE_STATS, taps, fd, fc)
        keep, env, pos = [], [], 0
        for c in cuts:
            c = min(c, n - pos)
            if c <= 0:
                break
            part = x[:, pos:pos + c]
            rows = sd._device_submit(ctx, kind, part, keep) if where == "device" else sd._host_submit(ctx, kind, part)
            if rows:
                env.append(ctx.read_dm(rows))
            pos += c
        ctx.sync()
        delivered = Counter((m.stream, m.chn) for m in ctx.drain())
        got = ctx.decode_stats()
        ctx.close()
        dm = np.concatenate(env, axis=1)                          # (S, rows, nch)
        want = [[dsr.restate_chain(oracle, dm[s, :, c])[0] for c in range(sd.NCH)] for s in range(sd.NSTREAMS)]
        for s in range(sd.NSTREAMS):
            for c in range(sd.NCH):
                g = {f: int(got[s, c][f]) for f in dsr.FIELDS}
                assert g == want[s][c], (cuts[:3], s, c, g, want[s][c])
                assert g["delivered"] == delivered[(s, c)]
        assert int(got["delivered"].sum()) > 0
        results.append(got)
    assert results[0].tobytes() == results[1].tobytes()
