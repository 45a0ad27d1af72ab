"""The exact IQ channelizer (k_channelize_iq4: four rows per thread, (c, d) tables, row units loaded straight from global
memory, the table through a chunked shared-memory ring) at shapes that reach every edge of its tiling, envelope bit-exact
to the CPU definitions: row windows that are and are not a whole number of table chunks (K = 160, 192, 200, 240), partial
channel groups and the (nch & 3) store path, taps < K and taps > K across ragged submits, u8 and CS16 (interleaved and
planar), a different table per stream; and pipelined submits (demodulator co-resident) equal to sync-per-submit ones at a
production-sized stream count."""
import numpy as np
import pytest

import fir_stream_refs
import ovl_refs
from acarsdec_b200 import api, synth
from common import bits_equal

pytestmark = pytest.mark.gpu

FLAG_CS16 = 4


def tables(rng, S, nch, taps):
    """one (nch, 2*taps) table per stream"""
    return [(rng.standard_normal((nch, 2 * taps)) / taps).astype(np.float32) for _ in range(S)]


# (K, taps, nch): units per row 20 / 24 / 25 / 30 against a 4-unit table chunk; taps < K padded to whole units
U8_FIR = [(160, 160, 8), (192, 192, 12), (200, 200, 3), (240, 240, 16), (200, 165, 1), (240, 97, 8), (160, 41, 12)]


@pytest.mark.parametrize("K,taps,nch", U8_FIR)
def test_u8_taps_le_k(native, oracle, K, taps, nch):
    rng = np.random.default_rng(K * 31 + taps + nch)
    S, nblk = 3, 2
    wfs = tables(rng, S, nch, taps)
    iq = rng.integers(0, 256, size=(S, nblk * 2048 * K), dtype=np.uint8)
    with api.Context(K, S, nch, nblk, taps=taps) as ctx:
        for s in range(S):
            ctx.set_wf(s, wfs[s])
        ctx.submit_host(iq, nblk)
        got = ctx.read_dm(nblk * 1024)
    for s in range(S):
        assert bits_equal(got[s], oracle.channelize_fir(iq[s], K, taps, wfs[s]).T.copy()), s


@pytest.mark.parametrize("K,taps,nch", [(160, 3 * 160 + 5, 3), (200, 2 * 200, 12), (240, 240 + 8, 16), (192, 5 * 192, 8)])
def test_u8_taps_gt_k_three_submits(native, K, taps, nch):
    rng = np.random.default_rng(K * 17 + taps)
    S, nblk = 2, 2
    wfs = tables(rng, S, nch, taps)
    bb = nblk * 2048 * K
    x = rng.integers(0, 256, size=(S, 3 * bb), dtype=np.uint8)
    with api.Context(K, S, nch, nblk, taps=taps) as ctx:
        for s in range(S):
            ctx.set_wf(s, wfs[s])
        got = []
        for i in range(3):
            ctx.submit_host(np.ascontiguousarray(x[:, i * bb:(i + 1) * bb]), nblk)
            got.append(ctx.read_dm(nblk * 1024))
        got = np.concatenate(got, axis=1)
    for s in range(S):
        assert bits_equal(got[s], ovl_refs.channelize_ovl(x[s], K, wfs[s]).T.copy()), s


def _cs16_run(ctx, x, cuts, planar):
    out, p = [], 0
    for n in cuts:
        part = np.ascontiguousarray(x[:, p:p + n])
        p += n
        got = (ctx.submit_cs16_planar(np.ascontiguousarray(part[..., 0]), np.ascontiguousarray(part[..., 1])) if planar
               else ctx.submit_cs16(part))
        if got:
            out.append(ctx.read_dm(got))
    return np.concatenate(out, axis=1)


@pytest.mark.parametrize("K,taps,nch,planar", [
    (160, 160, 8, False), (200, 150, 3, True), (240, 240, 12, False), (192, 61, 16, True),      # taps <= K
    (160, 2 * 160 + 4, 1, False), (200, 3 * 200, 12, True), (240, 240 + 12, 8, False),         # taps > K
])
def test_cs16_ragged_submits(native, K, taps, nch, planar):
    rng = np.random.default_rng(K * 13 + taps + planar)
    S, nblk = 2, 2
    wfs = tables(rng, S, nch, taps)
    n = 2 * nblk * 1024 * K + K // 3
    x = rng.integers(-32768, 32768, size=(S, n, 2), dtype=np.int16)
    cuts = [nblk * 1024 * K - 5, K // 2 + 1, 3 * K + 7]
    cuts.append(n - sum(cuts))
    with api.Context(K, S, nch, nblk + 1, flags=FLAG_CS16, taps=taps) as ctx:
        for s in range(S):
            ctx.set_wf(s, wfs[s])
        got = _cs16_run(ctx, x, cuts, planar)
    for s in range(S):
        want = (ovl_refs.channelize_ovl_cs16(x[s], K, wfs[s]) if taps > K
                else fir_stream_refs.channelize_fir_cs16(x[s], K, wfs[s]))
        assert got.shape[1] == want.shape[1]
        assert bits_equal(got[s], want.T.copy()), s


def test_pipelined_equals_sync_per_submit(native):
    """528 streams x 8 channels, K = 160, four submits of one block: with the submits in flight together (the demodulator
    of submit i under the channelizer of submit i+1) the frames, every demodulator state and the last envelope are the
    same bytes as with a sync after each submit."""
    K, S, nch, nsub = 160, 528, 8, 4
    fm = synth.DEFAULT_FREQS_MHZ[:nch]
    fd, _, fc = api.plan(K, fm)
    pool = []
    for i in range(4):
        plan = synth.make_plan(K, fm, fc, seconds=nsub * 1024 / 12500, seed=40 + i, msgs_per_chan_per_sec=3.0,
                               text_len=(5, 30), amp=(6.0, 12.0))
        pool.append(synth.render_blocks(plan, 0, nsub).reshape(-1))
    bb = 2048 * K
    x = np.empty((S, nsub * bb), dtype=np.uint8)
    for s in range(S):
        x[s] = np.roll(pool[s % 4], 2 * 977 * (s // 4))

    def run(sync_each):
        with api.Context(K, S, nch, 1) as ctx:
            for s in range(S):
                ctx.set_plan(s, fd)
            for i in range(nsub):
                ctx.submit_host(np.ascontiguousarray(x[:, i * bb:(i + 1) * bb]), 1)
                if sync_each:
                    ctx.sync()
            ctx.sync()
            msgs = sorted((m.stream,) + m.as_tuple() for m in ctx.drain())
            states = [ctx.get_state(s, c).vec() for s in range(S) for c in range(nch)]
            return msgs, states, ctx.read_dm(1024)

    a, b = run(False), run(True)
    assert len(a[0]) >= 100
    assert a[0] == b[0]
    assert a[1] == b[1]
    assert a[2].tobytes() == b[2].tobytes()
