"""Message positions, the framing state and the frame synchroniser's rare exits on the device, against the
restatement driven one envelope sample at a time (tests/frame_pos_refs.py).

Every message is compared as msg_tuple + pos + soh_pos, with block == pos // 1024, in the library's emission order;
every chain's whole acb_chan_state_t (vec() and the framing fields: state, blk_len, blk_err, the text, crc[0] in F_CRC2,
pos, soh_pos) is compared after every sync.  The fixture walks k_demod2 -> DevFrameAcc -> emit_frame -> k_block_fec
through every exit of frame_sm.h (tests/test_frame_pos_refs.py proves it).  Covered: the u8 exact path with submits
that end mid-byte in F_TXT / F_CRC1 / F_CRC2 and frames completing on the last sample of a block and on the first of
the next; acb_submit_dm_host at every lane form, with shadow groups behind a chain whose DLE finish reads its text
back; a mid-frame get_state / set_state round trip; the lean (MINB = 0) demodulator instantiations; the real and CS16
streaming front-ends at taps > K."""
import ctypes as C

import numpy as np
import pytest

import frame_pos_refs as F
import ovl_refs
from acarsdec_b200 import api, synth
from common import msg_tuple

pytestmark = pytest.mark.gpu

FLAG_NO_STAGING, FLAG_REAL, FLAG_CS16 = 1, 2, 4
NCH = F.NCH


@pytest.fixture(scope="module")
def nsm():
    """the device's SM count (cudaDevAttrMultiProcessorCount, as the demod launcher reads it)"""
    rt = C.CDLL("libcudart.so.12")
    n = C.c_int(0)
    assert rt.cudaDeviceGetAttribute(C.byref(n), 16, 0) == 0 and n.value > 0
    return n.value


def expected(oracle, tr, stream, chn, lo, hi, off=0):
    """(stream, msg_tuple, pos, soh_pos) of the frames of a one-sample trace completing in [lo, hi) that the block FEC
    delivers; positions shifted by `off` (a chain whose state was set to pos = soh_pos = off)"""
    out = []
    for f in tr.frames:
        if lo <= f.pos < hi:
            m = oracle.fec(f.msg)
            if m is not None:
                m.chn = chn
                out.append((stream,) + msg_tuple(m) + (f.pos + off, f.soh_pos + off))
    return out


def raw_count(tr, lo, hi):
    return sum(lo <= f.pos < hi for f in tr.frames)


def device_msgs(ctx):
    got = ctx.drain()
    for m in got:
        assert m.block == m.pos // api.OUTBLK
    return [(m.stream,) + msg_tuple(m) + (m.pos, m.soh_pos) for m in got]


def full_state(st):
    return st.vec(), F.device_framing(st), st.pos


def want_state(tr, n, off=0):
    vec, fr = tr.snaps[n]
    return vec, fr[:-1] + (fr[-1] + off,), n + off


def mid_byte(tr, n, states):
    """the chain is inside a byte of one of `states` after n samples"""
    return n > 0 and tr.states[n - 1] in states and 1 <= tr.nbits[n - 1] <= 7


def first_mid_byte(tr, states, after=0):
    return next(i + 1 for i in range(after, len(tr.states)) if tr.states[i] in states and 1 <= tr.nbits[i] <= 7)


# ------------------------------------------------------------------ 1. u8 IQ, exact path, ragged submit_host cuts

U8_CUTS = [1, 3, 2, 1, 4, 1, 2]


def shifted_iq(fx, d):
    """the fixture's IQ behind d rows of noise, padded with noise to whole blocks: its envelope is the fixture's
    shifted by d rows (taps = K: a row depends on its own K samples only)"""
    K, rowb = fx.K, 2 * fx.K
    noise = synth.StreamPlan(K=K, freqs_hz=fx.freqs_hz, fc_hz=fx.fc, noise_sigma=F.NOISE, seed=977)
    nz = synth.render_blocks(noise, 0, 2)
    rows = d + fx.iq.size // rowb
    pad = -rows % api.OUTBLK
    return np.concatenate([nz[0][(api.OUTBLK - d) * rowb:] if d else nz[0][:0], fx.iq, nz[1][:pad * rowb]])


def find_shift(oracle, fx, wf, target):
    """a shift d that makes a delivered frame of channel 0 complete on a sample with pos % 1024 == target.  Behind a
    different prefix the demodulator's bit clock settles a few samples differently (a frame's end moves by d + 0 or
    d - 3 here, so some residues are out of its reach), so the neighbours of each frame's plain guess are tried."""
    for f0 in [f.pos for f in F.traces()[0].frames if oracle.fec(f.msg) is not None][:4]:
        for delta in (0, 3, -3, 1, -1, 2, -2, 4, -4):
            d = (target - f0 + delta) % api.OUTBLK
            iq = shifted_iq(fx, d)
            tr = F.run(oracle, oracle.channelize(iq, fx.K, wf[:1])[0])
            if any(f.pos % api.OUTBLK == target and f.pos > 0 and oracle.fec(f.msg) is not None for f in tr.frames):
                return d, iq
    raise AssertionError(f"no shift puts a frame at pos % 1024 == {target}")


@pytest.fixture(scope="module")
def u8_case(native, oracle):
    fx = F.fixture()
    wf = oracle.wf(fx.K, F.FM)
    streams = [shifted_iq(fx, 0)] + [find_shift(oracle, fx, wf, t)[1] for t in (api.OUTBLK - 1, 0)]
    n = min(s.size for s in streams)
    iq = np.stack([s[:n] for s in streams])
    nblk = n // (2 * fx.K * api.OUTBLK)
    cuts, b = [], 0
    while b < nblk:
        cuts.append(min(U8_CUTS[len(cuts) % len(U8_CUTS)], nblk - b))
        b += cuts[-1]
    bounds = tuple(int(x) * api.OUTBLK for x in np.cumsum(cuts))
    trs = [[F.run(oracle, e, checkpoints=bounds) for e in oracle.channelize(iq[s], fx.K, wf)] for s in range(len(iq))]
    return fx, iq, cuts, bounds, trs


def test_u8_exact_path_positions_and_state(native, oracle, u8_case):
    """Three streams (the fixture, and the fixture shifted so that a delivered frame completes on the last sample of a
    1024 block, and on the first sample of one), K = 160, submits of 1 to 4 blocks: after every sync the messages in
    (block, stream, channel, time) order and every chain's whole state; raw_frames counts every frame the sink got,
    short ones included; fec_dropped = raw - delivered; nothing lost."""
    fx, iq, cuts, bounds, trs = u8_case
    S = len(iq)
    bb = 2 * fx.K * api.OUTBLK
    mid = {"txt": 0, "crc": 0}
    delivered = 0
    with api.Context(fx.K, S, NCH, max(cuts)) as ctx:
        for s in range(S):
            ctx.set_plan(s, fx.freqs_hz)
        b0, lo = 0, 0
        for nb, hi in zip(cuts, bounds):
            ctx.submit_host(np.ascontiguousarray(iq[:, b0 * bb:(b0 + nb) * bb]), nb)
            b0 += nb
            ctx.sync()
            got = device_msgs(ctx)
            want = sorted((w for s in range(S) for c in range(NCH) for w in expected(oracle, trs[s][c], s, c, lo, hi)),
                          key=lambda w: (w[-2] // api.OUTBLK, w[0], w[1], w[-2]))
            assert got == want, hi
            delivered += len(got)
            for s in range(S):
                for c in range(NCH):
                    assert full_state(ctx.get_state(s, c)) == want_state(trs[s][c], hi), (s, c, hi)
                    mid["txt"] += mid_byte(trs[s][c], hi, (F.TXT,))
                    mid["crc"] += mid_byte(trs[s][c], hi, (F.CRC1, F.CRC2))
            lo = hi
        st = ctx.stats()
    raw = sum(raw_count(trs[s][c], 0, bounds[-1]) for s in range(S) for c in range(NCH))
    assert st.raw_frames == raw and st.fec_dropped == raw - delivered and st.frames_lost == 0
    assert mid["txt"] > 0 and mid["crc"] > 0
    pos = {f.pos % api.OUTBLK for s in (1, 2) for f in trs[s][0].frames if oracle.fec(f.msg) is not None}
    assert {api.OUTBLK - 1, 0} <= pos


# ------------------------------------------------------------------ 2. submit_dm at every lane form

COL_SHIFT = 6          # chain (s, c) reads column (c + 6 s) % 11: the last chain reads column 5, which has a DLE finish


@pytest.fixture(scope="module")
def dm_case(native, oracle):
    """Two streams of the fixture's 11 columns; stream 1 starts from an inverted polarity (MskS ^= 2) and its first two
    chains at pos offsets that put a delivered frame on the last sample of a 1024 block and on the first of one.  Cuts
    end mid-byte in F_CRC1 (chain 0), F_TXT (chain 3) and F_CRC2 (the last chain)."""
    fx = F.fixture()
    n = fx.env.shape[1]
    cols = [[(c + COL_SHIFT * s) % NCH for c in range(NCH)] for s in range(2)]
    base = F.traces()
    inv = oracle.new_chan(0)
    inv.MskS ^= 2
    inv_last = F.run(oracle, fx.env[cols[1][NCH - 1]], chan=inv)
    e1 = first_mid_byte(base[cols[0][0]], (F.CRC1,), 2000)
    e2 = first_mid_byte(base[cols[0][3]], (F.TXT,), e1 + 500)
    e3 = first_mid_byte(inv_last, (F.CRC2,), e2 + 500)
    bounds = (e1, e2, e3, n)
    trs = [[F.run(oracle, fx.env[k], checkpoints=bounds) for k in cols[0]],
           [F.run(oracle, fx.env[k], chan=inv, checkpoints=bounds) for k in cols[1]]]
    offs = [[0] * NCH, [0] * NCH]
    for c, t in ((0, api.OUTBLK - 1), (1, 0)):
        f = next(f for f in trs[1][c].frames if oracle.fec(f.msg) is not None)
        offs[1][c] = 5 * api.OUTBLK + (t - f.pos) % api.OUTBLK
    assert "dle" in trs[1][NCH - 1].events
    return fx, bounds, trs, offs, inv


def run_dm(ctx, env_cols, bounds, trs, offs, oracle, S):
    """submit the columns in the given cuts, checking messages and states after every sync; returns delivered"""
    delivered, lo = 0, 0
    for hi in bounds:
        dm = np.ascontiguousarray(np.stack([env_cols[s][:, lo:hi].T for s in range(S)]))
        ctx.submit_dm(dm)
        ctx.sync()
        got = device_msgs(ctx)
        want = sorted((w for s in range(S) for c in range(len(trs[s]))
                       for w in expected(oracle, trs[s][c], s, c, lo, hi, offs[s][c])), key=lambda w: (w[0], w[1], w[-2]))
        assert got == want, hi
        delivered += len(got)
        for s in range(S):
            for c in range(len(trs[s])):
                assert full_state(ctx.get_state(s, c)) == want_state(trs[s][c], hi, offs[s][c]), (s, c, hi)
        lo = hi
    return delivered


def start_states(ctx, offs, inv):
    for s in range(len(offs)):
        for c in range(len(offs[s])):
            st = ctx.get_state(s, c)
            if s == 1:
                st.MskS = inv.MskS
            st.pos = st.soh_pos = offs[s][c]
            ctx.set_state(s, c, st)


@pytest.mark.parametrize("lanes", [1, 2, 4, 8, 17, 20, 24, 33, 34, 36, 40])
def test_dm_every_lane_form(native, oracle, dm_case, lanes, monkeypatch):
    """acb_submit_dm_host with ACB_DEMOD_LANES forcing each form, 2 streams x 11 channels: the last warp carries shadow
    groups of the last chain, whose DLE finish reads its text back from HBM.  Messages per submit in (stream, channel,
    time) order with positions, and every chain's whole state after every sync; a foreign start state (inverted
    polarity, positions offset) carries into the positions."""
    monkeypatch.setenv("ACB_DEMOD_LANES", str(lanes))
    fx, bounds, trs, offs, inv = dm_case
    cols = [[(c + COL_SHIFT * s) % NCH for c in range(NCH)] for s in range(2)]
    env_cols = [fx.env[cols[s]] for s in range(2)]
    cap = max(b - a for a, b in zip((0,) + bounds, bounds))
    with api.Context(F.K_FIX, 2, NCH, -(-cap // api.OUTBLK), flags=FLAG_NO_STAGING) as ctx:
        start_states(ctx, offs, inv)
        delivered = run_dm(ctx, env_cols, bounds, trs, offs, oracle, 2)
        st = ctx.stats()
    raw = sum(raw_count(trs[s][c], 0, bounds[-1]) for s in range(2) for c in range(NCH))
    assert st.raw_frames == raw and st.fec_dropped == raw - delivered and st.frames_lost == 0
    assert mid_byte(trs[0][0], bounds[0], (F.CRC1,)) and mid_byte(trs[0][3], bounds[1], (F.TXT,))
    assert mid_byte(trs[1][NCH - 1], bounds[2], (F.CRC2,))


# ------------------------------------------------------------------ 3. a mid-frame round trip

def test_state_round_trip_inside_a_frame(native, oracle):
    """Stop while chain 0 is inside F_TXT (mid-byte), read every chain's state, continue in a fresh context after
    set_state: the frames, positions and soh_pos equal the uninterrupted run's, including the frame whose SOH came
    before the cut."""
    fx = F.fixture()
    n = fx.env.shape[1]
    f = next(f for f in F.traces()[0].frames if oracle.fec(f.msg) is not None)
    cut = first_mid_byte(F.traces()[0], (F.TXT,), f.soh_pos + 100)
    assert cut <= f.pos
    trs = F.traces((cut, n))
    env = [fx.env]
    offs = [[0] * NCH]
    with api.Context(F.K_FIX, 1, NCH, -(-cut // api.OUTBLK), flags=FLAG_NO_STAGING) as a:
        run_dm(a, env, (cut,), [trs], offs, oracle, 1)
        states = [a.get_state(0, c) for c in range(NCH)]
    assert states[0].Acarsstate == F.TXT and 0 < states[0].soh_pos < cut
    with api.Context(F.K_FIX, 1, NCH, -(-(n - cut) // api.OUTBLK), flags=FLAG_NO_STAGING) as b:
        for c in range(NCH):
            b.set_state(0, c, states[c])
        dm = np.ascontiguousarray(fx.env[:, cut:].T[None])
        b.submit_dm(dm)
        b.sync()
        got = device_msgs(b)
        for c in range(NCH):
            assert full_state(b.get_state(0, c)) == want_state(trs[c], n), c
    want = sorted((w for c in range(NCH) for w in expected(oracle, trs[c], 0, c, cut, n)), key=lambda w: (w[1], w[-2]))
    assert got == want
    assert [w for w in want if w[1] == 0 and w[-1] < cut]        # chain 0's frame in progress at the cut


# ------------------------------------------------------------------ 4. the lean (MINB = 0) demodulator forms

LEAN_SAMPLES = 16 * 1024


def lean_chains(lanes, nsm):
    """kernels.cu launch_demod_pinned: the lean form runs when ceil(chains * L / 32) > 8 * SMs"""
    L = lanes & 15
    return (8 * nsm * 32) // L + 32, L


@pytest.mark.parametrize("lanes", [2, 4, 8, 20, 24])
def test_lean_demod_forms(native, oracle, nsm, lanes, monkeypatch):
    """ACB_DEMOD_LANES forcing a pinned width at more than 8 warps per SM (the MINB = 0 instantiation): chain g reads
    column g % 11 of the fixture's envelope; every chain's frames with positions and its whole state equal the
    restatement's run of its column."""
    monkeypatch.setenv("ACB_DEMOD_LANES", str(lanes))
    fx = F.fixture()
    n = LEAN_SAMPLES
    nchains, L = lean_chains(lanes, nsm)
    S = -(-nchains // NCH)
    nchains = S * NCH
    assert -(-nchains * L // 32) > 8 * nsm
    trs = F.traces((n,))
    col = np.arange(nchains) % NCH
    want_frames = [expected(oracle, trs[k], 0, 0, 0, n) for k in range(NCH)]
    raw = sum(raw_count(trs[k], 0, n) for k in col)
    with api.Context(F.K_FIX, S, NCH, n // api.OUTBLK, flags=FLAG_NO_STAGING) as ctx:
        dm = np.empty((S, n, NCH), dtype=np.float32)
        for c in range(NCH):
            dm[:, :, c] = fx.env[col[np.arange(S) * NCH + c]][:, :n]
        ctx.submit_dm(dm)
        del dm
        ctx.sync()
        rec = ctx.drain_records()
        st = ctx.stats()
        assert st.raw_frames == raw and st.frames_lost == 0
        assert np.array_equal(rec["block"], rec["pos"] // api.OUTBLK)
        g = rec["stream"].astype(np.int64) * NCH + rec["chn"]
        assert np.all(np.diff(g) >= 0)
        bounds = np.searchsorted(g, np.arange(nchains + 1))
        lvl = rec["lvl"].view(np.uint32)
        for ch in range(nchains):
            mine = [(0, 0, int(rec["len"][i]), int(rec["err"][i]), rec["txt"][i, :rec["len"][i]].tobytes(),
                     rec["crc"][i].tobytes(), int(lvl[i]), int(rec["pos"][i]), int(rec["soh_pos"][i]))
                    for i in range(bounds[ch], bounds[ch + 1])]
            assert mine == want_frames[col[ch]], ch
        assert st.fec_dropped == raw - len(rec)
        for ch in range(nchains):
            assert full_state(ctx.get_state(ch // NCH, ch % NCH)) == want_state(trs[col[ch]], n), ch


# ------------------------------------------------------------------ 5. streaming real and CS16 at taps > K

@pytest.mark.parametrize("kind", ["real", "cs16"])
def test_streaming_taps_over_k(native, oracle, kind):
    """The fixture's first four channels through the real (K = 200) or CS16 (K = 160, soapy) front-end at taps = 2K + 7,
    ragged submits: row m completes with sample (m+1)K - 1, so the positions are the one-sample run's on the
    definition's envelope (tests/host/ovl_oracle.c); per submit (its own emission group) in (channel, time) order."""
    nch = 4
    fx = F.fixture()
    K = 200 if kind == "real" else 160
    taps = 2 * K + 7
    fm = F.FM[:nch]
    rows = fx.env.shape[1]
    bursts = [b for b in fx.plan.bursts if b.chan < nch]
    if kind == "real":
        fd, fc, _ = api.air_plan(K * 12500, fm)
        plan = synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, bursts=bursts, noise_sigma=F.NOISE, seed=5)
        x = synth.render_real(plan, 0, rows * K).reshape(1, -1)
        wf = api.build_wf_air_lp(K * 12500, taps, fm)
        env = ovl_refs.channelize_ovl_real(x[0], K, wf)
    else:
        fd, _, fc = api.plan(K, fm)
        plan = synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, bursts=bursts, noise_sigma=F.NOISE, seed=5)
        x = synth.render_cs16(plan, 0, rows * K).reshape(1, rows * K, 2)
    with api.Context(K, 1, nch, 12, flags=FLAG_REAL if kind == "real" else FLAG_CS16, taps=taps) as ctx:
        if kind == "real":
            ctx.set_plan_air(0, fd)
        else:
            fc = ctx.set_plan_cs16(0, fd, 0)
            wf = api.build_wf_cs16_lp(0, K, taps, fd, fc)
            env = ovl_refs.channelize_ovl_cs16(x[0], K, wf)
        cuts = [K - 3, 5 * 1024 * K + 11, 3 * K + 1, 7 * 1024 * K - 5, 2 * 1024 * K + 17]
        while sum(cuts) < x.shape[1]:
            cuts.append(min(9 * 1024 * K + 7, x.shape[1] - sum(cuts)))
        trs = [F.run(oracle, env[c]) for c in range(nch)]
        p, lo, delivered = 0, 0, 0
        for n in cuts:
            part = np.ascontiguousarray(x[:, p:p + n])
            p += n
            got_rows = ctx.submit_real(part) if kind == "real" else ctx.submit_cs16(part)
            ctx.sync()
            hi = lo + got_rows
            got = device_msgs(ctx)
            want = sorted((w for c in range(nch) for w in expected(oracle, trs[c], 0, c, lo, hi)), key=lambda w: (w[1], w[-2]))
            assert got == want, (lo, hi)
            delivered += len(got)
            lo = hi
        for c in range(nch):
            s = ctx.get_state(0, c)
            assert s.pos == lo and s.vec() == trs[c].chan.vec() and F.device_framing(s) == F.framing(trs[c].chan, trs[c].soh_pos)
        st = ctx.stats()
    raw = sum(raw_count(tr, 0, lo) for tr in trs)
    assert lo == env.shape[1] and st.raw_frames == raw and st.fec_dropped == raw - delivered and delivered >= 8
    assert sum(len(tr.events.get(k, [])) for tr in trs for k in ("dle", "len241", "parity5")) >= 3
