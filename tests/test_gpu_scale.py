"""The kernel paths that only production-sized launches reach, against the CPU definitions.

Three launchers change what a kernel does once the workload is large compared with the device, and decide it from the
SM count: k_channelize_wb runs several tiles per CTA, k_block_fec strides over more frames than its grid has threads,
and the context gives each demodulator chain fewer lanes (down to 32 chains per warp, across stream boundaries).  The
heuristics are restated below (wb_tiles_per_cta, demod_lanes) and every case is sized from them and asserts the branch
it is for, so another SM count or a later change of a heuristic moves the shapes instead of silently dropping the
coverage.  Also here: the stream-count limit (streams are grid.y of the channelizer launches)."""
import ctypes as C

import numpy as np
import pytest

import refs
from acarsdec_b200 import api, synth
from common import bits_equal, msg_tuple
from test_gpu_ovl import run_stream_kind
from test_gpu_wideband import freqs_for
from test_oracle_vs_reference import _fec_cases
from test_wideband_oracle import FC, fast_envelope, planner

FLAG_NO_STAGING, FLAG_CS16, FLAG_WB = 1, 4, api.FLAG_FAST_WIDEBAND
ACB_ERR_ARG = -1
WB_CTILE = 256                      # channels per channel tile (acb_internal.h)


@pytest.fixture(scope="module")
def nsm():
    """the device's SM count, read with the attribute the launchers read (cudaDevAttrMultiProcessorCount).  The CUDA
    runtime is asked directly rather than torch (bench.py's way): torch's CUDA initialisation alone holds about 4.5 GB
    of host memory, more than this file's cases need together."""
    rt = C.CDLL("libcudart.so.12")
    n = C.c_int(0)
    assert rt.cudaDeviceGetAttribute(C.byref(n), 16, 0) == 0 and n.value > 0
    return n.value


# ------------------------------------------------------------------ the launchers' heuristics, restated

def wb_rows_per_tile(K):
    """kernels.cu:1473-1476 (wb_rb): tiles of 12 rows while Y' and E of two CTAs fit an SM, else 8"""
    return 12 if 16 * 3 * K + (2 * K - 1) * 8 <= 113 * 1024 else 8


def wb_tiles_per_cta(K, nsamp, nstreams, nch, nsm):
    """kernels.cu:1492-1496 (launch_wb_t): tiles per CTA of a k_channelize_wb launch over nsamp rows"""
    tiles = -(-nsamp // wb_rows_per_tile(K)) * nstreams * -(-nch // WB_CTILE)
    return max(1, min(8, tiles // (8 * nsm)))


def demod_lanes(nchains, nsm):
    """kernels.cu:2696-2703 (demod_pick_lanes, called by acb_create): lanes per demodulator chain"""
    for lanes in (1, 2, 4):
        if nchains * lanes >= 32 * 4 * nsm:
            return lanes
    return 8


def fec_threads(nsm):
    """kernels.cu:2858 (launch_block_fec): frames k_block_fec covers in one grid pass, 4 CTAs of 128 per SM"""
    return 4 * nsm * 128


def test_restated_heuristics_at_h100_size():
    """The worked examples at 132 SMs (H100 SXM)."""
    assert wb_rows_per_tile(1808) == 12 and wb_rows_per_tile(1816) == 8
    assert wb_tiles_per_cta(800, 13 * 1024, 8, 16, 132) == 8               # 8 880 tiles
    assert wb_tiles_per_cta(800, 12 * 1024, 8, 16, 132) == 7
    assert wb_tiles_per_cta(1600, 1024, 2, 300, 132) == 1
    assert [demod_lanes(n, 132) for n in (4223, 4224, 8447, 8448, 16895, 16896)] == [8, 4, 4, 2, 2, 1]
    assert fec_threads(132) == 67_584


# ------------------------------------------------------------------ A. wideband fast form, several tiles per CTA

def wb_slots(k):
    """context.cu upload_wb_plan restated: per channel tile, the channel of every slot (-1 = padding), sorted by the
    residue (k/2) mod 4 and each residue class padded to whole groups of 4"""
    tiles = []
    for z in range(0, len(k), WB_CTILE):
        slots = []
        for res in range(4):
            slots += [c for c in range(z, min(len(k), z + WB_CTILE)) if (int(k[c]) // 2) % 4 == res]
            slots += [-1] * (-len(slots) % 4)
        tiles.append(slots)
    return tiles


def channels_to_check(k, seed, extra=8):
    """A subset on which the CPU definition is computed: the first and last slot of every tile, the first and last
    channel of every residue class present in every tile (the last one sits next to a padding slot when its class is
    not a whole number of groups), and a few at random.  Returns (channels, the residue classes among them, whether
    one of them sits next to a padding slot)."""
    sel, padded = set(), False
    for slots in wb_slots(k):
        real = [c for c in slots if c >= 0]
        sel |= {real[0], real[-1]}
        for res in range(4):
            cls = [c for c in real if (int(k[c]) // 2) % 4 == res]
            sel |= {cls[0], cls[-1]} if cls else set()
        padded |= any(c >= 0 and slots[i + 1] < 0 for i, c in enumerate(slots[:-1]))
    rng = np.random.default_rng(seed)
    sel |= set(int(c) for c in rng.choice(len(k), size=min(extra, len(k)), replace=False))
    assert {c // WB_CTILE for c in sel} == set(range(-(-len(k) // WB_CTILE)))
    return sorted(sel), {(int(k[c]) // 2) % 4 for c in sel}, padded


def check_envelope(oracle, L, kind, x, K, taps, freqs, got, variant=-1, subset=True):
    """got (rows, nch) of one stream against the definition, on channels_to_check (or all of them); returns the
    residue classes checked and whether a channel next to a padding slot was"""
    k, _ = planner(L, kind, variant, K, freqs)
    sel, res, padded = channels_to_check(k, K + taps + len(freqs))
    if not subset:
        sel = list(range(len(freqs)))
    ks, tw = planner(L, kind, variant, K, [freqs[c] for c in sel])
    want = fast_envelope(oracle, kind, x, K, taps, ks, tw)
    assert got.shape[0] == want.shape[1]
    for j, c in enumerate(sel):
        assert bits_equal(got[:, c], want[j]), c
    return res, padded


def check_streams(oracle, L, kind, x, K, taps, fs, got, variant=-1, subset=True, padding=True):
    """every stream of a case; over the streams every residue class and (where the plans have padding slots: 16 or 64
    channels from freqs_for fill whole groups) a channel next to padding are checked"""
    res, padded = set(), False
    for s in range(len(fs)):
        r, p = check_envelope(oracle, L, kind, x[s], K, taps, fs[s], got[s], variant, subset)
        res, padded = res | r, padded or p
    assert res == {0, 1, 2, 3} and padded == padding


def tpc1_rows(K, nstreams, nch, nsm):
    """the most rows a launch may carry and still run one tile per CTA"""
    r = wb_rows_per_tile(K)
    while wb_tiles_per_cta(K, r + 1, nstreams, nch, nsm) == 1:
        r += 1
    return r


@pytest.mark.gpu
def test_wb_u8_host_eight_tiles_per_cta(native, oracle, nsm):
    """u8 host submit, K = 800, taps = K, 16 channels, 8 streams: 8 tiles per CTA, the last CTA running fewer tiles
    than the others and ending in a partial tile; every channel bit-exact to orc_channelize_dft8, and the envelope the
    same as the stream's in submits that run one tile per CTA."""
    K, taps, nch, S = 800, 800, 16, 8
    T = wb_rows_per_tile(K)
    # the fewest blocks at 8 tiles per CTA whose last CTA is short and ends in a partial tile (13 at 132 SMs: 96 rows
    # per CTA, the last CTA 64 rows, its 6th tile 4 rows long)
    nblk = next(n for n in range(1, 256) if wb_tiles_per_cta(K, n * 1024, S, nch, nsm) == 8 and n * 1024 % (8 * T) % T)
    small = tpc1_rows(K, S, nch, nsm) // 1024
    assert small >= 1 and wb_tiles_per_cta(K, small * 1024, S, nch, nsm) == 1
    fs = [freqs_for(K, nch, s) for s in range(S)]
    bb = 2048 * K
    x = np.random.default_rng(800).integers(0, 256, size=(S, nblk * bb), dtype=np.uint8)

    def run(pieces):
        with api.Context(K, S, nch, nblk, flags=FLAG_WB, taps=taps) as ctx:
            for s in range(S):
                ctx.set_plan_at(s, fs[s], FC)
            env, p = [], 0
            for n in pieces:
                ctx.submit_host(np.ascontiguousarray(x[:, p * bb:(p + n) * bb]), n)
                env.append(ctx.read_dm(n * 1024))
                p += n
            ctx.sync()
            assert ctx.stats().fast_chan_launches == len(pieces)
        return np.concatenate(env, axis=1)

    got = run([nblk])
    check_streams(oracle, native, "u8", x, K, taps, fs, got, subset=False, padding=False)   # 4 channels per class
    pieces = [small] * (nblk // small) + ([nblk % small] if nblk % small else [])
    assert bits_equal(run(pieces), got)


@pytest.mark.gpu
def test_wb_u8_device_ring_pitch_several_tiles(native, oracle, nsm):
    """u8 device submit from a ring with a pitch, K = 1600, taps = 4K + 3, 300 channels (two channel tiles):
    2 <= tiles per CTA < 8, bit-exact to orc_channelize_ovl_fast, and the same envelope as one-tile-per-CTA submits."""
    K, taps, nch, S = 1600, 4 * 1600 + 3, 300, 2
    nblk = next(n for n in range(1, 64) if wb_tiles_per_cta(K, n * 1024, S, nch, nsm) >= 2)
    assert 2 <= wb_tiles_per_cta(K, nblk * 1024, S, nch, nsm) < 8
    small = tpc1_rows(K, S, nch, nsm) // 1024
    assert 1 <= small < nblk
    fs = [freqs_for(K, nch, s) for s in range(S)]
    bb = 2048 * K
    x = np.random.default_rng(1600).integers(0, 256, size=(S, nblk * bb), dtype=np.uint8)
    pitch = nblk * bb + 4096
    with api.Context(K, S, nch, nblk, flags=FLAG_WB, taps=taps) as ctx:
        for s in range(S):
            ctx.set_plan_at(s, fs[s], FC)
        d = ctx.device_alloc(S * pitch)
        staged = np.full((S, pitch), 0xA5, dtype=np.uint8)
        staged[:, :nblk * bb] = x
        ctx.copy_to_device(d, staged)
        del staged
        ctx.submit_device(d, nblk, pitch)
        got = ctx.read_dm(nblk * 1024)
        ctx.sync()
        ctx.device_free(d)
        assert ctx.stats().fast_chan_launches == 1
    check_streams(oracle, native, "u8", x, K, taps, fs, got)
    with api.Context(K, S, nch, small, flags=FLAG_WB, taps=taps) as ctx:
        for s in range(S):
            ctx.set_plan_at(s, fs[s], FC)
        env = []
        for b0 in range(0, nblk, small):
            n = min(small, nblk - b0)
            ctx.submit_host(np.ascontiguousarray(x[:, b0 * bb:(b0 + n) * bb]), n)
            env.append(ctx.read_dm(n * 1024))
        ctx.sync()
    assert bits_equal(np.concatenate(env, axis=1), got)


def cs16_case(native, oracle, nsm, K, taps, nch, variant, planar, want_tpc, tail_rows, padding):
    """CS16 through one submit that runs want_tpc(tpc) tiles per CTA and a ragged tail, against the definition and
    against submits that each run one tile per CTA"""
    S = 2
    T = wb_rows_per_tile(K)
    big = T
    while not want_tpc(wb_tiles_per_cta(K, big, S, nch, nsm)):
        big += T
    cuts = [(big + 5) * K + 37, tail_rows * K + K // 3]
    n = sum(cuts)
    assert want_tpc(wb_tiles_per_cta(K, n // K - tail_rows, S, nch, nsm))
    fs = [freqs_for(K, nch, s) for s in range(S)]
    x = np.random.default_rng(K + taps + variant).integers(-32768, 32768, size=(S, n, 2), dtype=np.int16)
    maxb = -(-(n // K) // 1024)

    def run(pieces):
        with api.Context(K, S, nch, maxb, flags=FLAG_CS16 | FLAG_WB, taps=taps) as ctx:
            for s in range(S):
                ctx.set_plan_cs16(s, fs[s], variant, FC)
            env = run_stream_kind(ctx, "cs16", x, pieces, planar=planar)
            assert ctx.stats().fast_chan_launches >= len(pieces) - 1
        return env

    got = run(cuts)
    assert got.shape[1] == n // K
    check_streams(oracle, native, "cs16", x, K, taps, fs, got, variant, padding=padding)
    r1 = tpc1_rows(K, S, nch, nsm)
    assert wb_tiles_per_cta(K, r1, S, nch, nsm) == 1
    step = (r1 - 1) * K + K // 2 + 3                 # at most r1 rows per submit, carries a partial row
    pieces = [step] * (n // step) + ([n % step] if n % step else [])
    assert bits_equal(run(pieces), got)


@pytest.mark.gpu
def test_wb_cs16_interleaved_four_tiles_per_cta(native, oracle, nsm):
    """CS16 interleaved, variant 1, K = 2048 (8-row tiles), taps = 2K, 300 channels: a big submit at 4 or more tiles
    per CTA, then a ragged tail."""
    cs16_case(native, oracle, nsm, 2048, 2 * 2048, 300, 1, False, lambda t: t >= 4, 29, True)


@pytest.mark.gpu
def test_wb_cs16_planar_largest_12_row_tile(native, oracle, nsm):
    """CS16 planar, variant 0, K = 1808 (the largest K with 12-row tiles), taps = K + 8, 64 channels: 2 or more tiles
    per CTA."""
    assert wb_rows_per_tile(1808) == 12
    cs16_case(native, oracle, nsm, 1808, 1808 + 8, 64, 0, True, lambda t: t >= 2, 3, False)


# ------------------------------------------------------------------ B. block FEC beyond one grid pass

@pytest.mark.gpu
def test_block_fec_beyond_one_grid_pass(native, oracle, nsm):
    """acb_block_fec_batch on 2 grid passes + 1 234 frames, frame i = pool[i % 6007] (prime: every case lands in many
    thread, CTA and pass positions): keep / drop, len, err and the repaired text equal the restatement's blk_thread."""
    P = 6007
    n = 2 * fec_threads(nsm) + 1234
    pool = np.zeros(P, dtype=api.MSG_DTYPE)
    want_keep = np.zeros(P, dtype=bool)
    want_err = np.zeros(P, dtype=np.int32)
    want_txt = np.zeros((P, api.TXTMAX), dtype=np.uint8)
    for i, (chn, txt, crc) in enumerate(_fec_cases(np.random.default_rng(2779), P)):
        pool["chn"][i], pool["len"][i] = chn, len(txt)
        pool["txt"][i, :len(txt)] = np.frombuffer(txt, np.uint8)
        pool["crc"][i] = np.frombuffer(crc, np.uint8)
        o = refs.Msg()
        o.chn, o.len = chn, len(txt)
        o.txt[:len(txt)] = txt
        o.crc[:] = crc
        w = oracle.fec(o)
        if w is not None:
            want_keep[i], want_err[i] = True, w.err
            want_txt[i, :w.len] = np.frombuffer(bytes(w.txt[:w.len]), np.uint8)
    idx = np.arange(n) % P
    msgs = pool[idx]
    keep = np.zeros(n, dtype=np.int32)
    with api.Context(160, 1, 1, 1) as ctx:
        kept = native.acb_block_fec_batch(ctx.h, msgs.ctypes.data_as(C.POINTER(api.Msg)), n, keep.ctypes.data_as(C.POINTER(C.c_int)))
    keep = keep.astype(bool)
    assert kept == int(keep.sum())
    assert np.array_equal(keep, want_keep[idx])
    assert np.array_equal(msgs["len"], pool["len"][idx])
    assert np.array_equal(msgs["err"][keep], want_err[idx][keep])
    inside = np.arange(api.TXTMAX)[None, :] < msgs["len"][keep][:, None]
    assert np.array_equal(np.where(inside, msgs["txt"][keep], 0), want_txt[idx][keep])
    assert want_keep.sum() > 1000 and (want_err[want_keep] > 0).sum() > 200 and (~want_keep).sum() > 1000


# ------------------------------------------------------------------ C. demodulator at the chain counts where the context picks the lanes

DM_K, DM_FM, DM_BLOCKS, NCH = 16, tuple(131.475 + 0.025 * i for i in range(6)), 12, 13
P_COLS = 37                         # coprime with 32: every column lands in every lane position
FLIPS = [[(3, 0x04)], [(5, 0x01), (9, 0x80)], [(-2, 0x10)], [(1, 0x40), (-3, 0x02)], [(2, 1), (4, 2), (6, 4), (8, 8)],
         [(7, 0x21)], [(0, 0x08), (10, 0x08), (11, 0x08)]]


@pytest.fixture(scope="module")
def dm_pool(native, oracle):
    """(37, 12 * 1024) envelope columns: the oracle's channelizer on dense synthetic K = 16 captures (6 channels, short
    frames back to back), every third frame corrupted (repairable, double-bit, BCS and hopeless errors)"""
    _, _, fc = api.plan(DM_K, DM_FM)
    wf = oracle.wf(DM_K, DM_FM)
    cols = []
    for cap in range(-(-P_COLS // len(DM_FM))):
        plan = synth.make_plan(DM_K, DM_FM, fc, seconds=DM_BLOCKS * 1024 / 12500, seed=300 + cap, msgs_per_chan_per_sec=100.0,
                               text_len=(1, 6))
        for i, b in enumerate(plan.bursts):
            if i % 3 == 0:
                b.frame = synth.corrupt_frame(b.frame, FLIPS[(i // 3) % len(FLIPS)])
        cols.extend(oracle.channelize(synth.render_blocks(plan, 0, DM_BLOCKS).reshape(-1), DM_K, wf))
    return np.ascontiguousarray(np.stack(cols[:P_COLS]))


def oracle_column(oracle, col, cuts):
    """the restatement over one column in the given submits: (pre-FEC frames per submit, the frames each submit
    delivers as msg_tuple without chn, the final state)"""
    ch, sink = oracle.new_chan(0), refs.Sink()
    raw, want, p = [], [], 0
    for n in cuts:
        before = sink.c.nmsg
        oracle.demod(ch, col[p:p + n], sink)
        p += n
        raw.append(sink.c.nmsg - before)
        fixed = (oracle.fec(m) for m in sink.msgs()[before:])
        want.append([msg_tuple(f)[1:] for f in fixed if f is not None])
    return raw, want, ch.vec()


def device_frames(rec):
    """(chain index stream * NCH + chn, msg_tuple without chn) of drained records, in emission order"""
    g = rec["stream"].astype(np.int64) * NCH + rec["chn"]
    lvl = rec["lvl"].view(np.uint32)
    return g, [(int(rec["len"][i]), int(rec["err"][i]), rec["txt"][i, :rec["len"][i]].tobytes(), rec["crc"][i].tobytes(), int(lvl[i]))
               for i in range(len(rec))]


def chain_sizes(lanes, nsm, raw1):
    """streams of NCH chains for which the context picks `lanes`; at one lane also enough pre-FEC frames in the first
    submit for k_block_fec to need more than one grid pass"""
    lo = 32 * 4 * nsm // min(lanes, 4)              # the fewest chains at `lanes`; 8 lanes below the 4-lane bound
    if lanes == 8:
        nchains = lo * 3 // 4
    elif lanes > 1:
        nchains = lo + lo // 4
    else:
        per = raw1[np.arange(4 * lo) % P_COLS].cumsum()
        nchains = max(lo, int(np.searchsorted(per, fec_threads(nsm) + 1000)) + 1)
    return -(-nchains // NCH)


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", [1, 2, 4, 8])
def test_demod_lanes_chosen_by_context(native, oracle, nsm, dm_pool, lanes, monkeypatch):
    """acb_submit_dm_host at chain counts where acb_create picks 1, 2, 4 and 8 lanes by itself, 13 channels per stream
    (streams straddle warps irregularly), chain g fed column g % 37, two submits ending mid-bit: every chain's frames
    (lvl bits included) and its whole state equal the restatement's run of its column, frames come out per submit in
    (stream, channel, time) order, no frame is lost and raw = delivered + dropped.  At one lane the first submit
    carries more frames than one k_block_fec grid pass and goes through the consumer's helper threads."""
    monkeypatch.delenv("ACB_DEMOD_LANES", raising=False)
    cuts = [10 * 1024 + 517, 1111] if lanes == 1 else [2 * 1024 + 517, 1024 + 333]
    assert sum(cuts) <= dm_pool.shape[1]
    ref = [oracle_column(oracle, col, cuts) for col in dm_pool]
    raw1 = np.array([r[0][0] for r in ref])
    nstreams = chain_sizes(lanes, nsm, raw1)
    nchains = nstreams * NCH
    assert demod_lanes(nchains, nsm) == lanes
    col_of = np.arange(nchains) % P_COLS
    raw_want = [int(np.array([r[0][i] for r in ref])[col_of].sum()) for i in range(len(cuts))]
    if lanes == 1:
        assert raw_want[0] > fec_threads(nsm) and raw_want[0] >= 8192
    states = [None] * nchains
    with api.Context(DM_K, nstreams, NCH, -(-max(cuts) // 1024), flags=FLAG_NO_STAGING) as ctx:
        p = 0
        for i, n in enumerate(cuts):
            dm = np.empty((nstreams, n, NCH), dtype=np.float32)
            for c in range(NCH):
                dm[:, :, c] = dm_pool[(np.arange(nstreams) * NCH + c) % P_COLS, p:p + n]
            ctx.submit_dm(dm)
            del dm
            p += n
            ctx.sync()
            st = ctx.stats()
            g, got = device_frames(ctx.drain_records())
            assert st.raw_frames == sum(raw_want[:i + 1]) and st.frames_lost == 0
            if lanes == 1 and i == 0:
                assert st.raw_frames > fec_threads(nsm)
            assert np.all(np.diff(g) >= 0)               # (stream, channel) order; time order within a chain below
            bounds = np.searchsorted(g, np.arange(nchains + 1))
            for ch in range(nchains):
                mine = got[bounds[ch]:bounds[ch + 1]]
                assert mine == ref[col_of[ch]][1][i], (i, ch)
            delivered = len(got) if i == 0 else delivered + len(got)
        dropped_want = sum(raw_want) - sum(len(r[1][i]) for i in range(len(cuts)) for r in (ref[j] for j in col_of))
        assert st.raw_frames == delivered + st.fec_dropped and st.fec_dropped == dropped_want and delivered > 0
        for ch in range(nchains):
            states[ch] = ctx.get_state(ch // NCH, ch % NCH).vec()
    for ch in range(nchains):
        assert states[ch] == ref[col_of[ch]][2], ch


# ------------------------------------------------------------------ D. the stream-count limit

def test_stream_count_over_grid_limit_refused(native):
    """65 536 streams and more: ACB_ERR_ARG from acb_create before any device query, and from acb_multi_create when a
    part would get more than 65 535 (a channel split gives every part every stream)."""
    for n in (65536, 2**31 - 1):
        cfg = api.Config(0, 8, n, 1, 1, 0, 0)
        h = C.c_void_p()
        assert native.acb_create(C.byref(cfg), C.byref(h)) == ACB_ERR_ARG and not h
        assert b"exceeds 65535" in native.acb_last_error()
    for ndev, mode in ((1, 0), (2, 1)):
        cfg = api.Config(0, 8, 65536, 2, 1, 0, 0)
        dev = np.zeros(ndev, dtype=np.int32)
        h = C.c_void_p()
        assert native.acb_multi_create(C.byref(cfg), dev.ctypes.data, ndev, mode, C.byref(h)) == ACB_ERR_ARG
        native.acb_multi_destroy(h)


@pytest.mark.gpu
def test_largest_stream_count(native, oracle):
    """65 535 streams (grid.y at its limit), K = 8, one channel, one block, device submit without input staging
    (about 2 GB of device memory): streams 0, 32 767 and 65 534 bit-exact to the oracle's channelizer."""
    K, S, fm = 8, 65535, (131.525,)
    fd, _, _ = api.plan(K, fm)
    bb, chunk = 2048 * K, 4096
    check = (0, S // 2, S - 1)
    kept = {}
    with api.Context(K, S, 1, 1, flags=FLAG_NO_STAGING) as ctx:
        for s in range(S):
            ctx.set_plan(s, fd)
        d = ctx.device_alloc(S * bb)
        for s0 in range(0, S, chunk):
            x = np.random.default_rng([S, s0]).integers(0, 256, size=(min(chunk, S - s0), bb), dtype=np.uint8)
            ctx.copy_to_device(d + s0 * bb, x)
            kept.update({s: x[s - s0].copy() for s in check if s0 <= s < s0 + len(x)})
        ctx.submit_device(d, 1, bb)
        got = ctx.read_dm(1024)
        ctx.sync()
        ctx.device_free(d)
        assert ctx.stats().chan_launches == 1
    wf = oracle.wf(K, fm)
    for s in check:
        assert bits_equal(got[s], oracle.channelize(kept[s], K, wf).T.copy()), s
