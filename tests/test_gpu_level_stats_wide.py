"""Input and envelope levels (ACB_FLAG_LEVEL_STATS) at the shapes the large deployments run, against the scalable float64
definition (tests/level_stats_wide_refs.py): counts, rows, windows and peaks exact, sums and floor within 1e-10.

Each case asserts the launch geometry it is there for, restated below from kernels.cu (launch_level_input_t,
launch_level_dm): k_level_dm's channel tile (ct channels per CTA, gridDim.z tiles, a partial last tile), k_level_in's
chunks per stream and whether a stream's bytes end inside a 16-byte load (the scalar tail), and how many CTAs the two
final passes run.  A later change of a constant then moves the shapes, or fails the case, instead of leaving it covering
nothing.

NaN and Inf inputs are out of scope: the tables are defined for finite samples only."""
import zlib

import numpy as np
import pytest

import level_stats_wide_refs as wr
from acarsdec_b200 import api
from test_wideband_real_oracle import air_freqs

pytestmark = pytest.mark.gpu

LEVEL = api.FLAG_LEVEL_STATS
FLAG_NO_STAGING, FLAG_REAL, FLAG_CS16 = 1, 2, 4
FW, FWR = api.FLAG_FAST_WIDEBAND, api.FLAG_FAST_WIDEBAND_REAL
OUTBLK = 1024

# ------------------------------------------------------------------ the launchers' arithmetic, restated

LVL_CHUNK = 256 * 16 * 8            # acb_internal.h: input bytes per k_level_in CTA


def sample_bytes(kind):
    return 2 if kind == "u8" else 4


def level_ct(nch):
    """launch_level_dm: channels per tile, the channel count rounded up to a power of two, at most 32"""
    ct = 1
    while ct < nch and ct < 32:
        ct *= 2
    return ct


def level_tiles(nch):
    """launch_level_dm: gridDim.z of k_level_dm"""
    return -(-nch // level_ct(nch))


def in_chunks(kind, rows, K):
    """k_level_in CTAs (and k_level_in_fin partials) of one stream of `rows` rows"""
    return -(-rows * K * sample_bytes(kind) // LVL_CHUNK)


def in_fin_ctas(nstreams):
    """launch_level_input_t: k_level_in_fin, one warp per stream, 256 threads per CTA"""
    return -(-nstreams * 32 // 256)


def dm_fin_ctas(nstreams, nch):
    """launch_level_dm: k_level_dm_fin, one thread per chain, 256 per CTA"""
    return -(-nstreams * nch // 256)


def test_restated_arithmetic():
    assert [level_ct(n) for n in (1, 2, 3, 5, 8, 13, 31, 32, 33, 64, 255, 256, 300)] == \
        [1, 2, 4, 8, 8, 16, 32, 32, 32, 32, 32, 32, 32]
    assert [level_tiles(n) for n in (1, 31, 32, 33, 64, 255, 256, 300)] == [1, 1, 1, 2, 2, 8, 8, 10]
    assert in_chunks("u8", 3 * 1024, 160) == 30 and in_chunks("u8", 2 * 1024, 1600) == 200
    assert (in_fin_ctas(3), in_fin_ctas(8), in_fin_ctas(9), in_fin_ctas(300)) == (1, 1, 2, 38)
    assert (dm_fin_ctas(3, 4), dm_fin_ctas(300, 13)) == (1, 16)


# ------------------------------------------------------------------ contexts, signals and submits

def wide_freqs(kind, K, nch):
    """nch channels 25 kHz apart (real input: spread over the real band), inside one tuner band at K.  Below 2^27 Hz, where
    float32 holds every multiple of 8 Hz, so that the IQ fast plans (whole numbers of 12.5 kHz from Fc) apply"""
    if kind == "real":
        return air_freqs(K, nch)
    return [120_000_000 + 25_000 * i for i in range(nch)]


def make(kind, K, S, nch, max_blocks, flags=0, taps=0, multi=None):
    """a context (or, multi = devices, a channel split) of S streams planned on wide_freqs"""
    kf = FLAG_REAL if kind == "real" else FLAG_CS16 if kind in ("cs16", "planar") else 0
    fd = wide_freqs(kind, K, nch)
    if multi is None:
        ctx = api.Context(K, S, nch, max_blocks, flags=LEVEL | flags | kf, taps=taps)
    else:
        ctx = api.MultiContext(K, S, nch, max_blocks, multi, mode=1, flags=LEVEL | flags | kf, taps=taps)
    for s in range(S):
        if kind == "u8":
            ctx.set_plan(s, fd)
        elif kind == "real":
            ctx.set_plan_air(s, fd)
        else:
            ctx.set_plan_cs16(s, fd, 1 if kind == "planar" else 0)
    return ctx


class Dev:
    """device copies of submits' inputs, kept until the end of the test (the input lifetime rule)"""

    def __init__(self):
        self.keep = []

    def put(self, a):
        import torch
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self.keep.append(t)
        return t


def submit(ctx, kind, K, parts, counts, dev, store):
    """one ragged submit (parts[s]: u8 bytes of counts[s] blocks, CS16 (counts[s], 2), real (counts[s],)); returns each
    stream's new rows"""
    S = len(parts)
    if kind == "u8":
        w = max(counts) * OUTBLK * K * 2 + 48
        buf = np.zeros((S, w), np.uint8)
        for s, p in enumerate(parts):
            buf[s, :len(p)] = p
        nblk = np.asarray(counts, np.int32)
        if dev:
            ctx.submit_device(store.put(buf).data_ptr(), 0, w, counts=nblk)
        else:
            ctx.submit_host(buf, counts=nblk)
        return nblk.astype(np.int64) * OUTBLK
    w = max(counts) + 3
    buf = np.zeros((S, w), np.float32) if kind == "real" else np.zeros((S, w, 2), np.int16)
    for s, p in enumerate(parts):
        buf[s, :len(p)] = p
    if dev:
        if kind == "planar":
            return ctx.submit_tensor(store.put(buf[..., 0]), store.put(buf[..., 1]), counts=counts)
        return ctx.submit_tensor(store.put(buf), counts=counts)
    if kind == "real":
        return ctx.submit_real(buf, counts=counts)
    if kind == "cs16":
        return ctx.submit_cs16(buf, counts=counts)
    return ctx.submit_cs16_planar(np.ascontiguousarray(buf[..., 0]), np.ascontiguousarray(buf[..., 1]), counts=counts)


class Pool:
    """random input cut from one pool, each stream at its own offset (cheap at hundreds of streams)"""

    def __init__(self, kind, S, count, seed):
        n = 2 * (S * 7919 + count)                  # count: the most one stream takes in one submit
        rng = np.random.default_rng(seed)
        self.kind = kind
        if kind == "u8":
            self.x = rng.integers(0, 256, size=n, dtype=np.uint8)
        elif kind == "real":
            self.x = (rng.standard_normal(n) * 0.3).astype(np.float32)
            self.x[rng.random(n) < 1e-4] = np.float32(-1.0)         # some full-scale samples
        else:
            self.x = rng.integers(-12000, 12000, size=(n, 2), dtype=np.int16)
            self.x[rng.random(n) < 1e-4, 0] = -32768
        self.n = n

    def take(self, s, off, count):
        o = (s * 7919 + off) % (self.n // 2)
        assert o + count <= self.n
        return self.x[o:o + count]


class Run:
    """a context fed ragged submits (host and device alternating) and the definition following every stream"""

    def __init__(self, ctx, kind, K, S, nch, pool, chan_refs=True):
        self.ctx, self.kind, self.K, self.S, self.pool = ctx, kind, K, S, pool
        self.inp = [wr.InputLevels("u8" if kind == "u8" else "cs16" if kind == "planar" else kind, K) for _ in range(S)]
        self.ch = [wr.ChanLevels(nch) for _ in range(S)] if chan_refs else None
        self.off = [0] * S
        self.store = Dev()
        self.i = 0
        self.rows = []                              # per submit, each stream's rows

    def submit(self, counts, parts=None):
        u = OUTBLK * self.K * 2 if self.kind == "u8" else 1
        if parts is None:
            parts = [self.pool.take(s, self.off[s], counts[s] * u) for s in range(self.S)]
        rows = submit(self.ctx, self.kind, self.K, parts, counts, self.i % 2 == 1, self.store)
        dm = self.ctx.read_dm(int(max(rows))) if self.ch is not None and max(rows) else None
        for s in range(self.S):
            assert self.inp[s].feed(parts[s]) == rows[s], (s, rows[s])
            if dm is not None:
                self.ch[s].feed(dm[s, :int(rows[s])])
            self.off[s] += counts[s] * u
        self.rows.append(np.asarray(rows, np.int64))
        self.i += 1
        return rows

    def check(self):
        self.ctx.sync()
        inp, ch = self.ctx.level_stats()
        wr.check_inputs(inp, self.inp)
        if self.ch is not None:
            wr.check_chans(ch, self.ch)
        return inp, ch


def chunk_counts(run):
    """k_level_in chunks of every stream in every submit that gave it rows"""
    return [in_chunks(run.kind, int(r), run.K) for rows in run.rows for r in rows if r]


# ------------------------------------------------------------------ k_level_dm's channel tiles, on envelope input

TILES = [(1, 1, 1, False), (2, 2, 1, False), (3, 4, 1, True), (5, 8, 1, True), (8, 8, 1, False), (13, 16, 1, True),
         (31, 32, 1, True), (32, 32, 1, False), (33, 32, 2, True), (64, 32, 2, False), (255, 32, 8, True), (256, 32, 8, False),
         (300, 32, 10, True)]
ENV_SCHED = [1023, 1, 700, 8 * OUTBLK, 1, 1023, 5 * OUTBLK + 17, 8 * OUTBLK]


def test_tile_cases_cover_every_tile_shape():
    assert {ct for _, ct, _, _ in TILES} == {1, 2, 4, 8, 16, 32}
    assert {p for *_, p in TILES} == {True, False} and max(t for _, _, t, _ in TILES) == 10


@pytest.mark.parametrize("nch,ct,tiles,partial", TILES)
def test_channel_tiles(nch, ct, tiles, partial):
    """Envelope input (no channelizer) at max_blocks = 8: 1023 rows left open then 1 row, 8 * 1024 rows on top of an open
    window, windows straddling every submit.  Every channel and window has its own scale, so a tile offset or a swapped
    channel changes the result, and the lowest window of each chain is a different one."""
    assert (level_ct(nch), level_tiles(nch), nch % level_ct(nch) != 0) == (ct, tiles, partial)
    S = 3
    rng = np.random.default_rng(nch)
    ch = [wr.ChanLevels(nch) for _ in range(S)]
    pos = 0
    with api.Context(160, S, nch, 8, flags=LEVEL | FLAG_NO_STAGING) as ctx:
        for n in ENV_SCHED:
            r = pos + np.arange(n)
            w = r // OUTBLK                                  # the window each row falls in
            c = np.arange(nch)
            scale = np.exp2(((w[:, None] * 5 + c[None, :] * 3) % 23 - 11).astype(np.float64))
            dm = np.stack([(rng.random((n, nch)) * scale * (1 + s)).astype(np.float32) for s in range(S)])
            ctx.submit_dm(dm)
            for s in range(S):
                ch[s].feed(dm[s])
            pos += n
        ctx.sync()
        inp, got = ctx.level_stats()
    assert not inp["samples"].any()
    last = ch[S - 1]
    assert last.windows == pos // OUTBLK and last.floor[nch - 1] > 0
    # the floors come from different windows on neighbouring channels: a channel swap cannot hide
    assert nch == 1 or len(np.unique(ch[0].floor)) > 1
    wr.check_chans(got, ch)


# ------------------------------------------------------------------ through the channelizer at wide shapes

WIDE = [("u8", 1600, 300, 0), ("u8", 1600, 300, FW), ("cs16", 2048, 256, FW), ("real", 1608, 300, FWR)]


@pytest.mark.parametrize("kind,K,nch,form", WIDE)
@pytest.mark.parametrize("taps", ["K", "long"])
def test_wide_channelizer(kind, K, nch, form, taps):
    """Ragged submits (a stream sitting one out), host and device alternating: every stream of the input table, every
    chain of the channel table; the input spans well over 32 chunks per stream"""
    S, max_blocks = 3, 2
    rng = np.random.default_rng(zlib.crc32(f"{kind}{K}{nch}{form}{taps}".encode()))
    if kind == "u8":
        sched = [[2, 1, 0], [1, 2, 2], [0, 2, 1], [2, 2, 2]]
    else:
        top = max_blocks * OUTBLK * K - K
        sched = [[top, 1024 * K + 5, 0], [int(rng.integers(3, K)), top - 3 * K, top], [top, 0, 1500 * K + 11],
                 [int(rng.integers(1200 * K, top)) for _ in range(S)]]
    pool = Pool(kind, S, max_blocks * OUTBLK * K * 2, rng.integers(1 << 30))
    with make(kind, K, S, nch, max_blocks, form, 2 * K + 3 if taps == "long" else 0) as ctx:
        run = Run(ctx, kind, K, S, nch, pool)
        for c in sched:
            run.submit(c)
        run.check()
        assert ctx.stats().fast_chan_launches == (ctx.stats().chan_launches if form else 0)
    n = chunk_counts(run)
    assert max(n) > 64 and any(k % 32 for k in n), n
    assert level_ct(nch) == 32 and level_tiles(nch) >= 8
    assert min(r.windows for r in run.ch) > 0


# ------------------------------------------------------------------ hundreds of streams: several final-pass CTAs

@pytest.mark.parametrize("kind", ["u8", "real"])
def test_many_streams(kind):
    """300 streams x 13 channels, ragged counts with zeros: both final passes run several CTAs and a partial last one,
    and streams' chains straddle k_level_dm_fin's CTAs"""
    S, nch = 300, 13
    K = 160 if kind == "u8" else 200
    max_blocks = 2
    assert in_fin_ctas(S) > 1 and S % 8 != 0                    # a partial last k_level_in_fin CTA
    assert dm_fin_ctas(S, nch) > 1 and (S * nch) % 256 != 0      # and k_level_dm_fin's
    assert any((s * nch) // 256 != ((s + 1) * nch - 1) // 256 for s in range(S))
    rng = np.random.default_rng(300 + len(kind))
    sched = []
    for i in range(4):
        if kind == "u8":
            c = rng.integers(0, max_blocks + 1, size=S)
        else:
            c = rng.integers(0, max_blocks * OUTBLK * K - K, size=S)
            c[rng.random(S) < 0.1] = 0
        c[-4:] = c[-4:].clip(min=1) if i != 1 else 0                # the last CTA's streams: rows in 3 of the 4 submits
        sched.append([int(x) for x in c])
    u = OUTBLK * K * 2 if kind == "u8" else 1
    pool = Pool(kind, S, max_blocks * OUTBLK * K * 2, 5)
    with make(kind, K, S, nch, max_blocks) as ctx:
        run = Run(ctx, kind, K, S, nch, pool)
        for c in sched:
            run.submit(c)
        run.check()
    assert run.inp[-1].samples > 0 and run.ch[-1].windows > 0
    assert any(r == 0 for rows in run.rows for r in rows)


# ------------------------------------------------------------------ the scalar tail: bytes that end inside a 16-byte load

@pytest.mark.parametrize("kind", ["cs16", "planar", "real"])
@pytest.mark.parametrize("K", [161, 162])
def test_scalar_tail(kind, K):
    """K odd (rows * K * 4 mod 16 is 4, 8 or 12 as rows mod 4 is not 0) and K = 2 mod 4 (8 at odd rows); the streams of
    one ragged submit end aligned and unaligned side by side"""
    S, nch, max_blocks = 4, 4, 2
    rng = np.random.default_rng(K * 10 + len(kind))
    sched = [[int(x) for x in rng.integers(1, max_blocks * OUTBLK * K - K, size=S)] for _ in range(6)]
    sched[2][1] = 0
    sched[3] = [7 * K, 9 * K + 3, 1024 * K, 2 * K]
    pool = Pool(kind, S, max_blocks * OUTBLK * K, K)
    with make(kind, K, S, nch, max_blocks) as ctx:
        run = Run(ctx, kind, K, S, nch, pool)
        for c in sched:
            run.submit(c)
        run.check()
    tails = [[int(r) * K * 4 % 16 for r in rows if r] for rows in run.rows]
    seen = {t for ts in tails for t in ts}
    assert seen - {0} == ({4, 8, 12} if K % 2 else {8}), tails
    assert any(0 in ts and len(set(ts)) > 1 for ts in tails), tails      # aligned and unaligned streams in one submit


# ------------------------------------------------------------------ extreme codes

def _fill(kind, S, n, values, rng):
    out = []
    for s in range(S):
        v = values[s % len(values)]
        if kind == "u8":
            out.append(np.full(n, v, np.uint8))
        elif kind == "cs16":
            out.append(np.full((n, 2), v, np.int16))
        else:
            out.append(((1.0 + rng.random(n)) * np.where(rng.random(n) < 0.5, -1.0, 1.0) * v).astype(np.float32))
    return out


@pytest.mark.parametrize("kind,values", [("u8", (0, 255, 127, 128)), ("cs16", (-32768,)), ("real", (2.0 ** -60, 2.0 ** 60))])
def test_extreme_codes(kind, values):
    """Whole chunks of one code: u8 0, 255, 127 and 128 (both signs of the 127.37f offset, and the cancellation in
    k_level_in_fin's integer formula), CS16 -32768 (each thread's (unsigned)(i*i) + (unsigned)(q*q) reaches 2^31), real
    samples scaled by 2^-60 and 2^60.  Where every sample is at full scale, every sample counts as clipped."""
    S, nch, max_blocks = 4, 4, 2
    K = 160 if kind != "real" else 200
    rng = np.random.default_rng(len(values))
    u = OUTBLK * K * 2 if kind == "u8" else 1
    sched = [[2, 1, 2, 1], [1, 2, 0, 2]] if kind == "u8" else [[2 * OUTBLK * K - K, OUTBLK * K + 7, 5 * K, 2000 * K],
                                                                  [OUTBLK * K - 3, 0, 2 * OUTBLK * K - 2 * K, 33]]
    tot = [sum(c[s] for c in sched) * u for s in range(S)]
    sig = _fill(kind, S, max(tot), values, rng)
    with make(kind, K, S, nch, max_blocks) as ctx:
        run = Run(ctx, kind, K, S, nch, None, chan_refs=False)
        off = [0] * S
        for c in sched:
            run.submit(c, parts=[sig[s][off[s]:off[s] + c[s] * u] for s in range(S)])
            off = [off[s] + c[s] * u for s in range(S)]
        ctx.sync()
        inp, _ = ctx.level_stats()
    wr.check_inputs(inp, run.inp)
    assert min(chunk_counts(run)) >= 1 and max(chunk_counts(run)) >= 8       # whole chunks of the one code
    for s in range(S):
        v = values[s % len(values)]
        full = {"u8": v in (0, 255), "cs16": True, "real": v > 1}[kind]
        assert inp[s]["samples"] > 0
        assert (inp[s]["clipped"] == inp[s]["samples"]) == full, (s, inp[s])
        if not full:
            assert inp[s]["clipped"] == 0
    if kind == "cs16":
        assert all(float(inp[s]["power_sum"]) == inp[s]["samples"] * 2.0 ** 31 for s in range(S))


# ------------------------------------------------------------------ a channel split that cuts channel tiles

def test_channel_split_levels():
    """300 channels over 3 parts (100 each, every part's last tile partial, boundaries inside the single context's
    tiles): the input table equal to the single context's byte for byte, the channel table's rows, windows and peak
    equal and its sums within 1e-10; the single context against the definition"""
    kind, K, nch, S, max_blocks = "u8", 1600, 300, 2, 2
    assert level_tiles(100) == 4 and 100 % level_ct(100) and 100 % 32 and 200 % 32
    sched = [[2, 1], [1, 2], [2, 0], [1, 1]]
    pool = Pool(kind, S, max_blocks * OUTBLK * K * 2, 17)
    with make(kind, K, S, nch, max_blocks, FW) as one, make(kind, K, S, nch, max_blocks, FW, multi=[0, 0, 0]) as m:
        assert m.parts() == 3
        run = Run(one, kind, K, S, nch, pool)
        off = [0] * S
        u = OUTBLK * K * 2
        for c in sched:
            parts = [pool.take(s, off[s], c[s] * u) for s in range(S)]
            run.submit(c, parts=parts)
            buf = np.zeros((S, max(c) * u), np.uint8)
            for s in range(S):
                buf[s, :len(parts[s])] = parts[s]
            m.submit_host(buf, counts=c)
            off = [off[s] + c[s] * u for s in range(S)]
        i1, c1 = run.check()
        m.sync()
        im, cm = m.level_stats()
    assert i1.tobytes() == im.tobytes()
    for f in ("rows", "windows", "peak"):
        assert np.array_equal(c1[f], cm[f]), f
    for f in ("power_sum", "floor"):
        assert np.allclose(cm[f], c1[f], rtol=1e-10, atol=0), f
    assert c1["windows"].min() > 0
