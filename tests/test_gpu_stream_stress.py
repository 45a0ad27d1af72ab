"""Pipeline stress of the streaming front-ends (acb_submit_real_host, acb_submit_cs16_host, acb_submit_cs16_planar_host):
one seeded random walk per case, with up to three submits in flight and held to the CPU definitions throughout.

- Submit sizes: 1 sample, below and exactly up to the next row, whole blocks, and the largest a submit may carry;
  planar submits grow past the first one, so the planar staging buffer is reallocated mid-stream.
- Between submits, at random: nothing (most often), acb_collect, acb_sync, drains, state round trips, acb_reset.
- A refused submit (one sample over the limit) changes nothing.
- Every source is overwritten as soon as the rule in acars_b200.h frees it.  Pageable sources are freed when the call
  returns.  In the pinned cases, a buffer is freed when an acb_collect / acb_sync covers its submit, and the buffer of
  a submit that produced no row only at the next acb_sync.

Messages are compared in global emission order with an independent restatement of that order.  Every chain's state is
compared at every sync, and the last submit's envelope bit for bit.  The expected side runs the definition of the
case's channelizer in lockstep: taps < K (fir_stream_oracle.c), taps = K and taps > K (the reference's arithmetic,
ovl_oracle.c) or a fast form's bit-exact restatement.  Its envelope goes through the oracle demodulator and block FEC."""
import collections
from dataclasses import dataclass

import numpy as np
import pytest

import fir_stream_refs as fsr
import ovl_fast_real_refs
import ovl_fast_refs
import ovl_refs
import refs
from acarsdec_b200 import api, synth
from common import bits_equal, msg_tuple
from test_ovl_fast_oracle import fast_plan
from test_ovl_fast_real_oracle import fast_plan_air

pytestmark = pytest.mark.gpu

FLAG_REAL, FLAG_CS16, FAST_CHANNELIZER, FAST_FILTER, FAST_FILTER_REAL, FAST_WIDEBAND = 2, 4, 8, 16, 32, 64
GROUP_SUBMIT, GROUP_OUTPUTS, GROUP_INPUT = 0, 1, 2
REAL_FM = (131.525, 131.5375, 131.55)                  # on the raster around the Fc acb_air_choose_fc picks
CS16_FM = synth.DEFAULT_FREQS_MHZ[:3]
S, MAXBLK, PAD = 3, 2, 29                              # streams, max_blocks, stream stride - samples of a submit


@dataclass
class Case:
    kind: str                  # "real", "cs16" (interleaved), "planar"
    filt: str                  # "lt": taps < K via acb_set_wf; "eq" / "gt": taps = K / taps > K via the planner
    flags: int = 0             # a fast form on top of the input kind
    group: tuple = (GROUP_SUBMIT, 0)    # (unit, period); an INPUT period "short" / "long" is K // 3 + 1 / 5 K + 7
    pinned: bool = False       # sources from rotating acb_host_alloc buffers


CASES = {
    "real-lt": Case("real", "lt", group=(GROUP_OUTPUTS, 512)),
    "real-eq": Case("real", "eq", group=(GROUP_INPUT, "short")),
    "real-gt-pinned": Case("real", "gt", group=(GROUP_INPUT, "long"), pinned=True),
    "real-eq-fast": Case("real", "eq", FAST_CHANNELIZER, group=(GROUP_OUTPUTS, 1024)),
    "real-gt-fast": Case("real", "gt", FAST_FILTER_REAL, group=(GROUP_SUBMIT, 0)),
    "cs16-lt": Case("cs16", "lt", group=(GROUP_INPUT, "long")),
    "cs16-eq": Case("cs16", "eq", group=(GROUP_SUBMIT, 0)),
    "cs16-gt": Case("cs16", "gt", group=(GROUP_OUTPUTS, 1024)),
    "cs16-eq-fast": Case("cs16", "eq", FAST_CHANNELIZER, group=(GROUP_INPUT, "short")),
    "cs16-gt-wideband": Case("cs16", "gt", FAST_WIDEBAND, group=(GROUP_OUTPUTS, 512)),
    "planar-lt-pinned": Case("planar", "lt", group=(GROUP_INPUT, "short"), pinned=True),
    "planar-eq": Case("planar", "eq", group=(GROUP_OUTPUTS, 512)),
    "planar-gt": Case("planar", "gt", group=(GROUP_SUBMIT, 0)),
    "planar-gt-fast": Case("planar", "gt", FAST_FILTER, group=(GROUP_INPUT, "long")),
}


def setup(case, oracle, nrows, seed):
    """(K, taps, nch, input (S, n[, 2]), plan(ctx), define(s, x) -> (nch, rows) envelope of the definition)."""
    real = case.kind == "real"
    K = 200 if real else 160
    rate = K * 12500
    taps = {"lt": 3 * K // 4 + 1, "eq": K, "gt": 2 * K + 3}[case.filt]
    fm = REAL_FM if real else CS16_FM
    variant = 0 if case.kind == "cs16" else 1          # soapy.c for interleaved, sdrplay.c for planar
    if real:
        fd, fc, _ = api.air_plan(rate, fm)
    else:
        fd, _, fc = api.plan(K, fm)
    n = nrows * K + K // 2
    xs = []
    for s in range(S):
        p = synth.make_plan(K, fm, fc, seconds=n / rate, seed=seed * 10 + s, msgs_per_chan_per_sec=4.0, text_len=(5, 30),
                            amp=(6.0, 12.0))
        if real:
            p = synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, bursts=p.bursts, seed=p.seed)
            xs.append(synth.render_real(p, 0, n))
        else:
            xs.append(synth.render_cs16(p, 0, n))
    x = np.stack(xs)
    nch = len(fm)
    if case.filt == "lt":
        base = api.build_wf_air(rate, fm) if real else api.build_wf_cs16(variant, K, fd, fc)
        wfs = [np.ascontiguousarray(np.roll(base, s, axis=0)[:, :2 * taps]) for s in range(S)]      # a table per stream

        def plan(ctx):
            for s in range(S):
                ctx.set_wf(s, wfs[s])
        fn = fsr.channelize_fir_real if real else fsr.channelize_fir_cs16
        return K, taps, nch, x, plan, lambda s, seg: fn(seg, K, wfs[s])

    def plan(ctx):
        for s in range(S):
            assert (ctx.set_plan_air(s, fd) if real else ctx.set_plan_cs16(s, fd, variant)) == fc
    if case.flags == 0:
        if real:
            wf = api.build_wf_air(rate, fm) if taps == K else api.build_wf_air_lp(rate, taps, fm)
            return K, taps, nch, x, plan, lambda s, seg: ovl_refs.channelize_ovl_real(seg, K, wf)
        wf = api.build_wf_cs16(variant, K, fd, fc) if taps == K else api.build_wf_cs16_lp(variant, K, taps, fd, fc)
        return K, taps, nch, x, plan, lambda s, seg: ovl_refs.channelize_ovl_cs16(seg, K, wf)
    if real:
        k, tw = fast_plan_air(K, fd, fc)
        if taps == K:
            return K, taps, nch, x, plan, lambda s, seg: oracle.channelize_rdft(seg, K, k, tw)
        h = api.build_lowpass(K, taps)
        return K, taps, nch, x, plan, lambda s, seg: ovl_fast_real_refs.channelize_ovl_rdft(oracle, seg, K, h, k, tw)
    k, tw = fast_plan("cs16", variant, K, fd, fc)
    if taps == K:
        return K, taps, nch, x, plan, lambda s, seg: oracle.channelize_dft8_cs16(seg, K, k, tw)
    h = api.build_lowpass(K, taps)
    return K, taps, nch, x, plan, lambda s, seg: ovl_fast_refs.channelize_ovl_fast_cs16(seg, K, h, k, tw)


def group_of(unit, period, K, rows):
    """Emission group of each envelope row (counted from create / reset): the reference hands a channel's new samples
    to the demodulator per call (SUBMIT), per full buffer of `period` outputs (OUTPUTS), or per transfer of `period`
    input samples (INPUT), where row m completes with input sample (m + 1) K - 1."""
    rows = np.asarray(rows, dtype=np.int64)
    if unit == GROUP_SUBMIT:
        return np.zeros_like(rows)
    if unit == GROUP_OUTPUTS:
        return rows // period
    return ((rows + 1) * K - 1) // period


class Expected:
    """The oracle side: per chain a demodulator state and a sink, fed in the reference's emission order."""

    def __init__(self, oracle, nch):
        self.oracle, self.nch = oracle, nch
        self.msgs, self.raw, self.dropped = [], 0, 0
        self.restart()

    def restart(self):
        self.chans = [[self.oracle.new_chan(c) for c in range(self.nch)] for _ in range(S)]
        self.sinks = [[refs.Sink() for _ in range(self.nch)] for _ in range(S)]

    def feed(self, env, groups):
        """env[s]: (nch, rows) of one submit; groups: the group of each row.  Key order (group, stream, chn, time) within
        the submit; submits in call order."""
        cuts = [0, *(np.flatnonzero(np.diff(groups)) + 1).tolist(), len(groups)]
        for a, b in zip(cuts[:-1], cuts[1:]):
            for s in range(S):
                for c in range(self.nch):
                    sink = self.sinks[s][c]
                    n0 = sink.c.nmsg
                    self.oracle.demod(self.chans[s][c], env[s][c, a:b], sink)
                    for i in range(n0, sink.c.nmsg):
                        self.raw += 1
                        f = self.oracle.fec(sink.c.msgs[i])
                        if f is None:
                            self.dropped += 1
                        else:
                            self.msgs.append((s,) + msg_tuple(f))


def junk_fill(a):
    a[...] = np.float32(-3.0e38) if a.dtype == np.float32 else np.int16(0x5A7A)


@pytest.mark.parametrize("name", list(CASES))
def test_stream_random_walk(native, oracle, name):
    case = CASES[name]
    seed = list(CASES).index(name) + 1
    rng = np.random.default_rng(seed)
    K, taps, nch, x, plan, define = setup(case, oracle, 24 * 1024, seed)
    hrows = -(-max(taps - K, 0) // K)                  # rows whose window reaches into the previous rows
    unit, period = case.group
    if unit == GROUP_INPUT:
        period = K // 3 + 1 if period == "short" else 5 * K + 7
    real, planar = case.kind == "real", case.kind == "planar"
    flags = (FLAG_REAL if real else FLAG_CS16) | case.flags
    lmax = (MAXBLK * 1024 + 1) * K                     # one more than the most a submit may carry with no carry
    stride = lmax + PAD
    exp = Expected(oracle, nch)
    got = []
    total = x.shape[1]

    def src_arrays(buf_or_none, n):
        """Arrays to submit n samples from: pageable (fresh, rows wider than n) or a pinned buffer's views."""
        if buf_or_none is None:
            if planar:
                planes = np.empty((2, S, n + PAD), np.int16)
                return planes[0, :, :n], planes[1, :, :n]
            return (np.empty((S, n + PAD), np.float32) if real else np.empty((S, n + PAD, 2), np.int16))[:, :n],
        a = buf_or_none.array
        if planar:
            v = a.view(np.int16)[:2 * S * stride].reshape(2, S, stride)
            return v[0, :, :n], v[1, :, :n]
        if real:
            return a.view(np.float32)[:S * stride].reshape(S, stride)[:, :n],
        return a.view(np.int16)[:2 * S * stride].reshape(S, stride, 2)[:, :n],

    def call(arrs):
        if real:
            return ctx.submit_real(arrs[0])
        if planar:
            return ctx.submit_cs16_planar(arrs[0], arrs[1])
        return ctx.submit_cs16(arrs[0])

    with api.Context(K, S, nch, MAXBLK, flags=flags, taps=taps) as ctx:
        plan(ctx)
        ctx.set_emission_groups(unit, period)
        pool = []                                      # free pinned buffers
        by_collect = collections.deque()               # pinned buffers of submits that produced rows, oldest first
        by_sync = []                                   # pinned buffers of submits that produced none
        nbuf = 0
        p = seg0 = rows = 0                            # samples fed, start of the current segment, its rows so far
        last = None                                    # (rows, env) of the last submit that produced rows
        nsub = nsync = nreset = 0

        def release(buf):
            for arr in src_arrays(buf, stride):
                junk_fill(arr)
            pool.append(buf)

        def do_sync():
            nonlocal nsync
            ctx.sync()
            nsync += 1
            while by_collect:
                release(by_collect.popleft())
            while by_sync:
                release(by_sync.pop())
            for s in range(S):
                for c in range(nch):
                    assert ctx.get_state(s, c).vec() == exp.chans[s][c].vec(), (nsub, s, c)

        def do_collect():
            ctx.collect()
            if by_collect:
                release(by_collect.popleft())

        step = 0
        while p < total:
            carry = (p - seg0) - rows * K
            lim = lmax - 1 - carry
            if step == 0:
                n = K // 2                             # no row; the first planar submit sizes the staging buffer
            elif step == 1:
                n = K - carry                          # ends exactly on a row
            elif step == 2:
                n = lim                                # the largest: 2048 rows, more than the planar buffer held
            else:
                r = rng.random()
                n = (1 if r < 0.1 else int(rng.integers(1, K - carry)) if r < 0.25 and K - carry > 1 else K - carry if r < 0.35
                     else int(rng.integers(1, MAXBLK + 1)) * 1024 * K if r < 0.5 else lim if r < 0.6
                     else int(rng.integers(1, 700 * K)))
            n = int(min(n, total - p))
            if step == 3 or (step > 3 and rng.random() < 0.03):
                # one sample over the limit: refused, and the stream goes on as if it had not been made
                bad = src_arrays(None, lim + 1)
                for arr in bad:
                    junk_fill(arr)
                with pytest.raises(api.AcbError, match="error -1:"):
                    call(bad)
            buf = None
            if case.pinned:
                if not pool and nbuf == 6:
                    do_sync()
                if pool:
                    buf = pool.pop()
                else:
                    buf, nbuf = api.PinnedBuffer(S * stride * 4), nbuf + 1
            arrs = src_arrays(buf, n)
            seg = x[:, p:p + n]
            if planar:
                arrs[0][...], arrs[1][...] = seg[..., 0], seg[..., 1]
            else:
                arrs[0][...] = seg
            produced = call(arrs)
            nsub += 1
            new = (carry + n) // K
            assert produced == new, (nsub, n, carry)
            if buf is None:
                for arr in arrs:                       # pageable: the call has staged it
                    junk_fill(arr)
            else:
                (by_collect.append if new else by_sync.append)(buf)
            if new:
                r0, r1 = rows, rows + new
                h0 = max(0, r0 - hrows)
                env = [define(s, x[s, seg0 + h0 * K:seg0 + r1 * K])[:, r0 - h0:] for s in range(S)]
                exp.feed(env, group_of(unit, period, K, np.arange(r0, r1)))
                rows = r1
                last = (new, env)
            p += n
            step += 1
            act = rng.random()
            if act < 0.15:
                do_sync()
                if last is not None:
                    dm = ctx.read_dm(last[0])
                    for s in range(S):
                        assert bits_equal(dm[s], last[1][s].T.copy()), (nsub, s)
                if rng.random() < 0.3:                 # state round trip: must change nothing
                    s, c = int(rng.integers(S)), int(rng.integers(nch))
                    ctx.set_state(s, c, ctx.get_state(s, c))
                # initMsk / initAcars again (at least once, past the middle); the carried samples are dropped
                if step > 4 and (rng.random() < 0.15 or (nreset == 0 and 2 * p > total)):
                    got.extend((m.stream,) + msg_tuple(m) for m in ctx.drain())
                    ctx.reset()
                    nreset += 1
                    exp.restart()
                    seg0, rows, last = p, 0, None
            elif act < 0.45:
                do_collect()
            if rng.random() < 0.3:
                got.extend((m.stream,) + msg_tuple(m) for m in ctx.drain())
        do_sync()
        got.extend((m.stream,) + msg_tuple(m) for m in ctx.drain())
        st = ctx.stats()
        while pool:
            pool.pop().close()
    assert got == exp.msgs
    assert len(exp.msgs) >= 20 and nsub >= 30 and nsync >= 3 and nreset >= 1
    assert st.raw_frames == exp.raw and st.fec_dropped == exp.dropped and st.frames_lost == 0
    if case.flags:
        assert st.fast_chan_launches == st.chan_launches > 0
    else:
        assert st.fast_chan_launches == 0 and st.chan_launches > 0
