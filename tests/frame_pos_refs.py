"""Message positions, the framing state and the frame synchroniser's exits, defined by the restatement driven one
envelope sample at a time (TEST INFRASTRUCTURE).

The oracle (oracle/acars_oracle.c) carries no positions, and its result does not depend on how the envelope is cut
into orc_demod calls.  Feeding it one sample per call therefore observes the ordinary run and tells, for every event,
the sample after which it happened:
  - a frame's `pos`: the sample after which the sink grew (frames under 13 bytes included: they reach the sink);
  - `soh_pos`: the sample after which the state went from F_SOH1 to F_TXT (where the device stamps it);
  - the exits of the frame synchroniser (frame_sm.h / acars.c:246-375), see EXITS.
Samples are counted from the channel's start, or from `pos0` when the run continues a state.

The fixture (Fixture) is a set of crafted byte streams, one per channel, that walk the synchroniser through every
exit: missed ETX (the DLE finish, and too short to finish), text running past 240 bytes, exactly 4 and 5 parity
errors, blocks of 13, 240 and 241 bytes, frames under 13 bytes, SYN SYN + a non-SOH byte, frames back to back with no
gap after DEL, ETB-terminated frames and a preamble that inverts the polarity in F_SYN2 (SYN, ~SYN, then everything
inverted; the next frame then meets an inverted SYN in F_WSYN).
"""
from __future__ import annotations

import ctypes as C
import functools
from dataclasses import dataclass, field

import numpy as np

import refs
from acarsdec_b200 import synth

WSYN, SYN2, SOH1, TXT, CRC1, CRC2, END = range(7)
NSYN = 0xE9

# exit kinds the fixture must reach (see Trace.events)
EXITS = ("len241", "parity5", "dle", "nsyn_syn2", "nsyn_wsyn", "soh_mismatch", "end_resync", "short")


@dataclass
class Frame:
    msg: refs.Msg          # the pre-FEC block as the sink got it
    pos: int
    soh_pos: int


@dataclass
class Trace:
    frames: list = field(default_factory=list)
    events: dict = field(default_factory=dict)     # kind -> [sample index]
    snaps: dict = field(default_factory=dict)      # samples consumed -> (vec, framing)
    states: bytearray = field(default_factory=bytearray)   # F_* after every sample
    nbits: bytearray = field(default_factory=bytearray)    # nbits after every sample
    chan: refs.OrcChan | None = None               # the final state
    soh_pos: int = 0
    pos: int = 0


def framing(ch: refs.OrcChan, soh_pos: int) -> tuple:
    """The framing half of a channel's state: what acb_chan_state_t carries beyond vec()."""
    n = ch.blk.len
    return (ch.state, n, ch.blk.err, bytes(ch.blk.txt[:n]), ch.blk.crc[0] if ch.state == CRC2 else None, soh_pos)


def device_framing(st) -> tuple:
    """The same from an acb_chan_state_t (api.ChanState)."""
    n = st.blk_len
    return (st.Acarsstate, n, st.blk_err, bytes(st.blk_txt[:n]), st.blk_crc[0] if st.Acarsstate == CRC2 else None,
            st.soh_pos)


def copy_chan(ch: refs.OrcChan) -> refs.OrcChan:
    out = refs.OrcChan()
    C.memmove(C.byref(out), C.byref(ch), C.sizeof(refs.OrcChan))
    return out


def run(oracle, x: np.ndarray, *, chan: refs.OrcChan | None = None, pos0: int = 0, soh_pos0: int = 0,
        checkpoints=()) -> Trace:
    """Drive the restatement over the envelope x one sample per orc_demod call, from `chan` (copied; a fresh channel
    by default) whose samples so far number pos0.  Snapshots (vec(), framing()) are taken after each checkpoint (a count
    of samples of x)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    ch = copy_chan(chan) if chan is not None else oracle.new_chan(0)
    sink = refs.Sink()
    tr = Trace(soh_pos=soh_pos0)
    tr.states = bytearray(len(x))
    tr.nbits = bytearray(len(x))
    cps = set(int(c) for c in checkpoints)
    if 0 in cps:
        tr.snaps[0] = (ch.vec(), framing(ch, tr.soh_pos))
    demod, h, base = oracle.lib.orc_demod, oracle.h.ctypes.data, x.ctypes.data
    chp, sinkp, sc = C.byref(ch), C.byref(sink.c), sink.c
    ev = tr.events
    for i in range(len(x)):
        st0, nb0, bits0, n0 = ch.state, ch.nbits, ch.nbit_total, sc.nmsg
        demod(chp, h, base + 4 * i, 1, sinkp)
        if ch.nbit_total != bits0 and nb0 <= 1:          # a byte (or, hunting, a bit) went to the synchroniser
            st1, p = ch.state, pos0 + i
            if sc.nmsg != n0:
                m = refs.Msg()
                C.memmove(C.byref(m), C.byref(sc.msgs[sc.nmsg - 1]), C.sizeof(refs.Msg))
                tr.frames.append(Frame(m, p, tr.soh_pos))
                if st0 == TXT:
                    ev.setdefault("dle", []).append(p)
                if m.len < 13:
                    ev.setdefault("short", []).append(p)
            elif st0 == SOH1:
                if st1 == TXT:
                    tr.soh_pos = p
                else:
                    ev.setdefault("soh_mismatch", []).append(p)
            elif st0 == TXT and st1 == WSYN:
                if ch.blk.err > 4:
                    ev.setdefault("parity5", []).append(p)
                else:
                    assert ch.blk.len > 240
                    ev.setdefault("len241", []).append(p)
            elif st0 == SYN2 and st1 == SYN2:
                ev.setdefault("nsyn_syn2", []).append(p)
            elif st0 == WSYN and st1 == SYN2 and ch.outbits == NSYN:
                ev.setdefault("nsyn_wsyn", []).append(p)
            elif st0 == END:
                ev.setdefault("end_resync", []).append(p)
        tr.states[i] = ch.state
        tr.nbits[i] = ch.nbits
        if i + 1 in cps:
            tr.snaps[i + 1] = (ch.vec(), framing(ch, tr.soh_pos))
    tr.chan, tr.pos = ch, pos0 + len(x)
    return tr


def run_chunked(oracle, x: np.ndarray, cuts):
    """The same envelope in ordinary orc_demod calls of the given sizes (the rest in one call): [(frame keys of the
    call, [start, end) of the call)] and the channel's (vec, framing without soh_pos) after every call."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    ch, sink = oracle.new_chan(0), refs.Sink()
    calls, snaps, a = [], {}, 0
    bounds = [int(b) for b in np.cumsum([int(c) for c in cuts]) if b < len(x)] + [len(x)]
    for b in bounds:
        before = sink.c.nmsg
        oracle.demod(ch, x[a:b], sink)
        calls.append(([m.key() for m in sink.msgs()[before:]], (a, b)))
        snaps[b] = (ch.vec(), framing(ch, 0)[:-1])
        a = b
    return calls, snaps


# ------------------------------------------------------------------ the fixture

P = synth.odd_parity
HEAD = bytes([0xFF] * 16 + [P(ord("+")), P(ord("*"))])
SYN = 0x16
SOH = 0x01


def _body(rng, ntext: int, *, end: int | None = 0x03, stx: bool = True, perr: int = 0) -> bytes:
    """mode, address, ack, label, block id (12 bytes), STX, text, end byte (None: none), all with odd parity; `perr`
    text bytes get their parity bit flipped (before the BCS is computed)."""
    b = bytearray(P(c) for c in b"2.N123AB")
    b += bytes([P(0x15)]) + bytes(P(c) for c in b"H1") + bytes([P(0x30 + int(rng.integers(0, 10)))])
    if stx:
        b.append(P(0x02))
    t0 = len(b)
    b += bytes(P(c) for c in synth.random_text(rng, ntext))
    for k in range(perr):
        b[t0 + 1 + 3 * k] ^= 0x80
    if end is not None:
        b.append(P(end))
    return bytes(b)


def _tail(body: bytes) -> bytes:
    crc = synth.crc16_kermit(body)
    return bytes([crc & 0xFF, crc >> 8, 0x7F])


def _frame(body: bytes, *, pre=bytes([SYN, SYN, SOH])) -> bytes:
    return HEAD + pre + body + _tail(body)


def case_bytes(rng, kind: str) -> bytes:
    """The transmitted bytes of one burst of the given kind."""
    if kind == "etx":
        return _frame(_body(rng, int(rng.integers(20, 50))))
    if kind == "etb":
        return _frame(_body(rng, int(rng.integers(20, 50)), end=0x17))
    if kind == "dle":               # missed ETX, text long enough for the DLE finish
        return _frame(_body(rng, int(rng.integers(25, 45)), end=ord("A")))
    if kind == "dle_short":         # missed ETX with DEL at text length <= 20: no finish
        return _frame(_body(rng, 2, end=ord("A")))
    if kind == "run241":            # correct parity, no ETX/ETB/DLE, past 240 bytes
        return _frame(_body(rng, 236, end=None))
    if kind == "perr4":
        return _frame(_body(rng, 40, perr=4))
    if kind == "perr5":
        return _frame(_body(rng, 40, perr=5))
    if kind == "blk13":             # 12 header bytes + ETX
        return _frame(_body(rng, 0, stx=False))
    if kind == "blk240":
        return _frame(_body(rng, 226))
    if kind == "blk241":
        return _frame(_body(rng, 227))
    if kind == "short":             # SOH, a few bytes, ETX, BCS
        b = bytes(P(c) for c in b"2.N")[:int(rng.integers(1, 4))] + bytes([P(0x03)])
        return _frame(b)
    if kind == "soh_bad":           # SYN SYN and a byte other than SOH
        return _frame(_body(rng, 10), pre=bytes([SYN, SYN, 0x05]))
    if kind == "b2b":               # back to back, no gap after DEL (F_END takes the DEL, then 8 bits: the next SYN)
        f1 = _frame(_body(rng, int(rng.integers(10, 30))))
        b2 = _body(rng, int(rng.integers(10, 30)))
        b3 = _body(rng, 12)
        return f1 + bytes([SYN, SYN, SOH]) + b2 + _tail(b2) + HEAD + bytes([SYN, SYN, SOH]) + b3 + _tail(b3)
    if kind == "flip":              # SYN, ~SYN, then everything inverted: F_SYN2 meets NSYN
        b = _body(rng, int(rng.integers(20, 40)))
        rest = bytes([SYN, SOH]) + b + _tail(b)
        return HEAD + bytes([SYN, 0xFF ^ SYN]) + bytes(0xFF ^ c for c in rest)
    raise ValueError(kind)


KINDS = ("etx", "dle", "run241", "perr4", "blk13", "flip", "short", "perr5", "etb", "blk240", "soh_bad", "dle_short",
         "b2b", "blk241")
K_FIX = 160
NCH = 11                           # a prime, coprime with 32
FM = tuple(round(131.400 + 0.025 * i, 3) for i in range(NCH))
AMP, NOISE = 30.0, 1.0


def channel_kinds(c: int, per: int = 6):
    """Channel c's bursts: `per` consecutive kinds of KINDS starting at 5c (every kind on several channels; the ten
    bursts after a "flip" start with an inverted SYN in F_WSYN)."""
    return [KINDS[(5 * c + j) % len(KINDS)] for j in range(per)]


@dataclass
class Fixture:
    K: int
    freqs_hz: tuple
    fc: int
    nblk: int
    iq: np.ndarray                 # u8, (nblk * 1024 * K * 2,)
    env: np.ndarray                # (NCH, nblk * 1024) float32: the oracle's channelizer
    plan: synth.StreamPlan


def stream_plan(fd, fc, K: int, seed: int = 41):
    """(plan, seconds): every channel's bursts back to back with 30 ms gaps."""
    plan = synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, noise_sigma=NOISE, seed=seed)
    end = 0.0
    for c in range(len(fd)):
        rng = np.random.default_rng([seed, c])
        t = 0.01 + 0.003 * c
        for kind in channel_kinds(c):
            fr = case_bytes(rng, kind)
            plan.bursts.append(synth.Burst(chan=c, t0=t, frame=fr, amp=AMP, phase=float(rng.uniform(0, 2 * np.pi))))
            t += len(fr) * 8 / synth.BAUD + 0.03
        end = max(end, t)
    return plan, end


@functools.lru_cache(maxsize=None)
def fixture() -> Fixture:
    oracle = refs.OracleLib()
    fd, _, fc = oracle.plan(K_FIX, FM)
    plan, secs = stream_plan(fd, fc, K_FIX)
    nblk = synth.blocks_for_seconds(K_FIX, secs + 0.02)
    iq = synth.render_blocks(plan, 0, nblk).reshape(-1)
    env = oracle.channelize(iq, K_FIX, oracle.wf(K_FIX, FM))
    return Fixture(K_FIX, tuple(fd), fc, nblk, iq, env, plan)


@functools.lru_cache(maxsize=None)
def traces(checkpoints: tuple = ()) -> tuple:
    """The one-sample run of every fixture channel from a fresh state."""
    oracle = refs.OracleLib()
    fx = fixture()
    return tuple(run(oracle, fx.env[c], checkpoints=checkpoints) for c in range(NCH))


def coverage(trs) -> dict:
    """exit kind -> (occurrences, channels where it occurs)"""
    out = {}
    for c, tr in enumerate(trs):
        for k, v in tr.events.items():
            n, chans = out.get(k, (0, set()))
            out[k] = (n + len(v), chans | {c})
    return out
