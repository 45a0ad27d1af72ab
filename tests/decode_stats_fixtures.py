"""Seeded fixtures for the decode statistics (ACB_FLAG_DECODE_STATS), built on acarsdec_b200.synth.

A schedule of frames per channel that reaches every counter of acb_decode_stats_t: clean frames; 1-3 bad-parity bytes
(repaired) and 4 (dropped by the block FEC) and 5 or more (abandoned by the frame synchroniser); CRC-only errors, one
bit of the BCS or two bits of one byte (repaired) and two bits in each of two bytes (not repairable); blocks shorter
than 13 bytes and longer than 240; DLE-terminated text (the missed end); with noise between the bursts, and a
noise-free stream for silence.  Both polarities of the preamble occur: which one the demodulator sees is set by the
state of its bit counter when the burst starts (msk.c:115-118), and the bursts start at random times.

fec_parity_problem (acars.c:202-206) is reached by no input: every repair blk_thread makes leaves each byte's parity
odd (fixprerr flips one bit of each bad byte, fixdberr two bits of one byte).  The tests assert that the reference
prints it as rarely, and the counter stays 0.
"""
from __future__ import annotations

import numpy as np

from acarsdec_b200 import synth

SYN, SOH, ETX, ETB, DLE = 0x16, 0x01, 0x83, 0x97, 0x7F
KINDS = ("clean", "parity1", "parity2", "parity3", "parity4", "parity6", "bcs_bit", "byte_2bits", "two_bytes_2bits",
         "short", "long", "missed_end")


def _head(prekey: int = 16) -> bytes:
    return bytes([0xFF] * prekey) + bytes([synth.odd_parity(ord("+")), synth.odd_parity(ord("*")), SYN, SYN, SOH])


def _safe_crc(body: bytes) -> bytes | None:
    """BCS bytes of `body`, or None when one of them would end the text early (ETX, ETB, DLE)."""
    crc = synth.crc16_kermit(body)
    b = bytes([crc & 0xFF, crc >> 8])
    return None if any(x in (ETX, ETB, DLE) for x in b) else b


def frame_of(kind: str, rng) -> bytes:
    """One burst's bytes as transmitted (prekey .. DEL) for a fixture kind."""
    txt = synth.random_text(rng, int(rng.integers(20, 60)))
    addr = b"." + synth.random_text(rng, 6).replace(b" ", b"-")
    fr = synth.frame_bytes(txt, addr=addr)
    body0 = 13 + 1                      # first text byte after STX, counted from the mode character
    ntxt = len(txt)

    def flips(nbytes: int, masks):
        idx = rng.choice(ntxt, size=nbytes, replace=False) + body0
        return synth.corrupt_frame(fr, [(int(i), m) for i, m in zip(idx, masks)])

    if kind == "clean":
        return fr
    if kind.startswith("parity"):
        n = int(kind[6:])
        return flips(n, [1 << int(rng.integers(0, 7)) for _ in range(n)])
    if kind == "bcs_bit":
        return synth.corrupt_frame(fr, [(-3 + int(rng.integers(0, 2)), 1 << int(rng.integers(0, 8)))])
    if kind == "byte_2bits":
        return flips(1, [0x05 << int(rng.integers(0, 3))])
    if kind == "two_bytes_2bits":
        return flips(2, [0x05 << int(rng.integers(0, 3)), 0x0A << int(rng.integers(0, 3))])
    if kind == "short":                 # SOH + 7 bytes + ETX + BCS: len 8
        while True:
            body = bytes(synth.odd_parity(c) for c in synth.random_text(rng, 7)) + bytes([ETX])
            crc = synth.crc16_kermit(body)
            if DLE not in (crc & 0xFF, crc >> 8):
                return _head() + body + bytes([crc & 0xFF, crc >> 8, DLE])
    if kind == "long":                  # 250 text bytes and no end: abandoned after 241
        return _head() + bytes(synth.odd_parity(c) for c in synth.random_text(rng, 250)) + bytes([DLE] * 2)
    if kind == "missed_end":            # no ETX: the BCS follows the text, DEL ends it (acars.c:324-332)
        while True:
            t = synth.random_text(rng, int(rng.integers(20, 60)))
            body = bytes(synth.odd_parity(c) for c in b"2" + addr + bytes([0x15]) + b"H13" + bytes([0x02]) + t)
            b = _safe_crc(body)
            if b is not None:
                return _head() + body + b + bytes([DLE])
    raise ValueError(kind)


def make_plan(K: int, freqs_hz, fc_hz: int, *, seconds: float, seed: int, noise_sigma: float = 1.5) -> synth.StreamPlan:
    """Every channel cycles through KINDS (from a seeded offset) with seeded gaps of noise between the bursts."""
    plan = synth.StreamPlan(K=K, freqs_hz=tuple(freqs_hz), fc_hz=int(fc_hz), noise_sigma=noise_sigma, seed=seed)
    rng = np.random.default_rng([seed, 0xDEC5])
    for ch in range(len(freqs_hz)):
        t = 0.01 + rng.uniform(0, 0.05)
        k = int(rng.integers(0, len(KINDS)))
        while True:
            fr = frame_of(KINDS[k % len(KINDS)], rng)
            dur = len(fr) * 8 / synth.BAUD
            if t + dur + 0.01 > seconds:
                break
            plan.bursts.append(synth.Burst(chan=ch, t0=t, frame=fr, amp=float(rng.uniform(12.0, 30.0)),
                                           phase=float(rng.uniform(0, 2 * np.pi))))
            t += dur + 0.015 + rng.exponential(0.03)
            k += 1
    return plan


def plan_stream(K: int, seconds: float, seed: int, noise_sigma: float = 1.5):
    """(plan, freqs_hz as set_plan takes them) for the default 8-channel raster."""
    from acarsdec_b200 import api
    fd, _, fc = api.plan(K, synth.DEFAULT_FREQS_MHZ)
    return make_plan(K, fd, fc, seconds=seconds, seed=seed, noise_sigma=noise_sigma), fd
