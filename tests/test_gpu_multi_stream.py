"""acb_multi_* for the streaming front-ends: real input (air.c) and CS16 (soapy.c interleaved, sdrplay.c planar).

Parts go on devices i % device_count, so one GPU runs every case; the split and the merge are the same code either way.
The rule throughout: a multi-context gives exactly what one context gives.  That is every acb_msg_t field (stream, chn,
len, err, txt, crc, lvl bits, block, pos, soh_pos) in the same order, and the same demodulator state of the last stream
and channel.  The submits are ragged (shorter than K, not multiples of K, several in flight before a sync), the
emission-group periods do not divide the submit lengths, and some cases reset in the middle of the run.

A second part runs the shim's Airspy, SoapySDR and SDRplay front-ends (tests/host/fehost.c) over the same capture with
ACARSDEC_B200_DEVICES naming three contexts and without it: the printed blocks must be byte-identical."""
import os
import subprocess
from dataclasses import dataclass

import numpy as np
import pytest

from acarsdec_b200 import api, synth
from common import msg_tuple
from test_gpu_multi import _devices

pytestmark = pytest.mark.gpu

FLAG_REAL, FLAG_CS16 = 2, 4
FAST_CHANNELIZER, FAST_FILTER, FAST_FILTER_REAL, FAST_WIDEBAND, FAST_WIDEBAND_REAL = 8, 16, 32, 64, 128
GROUP_SUBMIT, GROUP_OUTPUTS, GROUP_INPUT = 0, 1, 2
SPLIT_STREAMS, SPLIT_CHANNELS = 0, 1
# on the 12.5 kHz raster around the centre chosen over all of them; subsets of them would choose other centres
REAL_FM = tuple(131.400 + 0.025 * i for i in range(11))
CS16_FM = tuple(130.000 + 0.025 * i for i in range(11))
SECONDS = 0.8


@dataclass
class Case:
    kind: str                  # "real", "cs16" (interleaved, soapy.c scale) or "planar" (sdrplay.c scale)
    mode: int                  # SPLIT_STREAMS / SPLIT_CHANNELS
    nstreams: int
    nch: int
    nparts: int
    flags: int = 0             # a fast form on top of the input kind
    over: bool = False         # taps > K (2K + 3) instead of taps = K
    group: tuple = (GROUP_SUBMIT, 0)
    reset: bool = False        # acb_reset after half the submits


CASES = {
    "real-streams-5x2": Case("real", SPLIT_STREAMS, 5, 4, 2, group=(GROUP_INPUT, 65536)),
    "real-streams-3x4-gt-fast": Case("real", SPLIT_STREAMS, 3, 4, 4, FAST_FILTER_REAL, over=True, group=(GROUP_OUTPUTS, 700)),
    "real-channels-11x3-fast": Case("real", SPLIT_CHANNELS, 1, 11, 3, FAST_CHANNELIZER, group=(GROUP_INPUT, 5 * 200 + 7)),
    "real-channels-11x3-gt-wideband-reset": Case("real", SPLIT_CHANNELS, 1, 11, 3, FAST_WIDEBAND_REAL, over=True,
                                                 group=(GROUP_OUTPUTS, 1000), reset=True),
    "real-channels-2ch-3parts": Case("real", SPLIT_CHANNELS, 2, 2, 3, over=True, group=(GROUP_SUBMIT, 0)),
    "cs16-streams-5x2-gt": Case("cs16", SPLIT_STREAMS, 5, 4, 2, over=True, group=(GROUP_OUTPUTS, 1000)),
    "cs16-channels-11x3-fast-reset": Case("cs16", SPLIT_CHANNELS, 1, 11, 3, FAST_CHANNELIZER, group=(GROUP_INPUT, 65536),
                                          reset=True),
    "cs16-streams-3x4-wideband": Case("cs16", SPLIT_STREAMS, 3, 8, 4, FAST_WIDEBAND, group=(GROUP_SUBMIT, 0)),
    "planar-channels-11x3-gt-fast": Case("planar", SPLIT_CHANNELS, 1, 11, 3, FAST_FILTER, over=True, group=(GROUP_OUTPUTS, 512)),
    "planar-streams-5x2": Case("planar", SPLIT_STREAMS, 5, 4, 2, group=(GROUP_INPUT, 3 * 160 + 1), reset=True),
    "planar-channels-2x8x2-gt-wideband": Case("planar", SPLIT_CHANNELS, 2, 8, 2, FAST_WIDEBAND, over=True,
                                              group=(GROUP_INPUT, 65536)),
}


def _key(m):
    return (m.stream,) + msg_tuple(m) + (int(m.block), int(m.pos), int(m.soh_pos))


def _signal(case):
    """(K, freqs_hz, input): float32 (S, n) for real input, int16 (S, n, 2) for CS16, a pair of int16 (S, n) planes for planar."""
    real = case.kind == "real"
    K = 200 if real else 160
    rate = K * 12500
    fm = (REAL_FM if real else CS16_FM)[:case.nch]
    if real:
        fd, fc, _ = api.air_plan(rate, fm)
    else:
        fd, _, fc = api.plan(K, fm)
    n = int(SECONDS * rate)
    xs = []
    for s in range(case.nstreams):
        p = synth.make_plan(K, fm, fc, seconds=SECONDS, seed=300 + 10 * s + case.nch, msgs_per_chan_per_sec=8.0,
                            text_len=(5, 30), amp=(6.0, 12.0))
        if real:
            xs.append(synth.render_real(synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, bursts=p.bursts, seed=p.seed), 0, n))
        else:
            xs.append(synth.render_cs16(p, 0, n))
    x = np.stack(xs)
    if case.kind == "planar":
        x = (np.ascontiguousarray(x[..., 0]), np.ascontiguousarray(x[..., 1]))
    return K, fd, x


def _chunks(K, n, seed):
    """Ragged submit lengths covering n samples: one shorter than K, odd lengths, whole blocks and more."""
    rng = np.random.default_rng(seed)
    sizes, at = [K // 3, 7 * K + 13], K // 3 + 7 * K + 13
    while at < n:
        sz = int(rng.choice([K - 1, 1024 * K + 5, 2048 * K - 17, int(rng.integers(1, 3 * 1024 * K))]))
        sizes.append(min(sz, n - at))
        at += sizes[-1]
    return sizes


def _run(ctx, case, K, fd, x):
    """Plan, set the groups, submit the chunks with collects between some of them; (messages, last chain's state)."""
    variant = 1 if case.kind == "planar" else 0
    for s in range(case.nstreams):
        ctx.set_plan_air(s, fd) if case.kind == "real" else ctx.set_plan_cs16(s, fd, variant)
    ctx.set_emission_groups(*case.group)
    n = (x[0] if case.kind == "planar" else x).shape[1]
    sizes = _chunks(K, n, n)
    out, at = [], 0
    for i, sz in enumerate(sizes):
        sl = slice(at, at + sz)
        if case.kind == "real":
            ctx.submit_real(x[:, sl])
        elif case.kind == "cs16":
            ctx.submit_cs16(x[:, sl])
        else:
            ctx.submit_cs16_planar(x[0][:, sl], x[1][:, sl])
        at += sz
        if i % 3 == 2:
            ctx.collect()
            out += [_key(m) for m in ctx.drain()]
        if case.reset and i == len(sizes) // 2:
            ctx.sync()
            out += [_key(m) for m in ctx.drain()] + ["reset"]
            ctx.reset()
    ctx.sync()
    out += [_key(m) for m in ctx.drain()]
    return out, ctx.get_state(case.nstreams - 1, case.nch - 1).vec()


@pytest.mark.parametrize("name", list(CASES))
def test_multi_stream_equals_single_context(native, name):
    case = CASES[name]
    K, fd, x = _signal(case)
    taps = 2 * K + 3 if case.over else 0
    flags = (FLAG_REAL if case.kind == "real" else FLAG_CS16) | case.flags
    maxblk = 3
    with api.Context(K, case.nstreams, case.nch, maxblk, flags=flags, taps=taps) as one:
        want, st_one = _run(one, case, K, fd, x)
        if case.flags:
            assert one.stats().fast_chan_launches > 0
    with api.MultiContext(K, case.nstreams, case.nch, maxblk, _devices(case.nparts), mode=case.mode, flags=flags,
                          taps=taps) as multi:
        nparts = multi.parts()
        assert nparts == min(case.nparts, case.nstreams if case.mode == SPLIT_STREAMS else case.nch)
        got, st_multi = _run(multi, case, K, fd, x)
        if case.flags:
            assert all(multi.part_stats(i).fast_chan_launches > 0 for i in range(nparts))
    nmsg = sum(1 for k in want if k != "reset")
    assert nmsg >= case.nstreams * case.nch
    assert len({k[:2] for k in want if k != "reset"}) > 1
    assert got == want
    assert st_multi == st_one


def test_multi_stream_wrong_kind_is_refused(native):
    K = 160
    with api.MultiContext(K, 2, 4, 1, _devices(2), mode=SPLIT_STREAMS, flags=FLAG_CS16) as cs, \
            api.MultiContext(200, 1, 4, 1, _devices(2), mode=SPLIT_CHANNELS, flags=FLAG_REAL) as air, \
            api.MultiContext(K, 2, 4, 1, _devices(2), mode=SPLIT_STREAMS) as u8:
        fd, _, _ = api.plan(K, CS16_FM[:4])
        with pytest.raises(api.AcbError, match="ACB_FLAG_REAL_INPUT"):
            cs.submit_real(np.zeros((2, 1000), np.float32))
        with pytest.raises(api.AcbError, match="u8-IQ"):
            cs.submit_host(np.zeros((2, 2048 * K), np.uint8), 1)
        with pytest.raises(api.AcbError, match="ACB_FLAG_CS16_INPUT"):
            air.submit_cs16(np.zeros((1, 1000, 2), np.int16))
        with pytest.raises(api.AcbError, match="ACB_FLAG_CS16_INPUT"):
            air.submit_cs16_planar(np.zeros((1, 1000), np.int16), np.zeros((1, 1000), np.int16))
        with pytest.raises(api.AcbError):
            u8.submit_real(np.zeros((2, 1000), np.float32))
        with pytest.raises(api.AcbError):
            u8.submit_cs16(np.zeros((2, 1000, 2), np.int16))
        with pytest.raises(api.AcbError, match="real-input"):
            cs.set_plan_air(0, fd)
        with pytest.raises(api.AcbError, match="CS16"):
            air.set_plan_cs16(0, fd, 0)
        with pytest.raises(api.AcbError, match="variant"):
            cs.set_plan_cs16(0, fd, 7)
        with pytest.raises(api.AcbError, match="unknown group unit"):
            cs.set_emission_groups(5, 10)
        # a refused call changed nothing: the contexts still serve their own kind
        cs.set_plan_cs16(0, fd, 0)
        cs.set_plan_cs16(1, fd, 0)
        assert cs.submit_cs16(np.zeros((2, 2 * K + 1, 2), np.int16)) == 2
        assert cs.sync() == 0


def test_set_plan_air_at_equals_set_plan_air(native):
    """acb_set_plan_air_at at the centre acb_set_plan_air chooses: the same envelope, bit for bit (exact and fast form)."""
    rate, K = 2500000, 200
    fd, fc, _ = api.air_plan(rate, REAL_FM[:5])
    p = synth.make_plan(K, REAL_FM[:5], fc, seconds=0.1, seed=5)
    x = synth.render_real(synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, bursts=p.bursts, seed=5), 0, 1024 * K + 77)
    for flags in (FLAG_REAL, FLAG_REAL | FAST_CHANNELIZER):
        dms = []
        for at in (False, True):
            with api.Context(K, 1, 5, 2, flags=flags) as ctx:
                if at:
                    ctx.set_plan_air_at(0, fd, fc)
                else:
                    assert ctx.set_plan_air(0, fd) == fc
                nout = ctx.submit_real(x.reshape(1, -1))
                ctx.sync()
                dms.append(ctx.read_dm(nout))
                assert ctx.stats().fast_chan_launches == (1 if flags & FAST_CHANNELIZER else 0)
        assert np.array_equal(dms[0].view(np.uint32), dms[1].view(np.uint32))
    with api.Context(K, 1, 5, 2, flags=FLAG_REAL) as ctx, pytest.raises(api.AcbError, match="centre frequency 0"):
        ctx.set_plan_air_at(0, fd, 0)


# ---------------------------------------------------------------- the shim's streaming front-ends over several contexts

def _air_capture(tmp_path, rate, fm):
    fd, fc, K = api.air_plan(rate, fm)
    plan = synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, seed=41, noise_sigma=1.0)
    rng = np.random.default_rng(41)
    for ch in range(len(fm)):
        t = 0.01 + 0.04 * ch
        for _ in range(3):
            fr = synth.frame_bytes(synth.random_text(rng, int(rng.integers(10, 60))))
            plan.bursts.append(synth.Burst(chan=ch, t0=t, frame=fr, amp=float(rng.uniform(10, 25)), phase=float(rng.uniform(0, 6))))
            t += len(fr) * 8 / 2400 + 0.05
    cap = tmp_path / "cap.f32"
    synth.render_real(plan, 0, int(1.2 * rate)).tofile(cap)
    return cap


@pytest.mark.parametrize("macro", ["WITH_AIR", "WITH_SOAPY", "WITH_SDRPLAY"])
@pytest.mark.parametrize("taps", ["", "2K+40"])
def test_shim_front_end_over_several_contexts(tmp_path, native, macro, taps):
    """The same capture through one context and through three (channel split, 4 channels): byte-identical output.
    With ACARSDEC_B200_TAPS the planner runs inside the library, so the parts must share the receiver's centre."""
    from test_compat import _cs16_capture
    from test_ovl_shim import fehost, run
    exe = fehost(tmp_path, macro)
    if macro == "WITH_AIR":
        rate, fm = 2500000, (131.525, 131.725, 131.825, 131.450)
        cap, K = _air_capture(tmp_path, rate, fm), rate // 12500
        cmd, env = [exe, cap, *fm], {"ACARSDEC_B200_AIRRATE": str(rate)}
    else:
        K = 160
        cap, freqs = _cs16_capture(tmp_path, 23 if macro == "WITH_SOAPY" else 29)
        cmd = [exe, K, cap, *freqs] if macro == "WITH_SOAPY" else [exe, *freqs]
        env = {"ACARSDEC_B200_CAPTURE": str(cap)}
    if taps:
        env["ACARSDEC_B200_TAPS"] = str(2 * K + 40)
    one = run(cmd, dict(env, ACARSDEC_B200_DEVICES=""))
    three = run(cmd, dict(env, ACARSDEC_B200_DEVICES=",".join(str(d) for d in _devices(3))))
    assert one.returncode == 0, one.stderr
    assert three.returncode == 0, three.stderr
    assert len(one.stdout.splitlines()) >= 10
    assert three.stdout == one.stdout


REFBIN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")


@pytest.mark.parametrize("front_end", ["air", "soapy", "sdrplay"])
def test_unmodified_program_over_several_contexts(tmp_path, native, front_end):
    """The reference's own acarsdec.c linked against the shim, ACARSDEC_B200_DEVICES naming three contexts: byte-identical
    stdout to the same program built with the reference's front-end, as tests/test_compat.py checks it on one context."""
    from test_compat import _cs16_capture, _strip_time
    mine_bin, ref_bin = (os.path.join(REFBIN, f"acarsdec_{w}_{front_end}") for w in ("b200", "ref"))
    if not (os.path.exists(mine_bin) and os.path.exists(ref_bin)):
        pytest.skip("oracle/_ref programs absent")
    devs = ",".join(str(d) for d in _devices(3))
    if front_end == "air":
        rate, fm = 2500000, (131.525, 131.725, 131.825, 131.450)
        cap = _air_capture(tmp_path, rate, fm)
        freqs = [str(f) for f in fm]
        ref_cmd, ref_env = [ref_bin, "-o", "2", "-s", "0", *freqs], {"ACARSDEC_STUB_AIR": str(cap), "ACARSDEC_STUB_AIRRATE": str(rate)}
        mine_cmd, mine_env = [mine_bin, "-o", "2", "-s", str(cap), *freqs], {"ACARSDEC_B200_AIRRATE": str(rate)}
    elif front_end == "soapy":
        cap, freqs = _cs16_capture(tmp_path, 23)
        ref_cmd, ref_env = [ref_bin, "-o", "2", "-d", str(cap), *freqs], {}
        mine_cmd, mine_env = [mine_bin, "-o", "2", "-d", str(cap), *freqs], {}
    else:
        cap, freqs = _cs16_capture(tmp_path, 29)
        ref_cmd, ref_env = [ref_bin, "-o", "2", "-s", *freqs], {"ACARSDEC_STUB_SDRPLAY": str(cap)}
        mine_cmd, mine_env = [mine_bin, "-o", "2", "-s", *freqs], {"ACARSDEC_B200_CAPTURE": str(cap)}
    ref = subprocess.run(ref_cmd, env=dict(os.environ, **ref_env), capture_output=True, text=True, timeout=120)
    mine = subprocess.run(mine_cmd, env=dict(os.environ, ACARSDEC_B200_DEVICES=devs, **mine_env), capture_output=True, text=True,
                          timeout=120)
    assert mine.returncode == 0, mine.stderr
    a, b = _strip_time(ref.stdout), _strip_time(mine.stdout)
    assert a.count("<time>") >= 10 and a == b
