"""ACARSDEC_B200_TAPS: the shim's front-ends use the overlapping-window low-pass when it is set.

Through tests/host/fehost.c, a host built here against the shim libraries of this tree (one per front-end): a bad value
is an init error with a message (no GPU needed); with a valid one, every front-end prints the messages a library context
with the same filter decodes from the same capture, and on the RTL front-end the variable is what makes a weak channel
next to a strong neighbour decodable.  The reference's unmodified acarsdec program is checked too where oracle/_ref holds
one built from this tree's compat.c."""
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

from acarsdec_b200 import api, build, synth
from test_compat import _cs16_capture
from test_ovl_oracle import weak_strong_scenario

ROOT = Path(__file__).resolve().parent.parent
PKG = ROOT / "acarsdec_b200"
REFBIN = ROOT / "oracle" / "_ref"
FLAG_REAL, FLAG_CS16 = 2, 4
SHIMS = dict(build.COMPAT_VARIANTS)            # WITH_* macro -> shim library


def fehost(tmp_path, macro) -> Path:
    build.build()
    exe = tmp_path / ("fehost_" + macro)
    subprocess.run(["gcc", "-O1", "-std=gnu11", "-D" + macro, "-I", str(ROOT / "include"), "-o", str(exe),
                    str(ROOT / "tests" / "host" / "fehost.c"), str(SHIMS[macro]), "-L", str(PKG), "-lacars_b200",
                    f"-Wl,-rpath,{PKG}", "-lpthread", "-lm"], check=True)
    return exe


def run(cmd, env):
    return subprocess.run([str(c) for c in cmd], env=dict(os.environ, **env), capture_output=True, text=True, timeout=120)


def host_msgs(stdout):
    out = []
    for line in stdout.split("\n"):
        if line.strip():
            chn, ln, err, crc, *txt = line.split()
            out.append((int(chn), int(ln), int(err), bytes.fromhex(txt[0] if txt else ""), bytes.fromhex(crc)))
    return sorted(out)


def ctx_msgs(ctx):
    ctx.sync()
    return sorted(m.as_tuple() for m in ctx.drain())


FM = (131.525, 131.725, 131.825, 131.450)


@pytest.mark.parametrize("macro", ["WITH_RTL", "WITH_AIR", "WITH_SOAPY", "WITH_SDRPLAY"])
@pytest.mark.parametrize("which", ["below_k", "above_16k", "not_a_number"])
def test_bad_taps_is_an_init_error(tmp_path, macro, which):
    """Below K, above 16K or not a number: initialisation stops with a message naming the variable, before any device
    work (K = 160 for RTL, Soapy and SDRplay here; 200 for Airspy at its 2.5 MS/s default)."""
    K = 200 if macro == "WITH_AIR" else 160
    value = {"below_k": str(K - 1), "above_16k": str(16 * K + 1), "not_a_number": "12x"}[which]
    exe = fehost(tmp_path, macro)
    cap = tmp_path / "empty"
    cap.write_bytes(b"")
    args = {"WITH_RTL": [K, cap], "WITH_AIR": [cap], "WITH_SOAPY": [K, cap], "WITH_SDRPLAY": []}[macro]
    r = run([exe, *args, *FM], {"ACARSDEC_B200_TAPS": value, "ACARSDEC_B200_CAPTURE": str(cap)})
    assert r.returncode != 0
    assert "ACARSDEC_B200_TAPS=" + value in r.stderr


@pytest.mark.gpu
def test_rtl_taps_matches_library_and_rescues_weak_channel(tmp_path, native):
    K, taps = 160, 8 * 160
    exe = fehost(tmp_path, "WITH_RTL")
    fm = (131.525, 131.725, 131.825, 131.450, 131.550)
    fd, _, fc = api.plan(K, fm)
    plan = synth.make_plan(K, fm, fc, seconds=1.2, seed=78, text_len=(10, 60), msgs_per_chan_per_sec=3.0)
    nblk = synth.blocks_for_seconds(K, 1.2)
    iq = synth.render_blocks(plan, 0, nblk)
    cap = tmp_path / "cap.iq"
    iq.tofile(cap)
    r = run([exe, K, cap, *fm], {"ACARSDEC_B200_TAPS": str(taps), "ACARSDEC_B200_BLOCKS": "4"})
    assert r.returncode == 0, r.stderr
    with api.Context(K, 1, len(fm), nblk, taps=taps) as ctx:
        ctx.set_plan(0, fd)
        ctx.submit_host(iq.reshape(1, -1), nblk)
        want = ctx_msgs(ctx)
    assert len(want) >= 8 and host_msgs(r.stdout) == want
    # the variable is what decodes the weak channel next to a strong neighbour
    iq, fm2, sent = weak_strong_scenario(K)
    cap2 = tmp_path / "weak.iq"
    iq.tofile(cap2)
    weak = {}
    for name, env in (("boxcar", {}), ("lowpass", {"ACARSDEC_B200_TAPS": str(taps)})):
        r = run([exe, K, cap2, *fm2], dict(env, ACARSDEC_B200_BLOCKS="4"))
        assert r.returncode == 0, r.stderr
        weak[name] = [m for m in host_msgs(r.stdout) if m[0] == 0]
    assert len(weak["lowpass"]) == len(sent) and all(m[2] == 0 for m in weak["lowpass"])
    assert not any(m[2] == 0 for m in weak["boxcar"])


@pytest.mark.gpu
def test_airspy_taps_matches_library(tmp_path, native):
    rate, taps = 2500000, 4 * 200 + 12
    exe = fehost(tmp_path, "WITH_AIR")
    fd, fc, K = api.air_plan(rate, FM)
    plan = synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, seed=19, noise_sigma=1.0)
    rng = np.random.default_rng(19)
    for ch in range(4):
        t = 0.01 + 0.04 * ch
        for _ in range(3):
            fr = synth.frame_bytes(synth.random_text(rng, int(rng.integers(10, 60))))
            plan.bursts.append(synth.Burst(chan=ch, t0=t, frame=fr, amp=float(rng.uniform(10, 25)), phase=float(rng.uniform(0, 6))))
            t += len(fr) * 8 / 2400 + 0.05
    x = synth.render_real(plan, 0, int(1.2 * rate))
    cap = tmp_path / "cap.f32"
    x.tofile(cap)
    r = run([exe, cap, *FM], {"ACARSDEC_B200_AIRRATE": str(rate), "ACARSDEC_B200_TAPS": str(taps)})
    assert r.returncode == 0, r.stderr
    with api.Context(K, 1, 4, len(x) // (1024 * K) + 2, flags=FLAG_REAL, taps=taps) as ctx:
        ctx.set_plan_air(0, fd)
        ctx.submit_real(x.reshape(1, -1))
        want = ctx_msgs(ctx)
    assert len(want) >= 10 and host_msgs(r.stdout) == want


@pytest.mark.gpu
@pytest.mark.parametrize("macro,variant", [("WITH_SOAPY", 0), ("WITH_SDRPLAY", 1)])
def test_cs16_taps_matches_library(tmp_path, native, macro, variant):
    K, taps = 160, 2 * 160 + 40
    exe = fehost(tmp_path, macro)
    cap, freqs = _cs16_capture(tmp_path, 23 + variant)
    env = {"ACARSDEC_B200_TAPS": str(taps), "ACARSDEC_B200_CAPTURE": str(cap)}
    r = run([exe, K, cap, *freqs] if macro == "WITH_SOAPY" else [exe, *freqs], env)
    assert r.returncode == 0, r.stderr
    x = np.fromfile(cap, dtype=np.int16).reshape(1, -1, 2)
    fd = [api.plan(K, [float(f)])[0][0] for f in freqs]
    with api.Context(K, 1, len(fd), x.shape[1] // (1024 * K) + 2, flags=FLAG_CS16, taps=taps) as ctx:
        ctx.set_plan_cs16(0, fd, variant)
        ctx.submit_cs16(x)
        want = ctx_msgs(ctx)
    assert len(want) >= 10 and host_msgs(r.stdout) == want


def _built_here(prog: str) -> bool:
    """oracle/_ref programs compile compat.c in; only a build from this tree's compat.c knows the variable."""
    p = REFBIN / prog
    return p.exists() and b"ACARSDEC_B200_TAPS" in p.read_bytes()


@pytest.mark.gpu
def test_unmodified_acarsdec_program_honours_taps(tmp_path, native):
    """The reference's own acarsdec.c linked against the shim (oracle/_ref/acarsdec_b200): with ACARSDEC_B200_TAPS set
    it prints (JSON) the messages the library context decodes; a bad value stops it."""
    if not _built_here("acarsdec_b200"):
        pytest.skip("oracle/_ref/acarsdec_b200 is absent or was built from a compat.c without ACARSDEC_B200_TAPS")
    import json
    K, taps = 160, 8 * 160
    fm = (131.525, 131.725, 131.825, 131.450, 131.550)
    fd, _, fc = api.plan(K, fm)
    plan = synth.make_plan(K, fm, fc, seconds=1.2, seed=78, text_len=(10, 60), msgs_per_chan_per_sec=3.0)
    nblk = synth.blocks_for_seconds(K, 1.2)
    iq = synth.render_blocks(plan, 0, nblk)
    cap = tmp_path / "cap.iq"
    iq.tofile(cap)
    prog = REFBIN / "acarsdec_b200"
    r = run([prog, "-o", "4", "-m", K, "-r", cap, *fm], {"ACARSDEC_B200_TAPS": str(taps), "ACARSDEC_B200_BLOCKS": "4"})
    assert r.returncode == 0, r.stderr
    printed = sorted(json.loads(l).get("text", "") for l in r.stdout.splitlines() if l.startswith("{"))
    with api.Context(K, 1, len(fm), nblk, taps=taps) as ctx:
        ctx.set_plan(0, fd)
        ctx.submit_host(iq.reshape(1, -1), nblk)
        ctx.sync()
        texts = []
        for m in ctx.drain():
            f = api.msg_fields(m)
            texts.append(bytes(m.txt[f.txt_off:f.txt_off + f.txt_len]).decode("latin-1") if f is not None else "")
    assert len(texts) >= 8 and printed == sorted(texts)
    bad = run([prog, "-o", "4", "-m", K, "-r", cap, *fm], {"ACARSDEC_B200_TAPS": "100"})
    assert bad.returncode != 0 and "ACARSDEC_B200_TAPS" in bad.stderr
