"""Wide-stream multi-GPU case for the streaming front-ends through acarsdec_b200.wide.WideStream (kind "real" and "cs16"):
ONE stream, channels split across ranks, one broadcast per submit, every rank appending the broadcast samples with the
device submits, messages merged in emission-group order.  On rank 0 the merged messages must equal one context's over
the whole stream, message for message and in order; at taps = K without fast flags they must also be the CPU oracle's.
Run under torchrun (or alone: world size 1)."""
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import torch  # noqa: E402

import refs  # noqa: E402
from acarsdec_b200 import api, sharding, synth, wide  # noqa: E402
from common import msg_tuple  # noqa: E402

FLAG_REAL, FLAG_CS16, FAST_WIDEBAND, FAST_WIDEBAND_REAL = 2, 4, 64, 128
NCH, MAXBLK = 24, 2
# (kind, taps relative to K, wideband flag): the wideband forms at taps = K and > K, the exact form at taps = K
CASES = [("cs16", "eq", True), ("cs16", "gt", True), ("cs16", "eq", False),
         ("real", "eq", True), ("real", "gt", True), ("real", "eq", False)]
GROUPS = {"cs16": (sharding.GROUP_OUTPUTS, 700), "real": (sharding.GROUP_INPUT, 65536)}


def _signal(kind):
    K = 200 if kind == "real" else 160
    rate = K * 12500
    fm = tuple((131.100 if kind == "real" else 130.000) + 0.025 * i for i in range(NCH))
    if kind == "real":
        fd, fc, _ = api.air_plan(rate, fm)
    else:
        fd, _, fc = api.plan(K, fm)
    # three ragged submits: the middle one completes no row
    sizes = [1024 * K + 3 * K // 2, K // 3, 2 * 1024 * K - 7]
    n = sum(sizes)
    p = synth.make_plan(K, fm, fc, seconds=n / rate, seed=61, msgs_per_chan_per_sec=10.0, text_len=(5, 25), amp=(8.0, 14.0))
    if kind == "real":
        x = synth.render_real(synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, bursts=p.bursts, seed=p.seed), 0, n)
    else:
        x = synth.render_cs16(p, 0, n)
    return K, fm, fd, fc, sizes, x


def _key(m):
    return (m.chn, m.len, m.err, bytes(m.txt[:m.len]), bytes(m.crc), int(np.float32(m.lvl).view(np.uint32)), int(m.pos))


def _one_context(kind, K, fd, fc, taps, flags, sizes, x):
    kflag = FLAG_REAL if kind == "real" else FLAG_CS16
    with api.Context(K, 1, len(fd), MAXBLK, device=0, flags=flags | kflag, taps=taps) as ctx:
        ctx.set_plan_air_at(0, fd, fc) if kind == "real" else ctx.set_plan_cs16(0, fd, 0, fc)
        ctx.set_emission_groups(*GROUPS[kind])
        at, rows = 0, []
        for n in sizes:
            part = x[None, at:at + n]
            rows.append(ctx.submit_real(part) if kind == "real" else ctx.submit_cs16(part))
            at += n
        ctx.sync()
        return [_key(m) for m in ctx.drain()], rows


def _oracle(kind, K, fm, fd, fc, x):
    orc = refs.OracleLib()
    nout = len(x) // K
    if kind == "real":
        dm = orc.channelize_real(x[:nout * K], K, orc.air_wf(K * 12500, fm))
    else:
        dm = orc.channelize_cs16(0, x[:nout * K], K, orc.cs16_osc(0, K, fd, fc))
    sink = refs.Sink()
    for c in range(len(fm)):
        orc.demod(orc.new_chan(c), dm[c], sink)
    return sorted(msg_tuple(f) for f in (orc.fec(m) for m in sink.msgs()) if f is not None)


def main():
    dist, rank, world, local = sharding.init_process_group()
    torch.cuda.set_device(local)
    results = []
    for kind, rel, wb in CASES:
        K, fm, fd, fc, sizes, x = _signal(kind)
        taps = 2 * K + 3 if rel == "gt" else 0
        flags = (FAST_WIDEBAND_REAL if kind == "real" else FAST_WIDEBAND) if wb else 0
        # the centre is chosen inside WideStream, once over all channels
        ws = wide.WideStream(dist, rank, world, local, K, fd, None, max_blocks=MAXBLK, taps=taps, flags=flags, kind=kind,
                             group=GROUPS[kind])
        assert ws.fc_hz == fc
        at, rows = 0, []
        for n in sizes:
            rows.append(ws.submit(x[at:at + n] if rank == 0 else None, n))
            at += n
        ws.sync()
        merged = ws.gather()
        if ws.ctx is not None and wb:
            assert ws.ctx.stats().fast_chan_launches > 0
        ws.close()
        if rank == 0:
            got = [(m[2],) + m[4:] + (m[3],) for m in merged]     # (chn, len, err, txt, crc, lvl bits, pos)
            want, want_rows = _one_context(kind, K, fd, fc, taps, flags, sizes, x)
            checks = {"rows": rows == want_rows and 0 in rows, "one_context": got == want, "frames": len(want) >= 5}
            if not wb and rel == "eq":
                checks["oracle"] = sorted(g[:6] for g in got) == _oracle(kind, K, fm, fd, fc, x)
            results.append({"kind": kind, "taps": taps, "wideband": wb, "frames": len(got), "checks": checks,
                            "match": all(checks.values())})
    if rank == 0:
        print(json.dumps({"world": world, "cases": results, "match": all(r["match"] for r in results)}), flush=True)
        assert all(r["match"] for r in results), results
    if dist is not None:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
