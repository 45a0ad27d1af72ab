"""Cost of the ragged submits at the bench's device-resident shape (4224 streams x 8 channels).

    python tools/bench_ragged.py [--out results/bench_ragged_h100.json] [--rounds 3] [--steps 10]

For u8 IQ and CS16 at K = 160, real input at K = 200, and one wideband shape (u8, ACB_FLAG_FAST_WIDEBAND), it times four
ways of feeding the same context from device memory:
  (a) the lockstep call;
  (b) the ragged call with every count equal;
  (c) counts spread +-10 % around the lockstep count (the channelizer still runs the largest);
  (d) the lockstep count with 1 % of the streams stalled (count 0).
Streaming counts are whole rows (multiples of K), so the carries stay 0 and (a) stays the lockstep path between the
others.  Per scenario: K1 and K2+K3 device time per submit (the context's CUDA-event counters, acb_get_stats) and the step
(wall time per submit over `steps` submits ending in acb_sync).  The scenarios alternate within each of `rounds` rounds;
the medians are reported, with the card's name, power limit and clock read in the same run.  `wasted_rows` is the
share of the channelizer's rows no stream reads: sum over streams of (largest - own) / (streams x largest).
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from acarsdec_b200 import api  # noqa: E402

S, NCH = 4224, 8
FM = (131.525, 131.550, 131.575, 131.600, 131.625, 131.650, 131.675, 131.700)
SHAPES = [  # name, kind, K, flags, rows per step (lockstep), max_blocks
    ("u8", "u8", 160, 1, 8 * 1024, 9),                 # ACB_FLAG_NO_INPUT_STAGING: device input only
    ("cs16", "cs16", 160, 4, 3 * 1024, 4),
    ("real", "real", 200, 2, 3 * 1024, 4),
    ("u8_wideband", "u8", 160, 1 | 64, 8 * 1024, 9),
]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [x.strip() for x in q[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def counts_for(scenario, rows, rng, unit_rows):
    """Per-stream counts in rows (u8: multiples of 1024, streaming: any)."""
    n = rows // unit_rows
    if scenario in ("a", "b"):
        c = np.full(S, n)
    elif scenario == "c":
        c = np.clip(np.round(n * rng.uniform(0.9, 1.1, S)), 1, None).astype(np.int64)
    else:
        c = np.full(S, n)
        c[rng.choice(S, S // 100, replace=False)] = 0
    return c * unit_rows


def run_shape(name, kind, K, flags, rows, maxblk, steps, warmup, rounds):
    import torch
    ctx = api.Context(K, S, NCH, maxblk, flags=flags)
    if kind == "u8":
        fd, _, fc = api.plan(K, FM)
        for s in range(S):
            ctx.set_plan_at(s, fd, fc)
    elif kind == "real":
        fd, fc, _ = api.air_plan(K * 12500, [round(f - 0.125, 3) for f in FM])
        for s in range(S):
            ctx.set_plan_air_at(s, fd, fc)
    else:
        fd, _, fc = api.plan(K, FM)
        for s in range(S):
            ctx.set_plan_cs16(s, fd, 0, fc)
    rmax = int(rows * 1.1) + 1024
    g = torch.Generator(device="cuda").manual_seed(1)
    if kind == "u8":
        width = (rmax // 1024 + 1) * 1024 * K * 2
        x = torch.randint(0, 256, (S, width), dtype=torch.uint8, device="cuda", generator=g)
    elif kind == "real":
        x = torch.randn((S, rmax * K), device="cuda", generator=g)
    else:
        x = torch.randint(-2000, 2000, (S, rmax * K, 2), dtype=torch.int16, device="cuda", generator=g)
    torch.cuda.synchronize()
    unit = 1024 if kind == "u8" else 1
    rng = np.random.default_rng(5)

    def submit(scen, c):
        if kind == "u8":
            if scen == "a":
                ctx.submit_device(x.data_ptr(), int(c[0]) // 1024, x.stride(0))
            else:
                ctx.submit_device(x.data_ptr(), 0, x.stride(0), counts=c // 1024)
        elif scen == "a":
            ctx.submit_tensor(x[:, :int(c[0]) * K])
        else:
            ctx.submit_tensor(x, counts=c * K)

    res = {s: {"k1_ms": [], "k2_ms": [], "step_ms": [], "wasted_rows": None} for s in "abcd"}
    for _ in range(rounds):
        for scen in "abcd":
            cs = [counts_for(scen, rows, rng, unit) for _ in range(warmup + steps)]
            for c in cs[:warmup]:
                submit(scen, c)
            ctx.sync()
            ctx.drain_records()
            ctx.stats(reset=True)
            t0 = time.perf_counter()
            for c in cs[warmup:]:
                submit(scen, c)
            ctx.sync()
            dt = (time.perf_counter() - t0) * 1e3 / steps
            st = ctx.stats(reset=True)
            ctx.drain_records()
            res[scen]["k1_ms"].append(st.chan_ms / steps)
            res[scen]["k2_ms"].append(st.demod_ms / steps)
            res[scen]["step_ms"].append(dt)
            w = [float((c.max() - c).sum()) / (S * c.max()) for c in cs[warmup:]]
            res[scen]["wasted_rows"] = float(np.mean(w))
    ctx.close()
    out = {"kind": kind, "K": K, "flags": flags, "streams": S, "channels": NCH, "rows_per_step": rows}
    for scen, r in res.items():
        out[scen] = {k: (statistics.median(v) if isinstance(v, list) else v) for k, v in r.items()}
        out[scen]["runs_step_ms"] = r["step_ms"]
    out["b_vs_a_step"] = out["b"]["step_ms"] / out["a"]["step_ms"] - 1
    out["c_vs_a_k1"] = out["c"]["k1_ms"] / out["a"]["k1_ms"] - 1
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(s[0] for s in SHAPES))
    a = ap.parse_args()
    result = {"tool": "tools/bench_ragged.py", **gpu_info(), "shapes": []}
    for name, kind, K, flags, rows, maxblk in SHAPES:
        if name in a.shapes.split(","):
            r = run_shape(name, kind, K, flags, rows, maxblk, a.steps, a.warmup, a.rounds)
            r["name"] = name
            result["shapes"].append(r)
            print(json.dumps(r), flush=True)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(result) + "\n")


if __name__ == "__main__":
    main()
