"""What ACB_FLAG_DECODE_STATS costs: the step time of the bench's device-resident shape (4224 streams x 8 channels, K = 160,
input resident in HBM, acb_submit_device, one drain per step) with and without the flag, exact and fast channelizer.
The two are alternated in one session, three runs each; a run is `steps` timed submits (the library's CUDA events from
the first channelizer to the last block FEC, acb_mark / acb_elapsed_ms) after `warmup` untimed ones, on a fresh
context.  Each run also reports the isolated K2 + K3 time (acb_stats_t.demod_ms per launch, one submit at a time).  The
card's name and power limit are read in the same call with read-only queries.  Prints one JSON line.
  python tools/bench_decode_stats.py [steps] [warmup] [blocks]"""
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np
import torch

from acarsdec_b200 import api, synth

args = [int(a) for a in sys.argv[1:]]
steps = args[0] if len(args) > 0 else 10
warmup = args[1] if len(args) > 1 else 3
B = args[2] if len(args) > 2 else 8
K, S, POOL = 160, 4224, 4
FM = synth.DEFAULT_FREQS_MHZ


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout
    return [v.strip() for v in out.strip().splitlines()[0].split(",")]


name, plimit = smi("name,power.limit")
fd, _, fc = api.plan(K, FM)
pool = np.stack([synth.render_blocks(synth.make_plan(K, FM, fc, seconds=B * 1024 / 12500, seed=1000 + p), 0, B).reshape(-1)
                 for p in range(POOL)])
din = torch.from_numpy(pool).cuda().index_select(0, torch.arange(S, device="cuda") % POOL).contiguous()
stride = din.stride(0)
torch.cuda.synchronize()                  # the contexts' streams are not ordered behind torch's


def run(fast: bool, stats: bool) -> dict:
    flags = 1 | (8 if fast else 0) | (api.FLAG_DECODE_STATS if stats else 0)
    with api.Context(K, S, len(FM), B, flags=flags) as ctx:
        for s in range(S):
            ctx.set_plan(s, fd)
        for _ in range(warmup):
            ctx.submit_device(din.data_ptr(), B, stride)
            ctx.drain_records()
        ctx.sync()
        ctx.drain_records()
        ctx.stats(reset=True)
        frames = 0
        ctx.mark(0)
        for _ in range(steps):
            ctx.submit_device(din.data_ptr(), B, stride)
            frames += len(ctx.drain_records())
        ctx.mark(1)
        ctx.sync()
        frames += len(ctx.drain_records())
        step_ms = ctx.elapsed_ms() / steps
        st = ctx.stats(reset=True)
        for _ in range(3):
            ctx.submit_device(din.data_ptr(), B, stride)
            ctx.sync()
        ctx.drain_records()
        iso = ctx.stats(reset=True)
        out = {"step_ms": round(step_ms, 3), "k2_k3_iso_ms": round(iso.demod_ms / max(1, iso.demod_launches), 3),
               "host_ms_per_step": round(st.host_ms / steps, 3), "frames": frames}
        if stats:
            d = ctx.decode_stats()
            out["delivered_counted"] = int(d["delivered"].sum())
        return out


results = {}
for channelizer in ("exact", "fast"):
    runs = {"off": [], "on": []}
    for rep in range(3):
        for mode in (("off", "on") if rep % 2 == 0 else ("on", "off")):
            runs[mode].append(run(channelizer == "fast", mode == "on"))
    off = np.median([r["step_ms"] for r in runs["off"]])
    on = np.median([r["step_ms"] for r in runs["on"]])
    results[channelizer] = {"runs": runs, "median_step_ms_off": round(float(off), 3), "median_step_ms_on": round(float(on), 3),
                            "cost_percent": round(float(100 * (on - off) / off), 2)}

print(json.dumps({"bench": "decode_stats", "gpu": name, "power_limit_w": float(plimit), "K": K, "streams": S,
                  "channels": len(FM), "blocks_per_step": B, "steps": steps, "warmup": warmup,
                  "input": "device-resident u8 IQ (acb_submit_device), 4 distinct synthetic streams tiled over 4224",
                  "results": results}))
