"""What ACB_FLAG_FREQ_STATS costs.  Step time with and without the flag, alternated in one session, three runs each, a run
being `steps` timed submits (the library's CUDA events from the first channelizer to the last block FEC, acb_mark /
acb_elapsed_ms) after `warmup` untimed ones on a fresh context.  Shapes:
  - the bench's device-resident shape: 4224 streams x 8 channels, K = 160, u8 IQ in HBM (acb_submit_device), exact and
    fast channelizer;
  - CS16 wideband: 8 streams x 256 channels, K = 1600, device-resident interleaved int16 (ACB_FLAG_FAST_WIDEBAND);
  - real wideband: 8 streams x 200 channels, K = 800, device-resident float32 (ACB_FLAG_FAST_WIDEBAND_REAL).
k_freq_in's own time comes from one more run per shape under torch.profiler (CUDA activity: the kernels' start and end
events), averaged per launch; its FMA rate counts 4 FMAs per complex sample (2 per real one) per chain over the 2*(K/2)
samples of every row, against 33.5 T FMA/s (the data sheet's 67 TFLOP/s FP32, H100 SXM).  The card's name, power limit
and SM clocks are read in the same call with read-only queries.  Writes results/bench_freq_stats_h100.json (or the path
given) and prints the same JSON line.
  python tools/bench_freq_stats.py [steps] [warmup] [out.json]"""
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np
import torch

from acarsdec_b200 import api, synth

args = sys.argv[1:]
steps = int(args[0]) if len(args) > 0 else 10
warmup = int(args[1]) if len(args) > 1 else 3
out_path = Path(args[2]) if len(args) > 2 else ROOT / "results" / "bench_freq_stats_h100.json"
B = 8


def fma_per_step(info, kind_real):
    K = info["K"]
    return B * 1024 * info["streams"] * info["channels"] * 2 * (K // 2) * (2 if kind_real else 4)


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout
    return [v.strip() for v in out.strip().splitlines()[0].split(",")]


def u8_shape():
    K, S, POOL = 160, 4224, 4
    FM = synth.DEFAULT_FREQS_MHZ
    fd, _, fc = api.plan(K, FM)
    pool = np.stack([synth.render_blocks(synth.make_plan(K, FM, fc, seconds=B * 1024 / 12500, seed=1000 + p), 0, B).reshape(-1)
                     for p in range(POOL)])
    din = torch.from_numpy(pool).cuda().index_select(0, torch.arange(S, device="cuda") % POOL).contiguous()

    def make(flags):
        ctx = api.Context(K, S, len(FM), B, flags=flags | 1)
        for s in range(S):
            ctx.set_plan(s, fd)
        return ctx

    def submit(ctx):
        ctx.submit_device(din.data_ptr(), B, din.stride(0))
    return dict(K=K, streams=S, channels=len(FM), input="device-resident u8 IQ, 4 synthetic streams tiled"), make, submit


def wide_shape(kind):
    K, S, NCH = (1600, 8, 256) if kind == "cs16" else (800, 8, 200)
    fm = tuple(round(129.0 + 0.025 * i, 3) for i in range(NCH))
    g = torch.Generator(device="cuda").manual_seed(5)
    n = B * 1024 * K
    if kind == "cs16":
        fd, _, fc = api.plan(K, fm)
        x = torch.randint(-3000, 3000, (S, n, 2), dtype=torch.int16, device="cuda", generator=g)
        flags = 4 | api.FLAG_FAST_WIDEBAND
    else:
        fd, fc, _ = api.air_plan(K * 12500, fm)
        x = (torch.rand((S, n), device="cuda", generator=g) - 0.5).to(torch.float32) * 0.2
        flags = 2 | api.FLAG_FAST_WIDEBAND_REAL

    def make(extra):
        ctx = api.Context(K, S, NCH, B, flags=flags | extra)
        for s in range(S):
            if kind == "cs16":
                ctx.set_plan_cs16(s, fd, 0, fc)
            else:
                ctx.set_plan_air_at(s, fd, fc)
        return ctx

    def submit(ctx):
        ctx.submit_tensor(x)
    return dict(K=K, streams=S, channels=NCH, input=f"device-resident {kind} noise, wideband form"), make, submit


def run(make, submit, flags) -> dict:
    ctx = make(flags)
    try:
        for _ in range(warmup):
            submit(ctx)
            ctx.drain_records()
        ctx.sync()
        ctx.drain_records()
        ctx.mark(0)
        for _ in range(steps):
            submit(ctx)
            ctx.drain_records()
        ctx.mark(1)
        ctx.sync()
        ctx.drain_records()
        return {"step_ms": round(ctx.elapsed_ms() / steps, 3)}
    finally:
        ctx.close()


def kernel_times(make, submit, flags) -> dict:
    ctx = make(flags)
    try:
        submit(ctx)
        ctx.sync()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                submit(ctx)
            ctx.sync()
        out = {}
        for e in prof.key_averages():
            if "k_freq" in e.key:
                out[e.key] = {"launches": e.count, "us_per_launch": round(e.device_time_total / max(1, e.count), 1)}
        return out
    finally:
        ctx.close()


name, plimit, smax = smi("name,power.limit,clocks.max.sm")
torch.cuda.synchronize()
results = {}
for label, shape, base in (("u8_exact", u8_shape, 0), ("u8_fast", u8_shape, 8),
                          ("cs16_wideband", lambda: wide_shape("cs16"), 0), ("real_wideband", lambda: wide_shape("real"), 0)):
    info, make, submit = shape()
    torch.cuda.synchronize()
    runs = {"off": [], "on": []}
    for rep in range(3):
        for mode in (("off", "on") if rep % 2 == 0 else ("on", "off")):
            runs[mode].append(run(make, submit, base | (api.FLAG_FREQ_STATS if mode == "on" else 0)))
    off = float(np.median([r["step_ms"] for r in runs["off"]]))
    on = float(np.median([r["step_ms"] for r in runs["on"]]))
    kt = kernel_times(make, submit, base | api.FLAG_FREQ_STATS)
    k_us = sum(v["us_per_launch"] for k, v in kt.items() if "k_freq_in" in k)
    fma = fma_per_step(info, label.startswith("real"))
    results[label] = {**info, "runs": runs, "median_step_ms_off": round(off, 3), "median_step_ms_on": round(on, 3),
                      "cost_percent": round(100 * (on - off) / off, 2), "freq_kernels": kt, "fma_per_step": fma,
                      "k_freq_in_tfma_per_s": round(fma / (k_us * 1e-6) / 1e12, 2) if k_us else None,
                      "k_freq_in_share_of_fp32_peak": round(fma / (k_us * 1e-6) / 33.5e12, 3) if k_us else None}
    del make, submit
    torch.cuda.empty_cache()

sm_now = smi("clocks.sm")[0]
line = json.dumps({"bench": "freq_stats", "gpu": name, "power_limit_w": float(plimit), "sm_clock_max_mhz": float(smax),
                   "sm_clock_after_run_mhz": float(sm_now), "blocks_per_step": B, "steps": steps, "warmup": warmup,
                   "results": results})
out_path.parent.mkdir(parents=True, exist_ok=True)
out_path.write_text(line + "\n")
print(line)
