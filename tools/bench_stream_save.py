"""What moving streams costs (acb_save_streams / acb_load_streams).  Per shape:
  - wall time of saving 1 stream and all streams, and of loading them back (the call alone, and the call followed by the
    device work it queued), median of `reps` after one untimed round;
  - k_stream_pack / k_stream_unpack kernel times from a run under torch.profiler (CUDA activity), and their bytes/s
    (each byte of the packed state read once and written once) against the H100 SXM's 3.35 TB/s;
  - blob bytes per stream;
  - the step time (acb_mark / acb_elapsed_ms: first channelizer to last block FEC) of a submit right after a load of every
    stream against one without, alternated, median of `reps` each.
Shapes: the bench's (4224 streams x 8 channels, K = 160, device-resident u8 IQ) at taps = K and taps = 8K, and one CS16
stream with K = 1600, 256 channels and taps = 16K (its tables left at zeros: the times do not depend on their values).
The card's name, power limit and SM clocks are read in the same call with read-only queries.
Writes results/bench_stream_save_h100.json (or the path given) and prints the same JSON line.
  python tools/bench_stream_save.py [reps] [out.json]"""
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np
import torch

from acarsdec_b200 import api, synth

args = sys.argv[1:]
reps = int(args[0]) if len(args) > 0 else 5
out_path = Path(args[1]) if len(args) > 1 else ROOT / "results" / "bench_stream_save_h100.json"
HBM = 3.35e12
B = 8


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout
    return [v.strip() for v in out.strip().splitlines()[0].split(",")]


def u8_shape(taps_mult):
    K, S, POOL = 160, 4224, 4
    FM = synth.DEFAULT_FREQS_MHZ
    fd, _, fc = api.plan(K, FM)
    pool = np.stack([synth.render_blocks(synth.make_plan(K, FM, fc, seconds=B * 1024 / 12500, seed=1000 + p), 0, B).reshape(-1)
                     for p in range(POOL)])
    din = torch.from_numpy(pool).cuda().index_select(0, torch.arange(S, device="cuda") % POOL).contiguous()
    ctx = api.Context(K, S, len(FM), B, flags=1, taps=K * taps_mult if taps_mult > 1 else 0)
    for s in range(S):
        ctx.set_plan(s, fd)

    def submit():
        ctx.submit_device(din.data_ptr(), B, din.stride(0))
    return dict(K=K, streams=S, channels=len(FM), taps=K * taps_mult, input="device-resident u8 IQ"), ctx, submit, din


def cs16_shape():
    K, NCH, taps = 1600, 256, 16 * 1600
    ctx = api.Context(K, 1, NCH, 1, flags=4, taps=taps)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randint(-2000, 2000, (1, 1024 * K, 2), dtype=torch.int16, device="cuda", generator=g)

    def submit():
        ctx.submit_tensor(x)
    return dict(K=K, streams=1, channels=NCH, taps=taps, input="device-resident CS16, tables unplanned"), ctx, submit, x


def wall(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def measure(shape):
    meta, ctx, submit, keep = shape
    S = meta["streams"]
    for _ in range(3):
        submit()
    ctx.sync()
    one, every = [S // 2], list(range(S))
    out = dict(meta)
    blob1, blob_all = ctx.save_streams(one), ctx.save_streams(every)
    out["blob_bytes_per_stream"] = api.blob_info(blob_all).record_bytes
    out["blob_bytes_all"] = len(blob_all)
    res = {k: [] for k in ("save_1_ms", "save_all_ms", "load_1_call_ms", "load_1_done_ms", "load_all_call_ms", "load_all_done_ms")}
    for _ in range(reps):
        res["save_1_ms"].append(wall(lambda: ctx.save_streams(one)))
        res["save_all_ms"].append(wall(lambda: ctx.save_streams(every)))
        for n, lst, b in (("1", one, blob1), ("all", every, blob_all)):
            ctx.sync()
            t = time.perf_counter()
            ctx.load_streams(lst, b)
            res[f"load_{n}_call_ms"].append((time.perf_counter() - t) * 1e3)
            torch.cuda.synchronize()
            res[f"load_{n}_done_ms"].append((time.perf_counter() - t) * 1e3)
    out.update({k: statistics.median(v) for k, v in res.items()})
    # kernel times: one save and one load of every stream under the profiler
    from torch.profiler import ProfilerActivity, profile
    ctx.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            ctx.save_streams(every)
            ctx.load_streams(every, blob_all)
        torch.cuda.synchronize()
    kt = {}
    for e in prof.key_averages():
        for name in ("k_stream_pack", "k_stream_unpack"):
            if name in e.key:
                kt[name] = e.device_time_total / max(1, e.count)
    dev_bytes = S * (out["blob_bytes_per_stream"] - 32)     # the record less its host part (no statistics flags here)
    for name, us in kt.items():
        out[f"{name}_us"] = us
        out[f"{name}_GBps"] = 2 * dev_bytes / (us * 1e-6) / 1e9
        out[f"{name}_share_of_hbm"] = 2 * dev_bytes / (us * 1e-6) / HBM
    # the step after a load of every stream against one without, alternated
    steps = {"plain": [], "after_load": []}
    for _ in range(reps):
        for kind in ("plain", "after_load"):
            ctx.sync()
            ctx.mark(0)
            if kind == "after_load":
                ctx.load_streams(every, blob_all)
            submit()
            ctx.mark(1)
            steps[kind].append(ctx.elapsed_ms())
    ctx.sync()
    out["step_ms"] = statistics.median(steps["plain"])
    out["step_after_load_ms"] = statistics.median(steps["after_load"])
    ctx.close()
    del keep
    return out


def main():
    name, plimit, sm_max, sm_now = smi("name,power.limit,clocks.max.sm,clocks.sm")
    rows = [measure(u8_shape(1)), measure(u8_shape(8)), measure(cs16_shape())]
    _, _, _, sm_after = smi("name,power.limit,clocks.max.sm,clocks.sm")
    res = dict(gpu=name, power_limit_w=plimit, sm_clock_max_mhz=sm_max, sm_clock_mhz_before=sm_now, sm_clock_mhz_after=sm_after,
               reps=reps, hbm_peak_Bps=HBM, shapes=rows)
    out_path.parent.mkdir(parents=True, exist_ok=True)
    out_path.write_text(json.dumps(res) + "\n")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
