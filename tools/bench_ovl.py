"""Cost of the overlapping-window channelizer (taps > K): K = 160, 8 channels, u8 IQ resident in device memory,
528 and 4224 streams, taps in {K, 2K, 4K, 8K, 16K} (taps = K is the reference's boxcar on the default kernel).
K1 time from the library's CUDA events (acb_stats_t.chan_ms, the channelizer plus, for taps > K, the copy of the
history), one sync per step so K1 runs alone.  FP32-issue fraction = 8*C*taps_pad/K lane-ops per complex sample over
132 SMs x 128 FP32 lanes x the SM clock sampled during the timed window.  The card's name, power limit and clocks are
read in the same run.  Prints one JSON line.
  python tools/bench_ovl.py [steps]"""
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np
from acarsdec_b200 import api, synth

K, C, B = 160, 8, 8
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout
    return [v.strip() for v in out.strip().splitlines()[0].split(",")]


name, plimit, maxclk = smi("name,power.limit,clocks.max.sm")
fd = [int(f) for f in api.plan(K, synth.DEFAULT_FREQS_MHZ)[0]]
stride = B * 2048 * K
rows = []
for S in (528, 4224):
    host = np.random.default_rng(S).integers(0, 256, size=(S, stride), dtype=np.uint8)
    for mult in (1, 2, 4, 8, 16):
        taps = mult * K
        ctx = api.Context(K, S, C, B, flags=1, taps=0 if mult == 1 else taps)     # ACB_FLAG_NO_INPUT_STAGING
        for s in range(S):
            ctx.set_plan(s, fd)
        d = ctx.device_alloc(S * stride)
        ctx.copy_to_device(d, host)
        for _ in range(2):
            ctx.submit_device(d, B, stride)
            ctx.sync()
        ctx.drain_records()
        ctx.stats(reset=True)
        mon = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0", "-lms", "100"],
                               stdout=subprocess.PIPE, text=True)
        try:
            for _ in range(steps):
                ctx.submit_device(d, B, stride)
                ctx.sync()
        finally:
            mon.terminate()
            clk_out, _ = mon.communicate()
        clks = [float(v) for v in clk_out.split() if v.strip().replace(".", "", 1).isdigit()]
        clk = float(np.median(clks)) if clks else float(maxclk)
        st = ctx.stats()
        k1 = st.chan_ms / st.chan_launches
        taps_pad = K + (-(-(taps - K) // 8) * 8) if taps > K else K
        nsamp = S * B * 1024 * K
        ops = 8 * C * taps_pad / K * nsamp
        rows.append({"streams": S, "taps": taps, "taps_pad": taps_pad, "k1_ms": round(k1, 4),
                     "gsamples_per_s": round(nsamp / k1 / 1e6, 2), "sm_clock_mhz_median": clk,
                     "fp32_issue_fraction": round(ops / (k1 * 1e-3) / (132 * 128 * clk * 1e6), 4),
                     "k1_ms_over_taps_eq_k": None, "fast_chan_launches": int(st.fast_chan_launches)})
        ctx.device_free(d)
        ctx.close()
    base = [r for r in rows if r["streams"] == S and r["taps"] == K][0]["k1_ms"]
    for r in rows:
        if r["streams"] == S:
            r["k1_ms_over_taps_eq_k"] = round(r["k1_ms"] / base, 3)
print(json.dumps({"bench": "ovl", "K": K, "channels": C, "blocks_per_submit": B, "steps": steps, "input": "u8 IQ, device-resident",
                  "gpu": name, "power_limit_w": float(plimit), "max_sm_clock_mhz": float(maxclk), "rows": rows}))
