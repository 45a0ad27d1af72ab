"""Cost of the overlapping-window channelizer (taps > K): K = 160, 8 channels, u8 IQ resident in device memory,
528 and 4224 streams, taps in {K, 2K, 4K, 8K, 16K} (taps = K is the reference's boxcar on the default kernel).
K1 time from the library's CUDA events (acb_stats_t.chan_ms, the channelizer plus, for taps > K, the copy of the
history), one sync per step so K1 runs alone.  FP32-issue fraction = 8*C*taps_pad/K lane-ops per complex sample over
132 SMs x 128 FP32 lanes x the SM clock sampled during the timed window.  The card's name, power limit and clocks are
read in the same run.  Prints one JSON line.
  python tools/bench_ovl.py [steps]

With --fast: the exact form and the polyphase fast form (ACB_FLAG_FAST_FILTER) alternately, taps in {2K, 4K, 8K, 16K},
same shape.  For the fast form each row also carries its algorithmic HBM bytes (the u8 input once, the envelope out)
and FP32 lane-ops (2*ceil(taps_pad/K) per component of the pre-sum plus the fold, split and K/8 MACs per channel, per
complex sample) as fractions of their peaks (3.35 TB/s; 132 SMs x 128 lanes x the sampled clock), the binding one
named, and the envelope of a few streams checked against the exact form's at the timed size: |fast - exact| <= 1e-5*S
per output row, S = sum |x||w| (bar (a) of tests/test_ovl_fast_oracle.py).
  python tools/bench_ovl.py [steps] --fast"""
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np
from acarsdec_b200 import api, synth

K, C, B = 160, 8, 8
args = [a for a in sys.argv[1:] if not a.startswith("--")]
steps = int(args[0]) if args else 5
FAST = "--fast" in sys.argv
HBM_PEAK = 3.35e12                     # H100 SXM5 80 GB HBM3, bytes/s
CHECK_STREAMS = 3                      # streams whose envelope is compared at the timed size


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
    runs = [(m, f) for m in (2, 4, 8, 16) for f in (False, True)] if FAST else [(m, False) for m in (1, 2, 4, 8, 16)]
    exact_env = {}
    for mult, fast in runs:
        taps = mult * K
        # ACB_FLAG_NO_INPUT_STAGING (1), + ACB_FLAG_FAST_FILTER (16) for the fast form
        ctx = api.Context(K, S, C, B, flags=1 | (16 if fast else 0), taps=0 if mult == 1 else taps)
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
        row = {"streams": S, "taps": taps, "taps_pad": taps_pad, "k1_ms": round(k1, 4),
               "gsamples_per_s": round(nsamp / k1 / 1e6, 2), "sm_clock_mhz_median": clk,
               "fp32_issue_fraction": round(ops / (k1 * 1e-3) / (132 * 128 * clk * 1e6), 4),
               "k1_ms_over_taps_eq_k": None, "fast_chan_launches": int(st.fast_chan_launches)}
        if FAST:
            row["form"] = "fast" if fast else "exact"
            env = np.empty((CHECK_STREAMS, B * 1024, C), dtype=np.float32)
            assert ctx.lib.acb_read_dm(ctx.h, env.ctypes.data, env.size) == 0
            if fast:
                R = -(-taps_pad // K)
                lane_ops = 2 * 2 * R + 3.25 + C / 2           # pre-sum (I, Q), fold + split, MACs
                hbm = 2 + 4 * C / K                           # u8 sample in, envelope out per complex sample
                fp = lane_ops * nsamp / (k1 * 1e-3) / (132 * 128 * clk * 1e6)
                mem = hbm * nsamp / (k1 * 1e-3) / HBM_PEAK
                row.update({"fp32_lane_ops_per_sample": lane_ops, "fp32_issue_fraction": round(fp, 4),
                            "hbm_bytes_per_sample": round(hbm, 3), "hbm_fraction": round(mem, 4),
                            "binding_roof": "fp32" if fp >= mem else "hbm",
                            "k1_ms_exact": exact_env[taps][1], "speedup_vs_exact": round(exact_env[taps][1] / k1, 2)})
                # bar (a) at the timed size: S = sum |x||w| per row from the exact form's table, in float64
                wf = api.build_wf_lp(K, taps, synth.DEFAULT_FREQS_MHZ).astype(np.float64)
                w = np.abs(wf[:, 0::2] + 1j * wf[:, 1::2])
                worst = 0.0
                for s in range(CHECK_STREAMS):
                    x = host[s].astype(np.float32) - np.float32(127.37)
                    ax = np.abs(x[0::2].astype(np.float64) + 1j * x[1::2])
                    xp = np.concatenate([ax[len(ax) - (taps - K):], ax])      # every submit is the same buffer: its tail is the history
                    win = np.lib.stride_tricks.sliding_window_view(xp, taps)[::K][:B * 1024]
                    Sb = win @ w.T
                    worst = max(worst, float((np.abs(env[s].astype(np.float64) - exact_env[taps][0][s]) / Sb).max()))
                row.update({"envelope_checked_streams": CHECK_STREAMS, "max_err_over_S_vs_exact": worst,
                            "envelope_within_1e-5_S": bool(worst <= 1e-5)})
            else:
                exact_env[taps] = (env, round(k1, 4))
        rows.append(row)
        ctx.device_free(d)
        ctx.close()
    if not FAST:
        base = [r for r in rows if r["streams"] == S and r["taps"] == K][0]["k1_ms"]
        for r in rows:
            if r["streams"] == S:
                r["k1_ms_over_taps_eq_k"] = round(r["k1_ms"] / base, 3)
print(json.dumps({"bench": "ovl_fast" if FAST else "ovl", "K": K, "channels": C, "blocks_per_submit": B, "steps": steps, "input": "u8 IQ, device-resident",
                  "gpu": name, "power_limit_w": float(plimit), "max_sm_clock_mhz": float(maxclk), "rows": rows}))
