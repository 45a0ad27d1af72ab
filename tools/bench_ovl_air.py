"""Cost of the overlapping-window channel filter for real input (air.c front-end, float32 samples): the exact form
(ACB_FLAG_REAL_INPUT) and the polyphase fast form (+ ACB_FLAG_FAST_FILTER_REAL) alternately, K = 200 and 800, 8 channels,
taps in {2K, 4K, 8K, 16K}.  64 streams, 8 blocks per submit at K = 200 and 2 at K = 800: 105 M samples = 420 MB of input
per submit, far above the 50 MB L2, so every step reads its input from HBM; 512 1024-row blocks, about four per SM.  K1 time from the library's CUDA events
(acb_stats_t.chan_ms: the channelizer kernel alone; the host-to-device copy runs before it on its own stream), after two
warm-up submits, one sync per step so K1 runs alone.  The card's name, power limit and the SM clock sampled during each
timed window are read in the same run.

Each row carries the algorithm's FP32 lane-ops per sample (exact: 4*C*taps_pad/K; fast: ceil(taps_pad/K) pre-sum FMAs
plus the real-row DFT's 1.5 additions and 0.5 (k even) or 1 (k odd) MAC lane-ops per channel) and HBM bytes per sample
(4 in, 4*C/K out) as fractions of their peaks (132 SMs x 128 lanes x the sampled clock; 3.35 TB/s), the binding one named.
The fast envelope of a few streams is checked against the exact one at the timed size: |fast - exact| <= 1e-5*S per
output row, S = sum |x||w| (bar (a) of tests/test_ovl_fast_real_oracle.py).  Prints one JSON line.
  python tools/bench_ovl_air.py [steps]"""
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np
from acarsdec_b200 import api, synth

C = 8
SHAPES = {200: (64, 8), 800: (64, 2)}     # K: (streams, blocks per submit)
args = [a for a in sys.argv[1:] if not a.startswith("--")]
steps = int(args[0]) if args else 5
HBM_PEAK = 3.35e12                     # H100 SXM5 80 GB HBM3, bytes/s
CHECK_STREAMS = 3                      # streams whose envelope is compared at the timed size
FLAG_REAL, FLAG_FAST_FILTER_REAL = 2, 32


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout
    return [v.strip() for v in out.strip().splitlines()[0].split(",")]


def kbins(K, fd, fc):
    f = np.asarray(fd, dtype=np.uint32)
    k = np.zeros(len(f), dtype=np.int32)
    assert api.load().acb_fast_plan_air(f.ctypes.data, len(f), K, fc, k.ctypes.data, None) == 1
    return k


name, plimit, maxclk = smi("name,power.limit,clocks.max.sm")
fm = synth.DEFAULT_FREQS_MHZ[:C]
rows = []
for K, (S, B) in SHAPES.items():
    fd, fc, _ = api.air_plan(K * 12500, fm)
    k = kbins(K, fd, fc)
    n = B * 1024 * K
    host = (np.random.default_rng(K).standard_normal((S, n)) * 100).astype(np.float32)
    exact_env = {}
    for mult in (2, 4, 8, 16):
        for fast in (False, True):
            taps = mult * K
            ctx = api.Context(K, S, C, B, flags=FLAG_REAL | (FLAG_FAST_FILTER_REAL if fast else 0), taps=taps)
            for s in range(S):
                ctx.set_plan_air(s, fd)
            for _ in range(2):
                ctx.submit_real(host)
                ctx.sync()
            ctx.drain_records()
            ctx.stats(reset=True)
            mon = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0", "-lms", "100"],
                                   stdout=subprocess.PIPE, text=True)
            try:
                for _ in range(steps):
                    ctx.submit_real(host)
                    ctx.sync()
            finally:
                mon.terminate()
                clk_out, _ = mon.communicate()
            clks = [float(v) for v in clk_out.split() if v.strip().replace(".", "", 1).isdigit()]
            clk = float(np.median(clks)) if clks else float(maxclk)
            st = ctx.stats()
            k1 = st.chan_ms / st.chan_launches
            env = np.empty((CHECK_STREAMS, B * 1024, C), dtype=np.float32)
            assert ctx.lib.acb_read_dm(ctx.h, env.ctypes.data, env.size) == 0
            ctx.drain_records()
            ctx.close()
            taps_pad = K + (-(-(taps - K) // 4) * 4)
            nsamp = S * n
            R = -(-taps_pad // K)
            lane_ops = R + 1.5 + float(sum(0.5 if kk % 2 == 0 else 1.0 for kk in k)) if fast else 4 * C * taps_pad / K
            hbm = 4 + 4 * C / K
            fp = lane_ops * nsamp / (k1 * 1e-3) / (132 * 128 * clk * 1e6)
            mem = hbm * nsamp / (k1 * 1e-3) / HBM_PEAK
            row = {"K": K, "streams": S, "blocks_per_submit": B, "taps": taps, "taps_pad": taps_pad, "form": "fast" if fast else "exact",
                   "k1_ms": round(k1, 4), "gsamples_per_s": round(nsamp / k1 / 1e6, 2), "sm_clock_mhz_median": clk,
                   "fp32_lane_ops_per_sample": lane_ops, "fp32_issue_fraction": round(fp, 4),
                   "hbm_bytes_per_sample": round(hbm, 3), "hbm_fraction": round(mem, 4),
                   "binding_roof": "fp32" if fp >= mem else "hbm", "fast_chan_launches": int(st.fast_chan_launches)}
            if fast:
                row.update({"k1_ms_exact": exact_env[taps][1], "speedup_vs_exact": round(exact_env[taps][1] / k1, 2)})
                # bar (a) at the timed size: S = sum |x||w| per row from the exact form's table, in float64; every submit
                # is the same buffer, so its tail is the history of the next
                wf = api.build_wf_air_lp(K * 12500, taps, fm).astype(np.float64)
                w = np.abs(wf[:, 0::2] + 1j * wf[:, 1::2])
                worst = 0.0
                for s in range(CHECK_STREAMS):
                    ax = np.abs(host[s].astype(np.float64))
                    xp = np.concatenate([ax[len(ax) - (taps - K):], ax])
                    win = np.lib.stride_tricks.sliding_window_view(xp, taps)[::K][:B * 1024]
                    Sb = win @ w.T
                    worst = max(worst, float((np.abs(env[s].astype(np.float64) - exact_env[taps][0][s]) / Sb).max()))
                row.update({"envelope_checked_streams": CHECK_STREAMS, "max_err_over_S_vs_exact": worst,
                            "envelope_within_1e-5_S": bool(worst <= 1e-5)})
            else:
                exact_env[taps] = (env, round(k1, 4))
            rows.append(row)
print(json.dumps({"bench": "ovl_air_fast", "channels": C, "steps": steps,
                  "input": "float32 real (air.c), host submits", "gpu": name, "power_limit_w": float(plimit),
                  "max_sm_clock_mhz": float(maxclk), "rows": rows}))
