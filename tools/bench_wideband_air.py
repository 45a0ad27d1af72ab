"""Cost of the real-input wideband fast form (ACB_FLAG_FAST_WIDEBAND_REAL) against the exact form and the narrow real-input
fast kernels (ACB_FLAG_FAST_CHANNELIZER at taps = K, ACB_FLAG_FAST_FILTER_REAL at taps > K), alternately in one run, on
float32 real host submits (acb_submit_real_host): K = 800 x 200 channels (a 10 MS/s receiver's whole band) at taps K, 2K,
8K and 16K; K = 1600 x 256 channels at taps K and 8K (no narrow kernel takes K = 1600); and K = 200 x 8 channels at taps K,
the narrow kernels' own shape.  K1 time from the library's CUDA events (acb_stats_t.chan_ms: the channelizer kernel alone),
after two warm-up submits, one sync per step.  The card's name, power limit and SM clock (sampled during each timed
window) are read in the same run with read-only queries.

Each row carries a lane-op model of FP32 work per input sample (a model, not a measurement) — exact: 4*C*taps_pad/K;
narrow: per group of 8 channels the quarter split (1.5), the MACs (6) and at taps > K the pre-sum (taps_pad/K);
wideband: the split and the pre-sum once (1.5 + taps_pad/K) and 0.75 per channel — and that count over the kernel time as
a fraction of the FP32 issue peak (132 SMs x 128 lanes x the sampled clock).  The envelope of 3 streams of each fast form
is checked against the exact form's at the timed size: |fast - exact| <= 1e-5*S per output row, S = sum |x||w| (bar (a)
of tests/test_wideband_real_oracle.py).  Prints one JSON line.
  python tools/bench_wideband_air.py [steps]"""
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np
from acarsdec_b200 import api

args = [a for a in sys.argv[1:] if not a.startswith("--")]
steps = int(args[0]) if args else 5
CHECK_STREAMS = 3
FLAG_REAL, FLAG_FAST, FLAG_FAST_FILTER_REAL = 2, 8, 32
FCR = 131_500_000
# (K, channels, taps multiple, streams, rows per submit, compared forms); the exact form is the reference of the check
SHAPES = [(800, 200, m, 8, 4096, ("exact", "narrow", "wideband")) for m in (1, 2, 8, 16)] + [
    (1600, 256, m, 4, 4096, ("exact", "wideband")) for m in (1, 8)] + [
    (200, 8, 1, 64, 2048, ("exact", "narrow", "wideband"))]


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout
    return [v.strip() for v in out.strip().splitlines()[0].split(",")]


def air_freqs(K, nch):
    """nch channels on the 12.5 kHz raster across the real band around FCR, every residue k mod 4 (as
    tests/test_wideband_real_oracle.py: air_freqs)"""
    D = K // 4 - 1
    d = np.rint(np.linspace(-D, D - 1, nch)).astype(np.int64)
    if nch > 1 and (2 * D - 1) / (nch - 1) >= 4:
        d -= (d - np.arange(nch)) % 4
    return [int(FCR + 12_500 * v) for v in d]


def exact_weights(K, taps, freqs, fc):
    L = api.load()
    wf = np.zeros((len(freqs), 2 * taps), dtype=np.float32)
    for i, f in enumerate(freqs):
        if taps > K:
            L.acb_air_build_wf_lp(f, fc, K * 12_500, taps, wf[i].ctypes.data)
        else:
            L.acb_air_build_wf(f, fc, K * 12_500, wf[i].ctypes.data)
    return np.abs(wf[:, 0::2].astype(np.float64) + 1j * wf[:, 1::2])


def row_totals(x, K, taps, w, nrows):
    """S = sum |x||w| per output row and channel, (nrows, nch); every submit is the same buffer of whole rows, so its
    tail is the history"""
    a = np.abs(x.astype(np.float64))
    xp = np.concatenate([a[len(a) - (taps - K):], a]) if taps > K else a
    win = np.lib.stride_tricks.sliding_window_view(xp, taps)[::K][:nrows]
    return win @ w.T


def lane_ops(form, K, C, taps_pad):
    R = taps_pad / K
    pre = R if taps_pad > K else 0.0
    if form == "exact":
        return 4 * C * R
    if form == "narrow":
        return -(-C // 8) * (1.5 + 6 + pre)
    return 1.5 + pre + 0.75 * C


name, plimit, maxclk = smi("name,power.limit,clocks.max.sm")
rows = []
for K, C, mult, S, nrows, forms in SHAPES:
    taps = mult * K
    taps_pad = K + (-(-(taps - K) // 4) * 4)
    freqs = air_freqs(K, C)
    host = (np.random.default_rng(K + taps).standard_normal((S, nrows * K)) * 100).astype(np.float32)
    env_ref, k1_ref, k1_narrow = None, None, None
    for form in forms:
        flags = FLAG_REAL | {"exact": 0, "narrow": FLAG_FAST if taps == K else FLAG_FAST_FILTER_REAL,
                             "wideband": api.FLAG_FAST_WIDEBAND_REAL}[form]
        ctx = api.Context(K, S, C, -(-nrows // 1024) + 1, flags=flags, taps=taps)
        fc = 0
        for s in range(S):
            fc = ctx.set_plan_air(s, freqs)
        step = lambda: ctx.submit_real(host)
        for _ in range(2):
            step()
            ctx.sync()
        ctx.drain_records()
        ctx.stats(reset=True)
        mon = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0", "-lms", "100"],
                               stdout=subprocess.PIPE, text=True)
        try:
            for _ in range(steps):
                step()
                ctx.sync()
        finally:
            mon.terminate()
            clk_out, _ = mon.communicate()
        clks = [float(v) for v in clk_out.split() if v.strip().replace(".", "", 1).isdigit()]
        clk = float(np.median(clks)) if clks else float(maxclk)
        st = ctx.stats()
        k1 = st.chan_ms / st.chan_launches
        env = ctx.read_dm(nrows)[:CHECK_STREAMS].copy()
        ctx.drain_records()
        ctx.close()
        ops = lane_ops(form, K, C, taps_pad)
        nsamp = S * nrows * K
        fp = ops * nsamp / (k1 * 1e-3) / (132 * 128 * clk * 1e6)
        row = {"K": K, "channels": C, "taps": taps, "streams": S, "rows_per_submit": nrows, "form": form,
               "k1_ms": round(k1, 4), "msamples_per_s": round(nsamp / k1 / 1e3, 1), "sm_clock_mhz_median": clk,
               "fp32_lane_ops_per_sample_model": round(ops, 2), "fp32_issue_fraction": round(fp, 4),
               "fast_chan_launches": int(st.fast_chan_launches), "chan_launches": int(st.chan_launches)}
        if form == "exact":
            env_ref, k1_ref = env, k1
        else:
            w = exact_weights(K, taps, freqs, fc)
            worst = 0.0
            for s in range(CHECK_STREAMS):
                Sb = row_totals(host[s], K, taps, w, nrows)
                worst = max(worst, float((np.abs(env[s].astype(np.float64) - env_ref[s]) / np.maximum(Sb, 1e-300)).max()))
            row.update({"speedup_vs_exact": round(k1_ref / k1, 2), "envelope_checked_streams": CHECK_STREAMS,
                        "max_err_over_S_vs_exact": worst, "envelope_within_1e-5_S": bool(worst <= 1e-5)})
            if form == "narrow":
                k1_narrow = k1
            elif k1_narrow is not None:
                row["speedup_vs_narrow"] = round(k1_narrow / k1, 2)
        rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
print(json.dumps({"bench": "wideband_air", "steps": steps, "input": "float32 real host submits (acb_submit_real_host)",
                  "gpu": name, "power_limit_w": float(plimit), "max_sm_clock_mhz": float(maxclk), "rows": rows}))
