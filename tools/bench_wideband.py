"""Cost of the wideband fast form (ACB_FLAG_FAST_WIDEBAND) against the exact form, alternately, on the shapes it is for:
u8 K = 1600 x 256 channels at taps K, 2K, 8K and 16K and K = 192 x 64 channels (device-resident input), CS16 K = 800 x 128
channels (host input), and K = 160 x 8 channels where the narrow kernel (ACB_FLAG_FAST_CHANNELIZER) also runs.  K1 time
from the library's CUDA events (acb_stats_t.chan_ms: the channelizer kernel alone), after two warm-up submits, one sync
per step.  The card's name, power limit and SM clock (sampled during each timed window) are read in the same run with
read-only queries.

Each row carries the algorithm's FP32 lane-ops per complex sample — exact: 8*C*R (R = taps_pad/K); wideband: the pre-sum
2*ceil(R) (taps > K), about 3.25 for the fold and split, and C/2 for the MACs (4 FMAs per channel per K/8 of the row) —
and that count over the kernel time as a fraction of the FP32 issue peak (132 SMs x 128 lanes x the sampled clock).  The
envelope of 3 streams is checked against the exact form's at the timed size: |fast - exact| <= 1e-5*S per output row,
S = sum |x||w| (bar (a) of tests/test_wideband_oracle.py).  Prints one JSON line.
  python tools/bench_wideband.py [steps]"""
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
FLAG_CS16, FLAG_FAST = 4, 8
FC = 120_000_000
# (kind, K, channels, taps multiple, streams, blocks per submit (u8) / rows per submit (CS16), compared forms)
SHAPES = [("u8", 1600, 256, m, 8, 2, ("exact", "wideband")) for m in (1, 2, 8, 16)] + [
    ("u8", 192, 64, 1, 64, 4, ("exact", "wideband")),
    ("cs16", 800, 128, 1, 16, 4096, ("exact", "wideband")),
    ("u8", 160, 8, 1, 256, 4, ("exact", "narrow", "wideband"))]


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout
    return [v.strip() for v in out.strip().splitlines()[0].split(",")]


def raster(K, nch):
    step = max(1, (K // 2 - 4) // (2 * nch + 2))
    return [FC + 25_000 * step * (i // 2 + 1) * (1 if i % 2 == 0 else -1) for i in range(nch)]


def exact_tables(kind, K, taps, freqs):
    L = api.load()
    wf = np.zeros((len(freqs), 2 * taps), dtype=np.float32)
    for i, f in enumerate(freqs):
        if kind == "u8":
            fr = L.acb_stored_fr(f)
            (L.acb_build_wf_lp(fr, FC, K, taps, wf[i].ctypes.data) if taps > K else L.acb_build_wf(fr, FC, K, wf[i].ctypes.data))
        else:
            (L.acb_cs16_build_wf_lp(0, f, FC, K, taps, wf[i].ctypes.data) if taps > K else L.acb_cs16_build_wf(0, f, FC, K, wf[i].ctypes.data))
    return np.abs(wf[:, 0::2].astype(np.float64) + 1j * wf[:, 1::2])


def row_totals(kind, x, K, taps, w, nrows):
    """S = sum |x||w| per output row and channel, (nrows, nch); every submit is the same buffer, so its tail is the history"""
    if kind == "u8":
        ax = np.abs(x[0::2].astype(np.float32) - np.float32(127.37)) + 1j * np.abs(x[1::2].astype(np.float32) - np.float32(127.37))
        if taps == K:
            ax = np.abs(x[0::2].astype(np.float64) - 127.5) + 1j * np.abs(x[1::2].astype(np.float64) - 127.5)
    else:
        ax = np.abs(x[:, 0].astype(np.float64)) + 1j * np.abs(x[:, 1].astype(np.float64))
    a = np.abs(ax.real + 1j * ax.imag)
    xp = np.concatenate([a[len(a) - (taps - K):], a]) if taps > K else a
    win = np.lib.stride_tricks.sliding_window_view(xp, taps)[::K][:nrows]
    return win @ w.T


name, plimit, maxclk = smi("name,power.limit,clocks.max.sm")
rows = []
for kind, K, C, mult, S, B, forms in SHAPES:
    taps = mult * K
    freqs = raster(K, C)
    rng = np.random.default_rng(K + taps)
    if kind == "u8":
        host = rng.integers(0, 256, size=(S, B * 2048 * K), dtype=np.uint8)
        nrows = B * 1024
    else:
        host = rng.integers(-32768, 32768, size=(S, B * K, 2), dtype=np.int16)
        nrows = B
    env_ref, k1_ref = None, None
    for form in forms:
        flags = {"exact": 0, "narrow": FLAG_FAST, "wideband": api.FLAG_FAST_WIDEBAND}[form]
        if kind == "cs16":
            flags |= FLAG_CS16
        ctx = api.Context(K, S, C, B if kind == "u8" else -(-B // 1024) + 1, flags=flags, taps=taps)
        dev = None
        for s in range(S):
            if kind == "u8":
                ctx.set_plan_at(s, freqs, FC)
            else:
                ctx.set_plan_cs16(s, freqs, 0, FC)
        if kind == "u8":
            dev = ctx.device_alloc(host.nbytes)
            ctx.copy_to_device(dev, host)
            step = lambda: ctx.submit_device(dev, B, host.shape[1])
        else:
            step = lambda: ctx.submit_cs16(host)
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
        if dev is not None:
            ctx.device_free(dev)
        ctx.close()
        per_unit = 8 if kind == "u8" else 4
        taps_pad = K + (-(-(taps - K) // per_unit) * per_unit)
        R = taps_pad / K
        if form == "exact":
            lane_ops = 8 * C * R
        else:
            lane_ops = (2 * -(-taps_pad // K) if taps > K else 0) + 3.25 + C / 2
        nsamp = S * nrows * K
        fp = lane_ops * nsamp / (k1 * 1e-3) / (132 * 128 * clk * 1e6)
        row = {"kind": kind, "K": K, "channels": C, "taps": taps, "streams": S, "rows_per_submit": nrows, "form": form,
               "k1_ms": round(k1, 4), "gsamples_per_s": round(nsamp / k1 / 1e6, 2), "sm_clock_mhz_median": clk,
               "fp32_lane_ops_per_sample": round(lane_ops, 2), "fp32_issue_fraction": round(fp, 4),
               "fast_chan_launches": int(st.fast_chan_launches)}
        if form == "exact":
            env_ref, k1_ref = env, k1
        else:
            w = exact_tables(kind, K, taps, freqs)
            worst = 0.0
            for s in range(CHECK_STREAMS):
                Sb = row_totals(kind, host[s], K, taps, w, nrows)
                worst = max(worst, float((np.abs(env[s].astype(np.float64) - env_ref[s]) / np.maximum(Sb, 1e-300)).max()))
            row.update({"speedup_vs_exact": round(k1_ref / k1, 2), "envelope_checked_streams": CHECK_STREAMS,
                        "max_err_over_S_vs_exact": worst, "envelope_within_1e-5_S": bool(worst <= 1e-5)})
        rows.append(row)
        print(json.dumps(row), file=sys.stderr, flush=True)
print(json.dumps({"bench": "wideband", "steps": steps, "input": "u8: device-resident submits; cs16: host submits (soapy variant)",
                  "gpu": name, "power_limit_w": float(plimit), "max_sm_clock_mhz": float(maxclk), "rows": rows}))
