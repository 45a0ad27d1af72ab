"""What the streaming kinds' device submits save: per submit, the host submit's H2D copy (acb_submit_real_host /
acb_submit_cs16_host from pinned memory) against the device submit's append kernel (acb_submit_real_device /
acb_submit_cs16_device / acb_submit_cs16_planar_device from device memory), and the channelizer (K1) of both paths.

Shapes: CS16 K = 1600 x 256 channels at taps K and 4K and real input K = 800 x 200 channels, with the wideband fast forms
(ACB_FLAG_FAST_WIDEBAND / _REAL), and one narrow shape each (CS16 K = 160, real K = 200, 8 channels).  The copy and append
times are the kernels' and copies' device durations from torch.profiler (CUDA activities) over the timed submits, in a
run of their own; K1 is the library's CUDA-event time of the channelizer (acb_stats_t.chan_ms / chan_launches) in a run
without the profiler.  Beside the append kernel, a cudaMemcpy2DAsync device-to-device copy of the same rows to the same
unaligned destination offset is timed with CUDA events, for the interleaved forms.  The card's name, power limit and SM
clock are read in the same run with read-only queries.  Prints one JSON line.
  python tools/bench_stream_device.py [steps]"""
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

from acarsdec_b200 import api

args = [a for a in sys.argv[1:] if not a.startswith("--")]
steps = int(args[0]) if args else 10
FLAG_REAL, FLAG_CS16 = 2, 4
FC = 130_000_000
# (kind, K, channels, taps multiple, streams, rows per submit, flags)
SHAPES = [("cs16", 1600, 256, 1, 4, 4096, api.FLAG_FAST_WIDEBAND), ("cs16", 1600, 256, 4, 4, 4096, api.FLAG_FAST_WIDEBAND),
          ("planar", 1600, 256, 1, 4, 4096, api.FLAG_FAST_WIDEBAND),
          ("real", 800, 200, 1, 8, 4096, api.FLAG_FAST_WIDEBAND_REAL),
          ("cs16", 160, 8, 1, 64, 2048, 0), ("real", 200, 8, 1, 64, 2048, 0)]


def smi(fields):
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout
    return [v.strip() for v in out.strip().splitlines()[0].split(",")]


def freqs(kind, K, nch):
    if kind == "real":                   # on the raster across the real band (tools/bench_wideband_air.py: air_freqs)
        D = K // 4 - 1
        d = np.rint(np.linspace(-D, D - 1, nch)).astype(np.int64)
        return [int(131_500_000 + 12_500 * v) for v in d]
    return [FC + 25_000 * (i - nch // 2 + (i >= nch // 2)) for i in range(nch)]     # the fast plans leave out Fc itself


def make(kind, K, nch, taps, S, nrows, flags):
    ctx = api.Context(K, S, nch, -(-nrows // 1024) + 1, flags=flags | (FLAG_REAL if kind == "real" else FLAG_CS16), taps=taps)
    f = freqs(kind, K, nch)
    for s in range(S):
        ctx.set_plan_air(s, f) if kind == "real" else ctx.set_plan_cs16(s, f, 0, FC)
    return ctx


def cudart():
    for name in ("libcudart.so.12", "libcudart.so"):
        try:
            return C.CDLL(name)
        except OSError:
            continue
    return None


def memcpy2d_ms(rt, S, n, reps=20):
    """cudaMemcpy2DAsync of S rows of n 4-byte samples to a destination 13 samples into rows of n + 77: ms per copy"""
    if rt is None:
        return None
    src = torch.empty((S, n), dtype=torch.float32, device="cuda")
    dst = torch.empty((S, n + 77), dtype=torch.float32, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = (C.c_void_p(dst.data_ptr() + 13 * 4), C.c_size_t((n + 77) * 4), C.c_void_p(src.data_ptr()), C.c_size_t(n * 4),
            C.c_size_t(n * 4), C.c_size_t(S), C.c_int(3), st)
    assert rt.cudaMemcpy2DAsync(*args) == 0
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        rt.cudaMemcpy2DAsync(*args)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def device_ms(prof, match):
    """mean device duration (ms) and count of the profiled kernels / copies whose name matches"""
    ts = [e.time_range.elapsed_us() for e in prof.events() if e.device_type.name == "CUDA" and match(e.name)]
    return (float(np.mean(ts)) / 1e3, len(ts)) if ts else (None, 0)


name, plimit, maxclk = smi("name,power.limit,clocks.max.sm")
rt = cudart()
rows = []
mon = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0", "-lms", "200"],
                       stdout=subprocess.PIPE, text=True)
for kind, K, nch, mult, S, nrows, flags in SHAPES:
    taps = mult * K
    n = nrows * K
    rng = np.random.default_rng(K + taps)
    if kind == "real":
        host = torch.from_numpy((rng.standard_normal((S, n)) * 100).astype(np.float32)).pin_memory()
    else:
        host = torch.from_numpy(rng.integers(-2000, 2000, size=(S, n, 2), dtype=np.int16)).pin_memory()
    dev_in = host.cuda()
    res = {"kind": kind, "K": K, "channels": nch, "taps": taps, "streams": S, "rows_per_submit": nrows,
           "bytes_per_submit": host.numel() * host.element_size(), "flags": flags}
    for path in ("host", "device"):
        ctx = make(kind, K, nch, taps if mult > 1 else 0, S, nrows, flags)
        if path == "host":
            hn = host.numpy()
            if kind == "planar":
                hi, hq = (host[..., i].contiguous().pin_memory().numpy() for i in (0, 1))
                step = lambda: ctx.submit_cs16_planar(hi, hq)
            else:
                step = (lambda: ctx.submit_real(hn)) if kind == "real" else (lambda: ctx.submit_cs16(hn))
        else:
            if kind == "planar":
                di, dq = dev_in[..., 0].contiguous(), dev_in[..., 1].contiguous()
                step = lambda: ctx.submit_tensor(di, dq)
            else:
                step = lambda: ctx.submit_tensor(dev_in)
        torch.cuda.synchronize()
        for _ in range(2):
            step()
            ctx.sync()
        ctx.drain_records()
        ctx.stats(reset=True)
        for _ in range(steps):
            step()
            ctx.sync()
        st = ctx.stats()
        res[f"k1_ms_{path}"] = round(st.chan_ms / st.chan_launches, 4)
        res[f"fast_chan_launches_{path}"] = int(st.fast_chan_launches)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                step()
                ctx.sync()
        if path == "host":
            ms, cnt = device_ms(prof, lambda s: "HtoD" in s)
            res["h2d_ms_per_submit"] = round(ms * cnt / 3, 4) if ms else None
            if kind == "planar":
                ms2, _ = device_ms(prof, lambda s: "interleave" in s)
                res["host_interleave_ms_per_submit"] = round(ms2, 4) if ms2 else None
        else:
            ms, cnt = device_ms(prof, lambda s: "append4" in s)
            res["append_ms_per_submit"] = round(ms * cnt / 3, 4) if ms else None
            res["append_gbytes_per_s"] = round(2 * res["bytes_per_submit"] / (ms * cnt / 3) / 1e6, 1) if ms else None
        ctx.drain_records()
        ctx.close()
    if flags:
        assert res["fast_chan_launches_host"] > 0 and res["fast_chan_launches_device"] == res["fast_chan_launches_host"]
    if kind != "planar":
        m2 = memcpy2d_ms(rt, S, n)
        res["memcpy2d_d2d_ms_same_rows"] = round(m2, 4) if m2 is not None else None
    rows.append(res)
    del host, dev_in
    torch.cuda.empty_cache()

mon.terminate()
clk_out, _ = mon.communicate()
clks = [float(v) for v in clk_out.split() if v.strip().replace(".", "", 1).isdigit()]
print(json.dumps({"bench": "stream_device", "steps": steps, "gpu": name,
                  "input": "host path: pinned host memory (acb_submit_real_host / acb_submit_cs16_host / acb_submit_cs16_planar_host); "
                           "device path: device-resident tensors (acb_submit_*_device); one stream of submits each, sync per submit", "power_limit_w": float(plimit),
                  "max_sm_clock_mhz": float(maxclk), "sm_clock_mhz_median": float(np.median(clks)) if clks else None,
                  "rows": rows}))
