"""The streaming front-ends' device submits (acb_submit_real_device, acb_submit_cs16_device, acb_submit_cs16_planar_device).

The rule throughout: a context fed through the device calls gives exactly what an identical context fed the same samples
through the host calls gives.  That is the row count of every submit, the envelope of the last one bit for bit, every
channel's demodulator state, and every message field (text, CRC, err, lvl bits, pos, soh_pos) in the same order.  The
inputs are three streams whose rows sit further apart than the samples they carry, and ragged counts: 1, K-1, K, K+1, a
count that completes no row, and the largest a submit may carry."""
import ctypes as C

import numpy as np
import pytest

from acarsdec_b200 import api, synth

pytestmark = pytest.mark.gpu

FLAG_REAL, FLAG_CS16 = 2, 4
FAST_CHANNELIZER, FAST_FILTER, FAST_FILTER_REAL, FAST_WIDEBAND, FAST_WIDEBAND_REAL = 8, 16, 32, 64, 128
NO_INPUT_STAGING, ERR_ARG = 1, -1
NSTREAMS, NCH, MAXBLK = 3, 4, 2
REAL_FM = (131.400, 131.425, 131.450, 131.500)
CS16_FM = (130.000, 130.025, 130.050, 130.100)
PAD = 37                       # device rows are nsamples + PAD samples apart


def _kind_K(kind):
    return 200 if kind == "real" else 160


def _signal(kind, seed, n):
    """(freqs_hz, fc, input): float32 (S, n) real, int16 (S, n, 2) CS16 (interleaved and planar alike)."""
    K = _kind_K(kind)
    rate = K * 12500
    if kind == "real":
        fd, fc, _ = api.air_plan(rate, REAL_FM)
        fm = REAL_FM
    else:
        fd, _, fc = api.plan(K, CS16_FM)
        fm = CS16_FM
    xs = []
    for s in range(NSTREAMS):
        p = synth.make_plan(K, fm, fc, seconds=n / rate, seed=seed + 7 * s, msgs_per_chan_per_sec=14.0, text_len=(5, 20),
                            amp=(8.0, 14.0))
        if kind == "real":
            xs.append(synth.render_real(synth.StreamPlan(K=K, freqs_hz=tuple(fd), fc_hz=fc, bursts=p.bursts, seed=p.seed), 0, n))
        else:
            xs.append(synth.render_cs16(p, 0, n))
    return fd, fc, np.stack(xs)


def _make(kind, flags, taps, fd, fc):
    K = _kind_K(kind)
    ctx = api.Context(K, NSTREAMS, NCH, MAXBLK, flags=flags | (FLAG_REAL if kind == "real" else FLAG_CS16), taps=taps)
    for s in range(NSTREAMS):
        if taps and taps < K:                          # the planners build K-tap tables only: the first taps of them
            wf = api.build_wf_air(K * 12500, REAL_FM) if kind == "real" else api.build_wf_cs16(1 if kind == "planar" else 0, K, fd, fc)
            ctx.set_wf(s, wf[:, :2 * taps])
        elif kind == "real":
            ctx.set_plan_air_at(s, fd, fc)
        else:
            ctx.set_plan_cs16(s, fd, 1 if kind == "planar" else 0, fc)
    return ctx


def _host_submit(ctx, kind, part):
    if kind == "real":
        return ctx.submit_real(np.ascontiguousarray(part))
    if kind == "cs16":
        return ctx.submit_cs16(np.ascontiguousarray(part))
    return ctx.submit_cs16_planar(np.ascontiguousarray(part[..., 0]), np.ascontiguousarray(part[..., 1]))


def _to_device(kind, part, keep):
    """The part on the GPU in rows PAD samples wider than it (kept alive in `keep`); the tensors submit_tensor takes."""
    import torch
    S, n = part.shape[:2]
    if kind == "planar":
        wide = torch.empty((2, S, n + PAD), dtype=torch.int16, device="cuda")
        wide[0, :, :n] = torch.from_numpy(np.ascontiguousarray(part[..., 0])).cuda()
        wide[1, :, :n] = torch.from_numpy(np.ascontiguousarray(part[..., 1])).cuda()
        keep.append(wide)
        return wide[0, :, :n], wide[1, :, :n]
    shape = (S, n + PAD) + part.shape[2:]
    wide = torch.empty(shape, dtype=torch.float32 if kind == "real" else torch.int16, device="cuda")
    wide[:, :n] = torch.from_numpy(np.ascontiguousarray(part)).cuda()
    keep.append(wide)
    return wide[:, :n], None


def _device_submit(ctx, kind, part, keep):
    x, xq = _to_device(kind, part, keep)
    return ctx.submit_tensor(x, xq)


def _counts(K):
    """Ragged submit lengths: 1, K-1, K, K+1, one that completes no row, the largest allowed, then two more."""
    out, carry = [], 0

    def add(n):
        nonlocal carry
        out.append(n)
        carry = (carry + n) % K
    for n in (1, K - 1, K, K + 1):
        add(n)
    add(K - 1 - carry)                                  # completes no row: the carry is 1 here, K - 1 after
    add(MAXBLK * 1024 * K + K - 1 - carry)              # every row a submit may produce (the carry stays K - 1)
    add(7 * K + 13)
    add(1024 * K + 5)
    return out


def _msgs(ctx):
    return [(m.stream, m.chn, m.len, m.err, bytes(m.txt[:m.len]), bytes(m.crc), int(np.float32(m.lvl).view(np.uint32)),
             int(m.pos), int(m.soh_pos)) for m in ctx.drain()]


def _finish(ctx, last_rows):
    ctx.sync()
    return (_msgs(ctx), ctx.read_dm(last_rows).view(np.uint32),
            [ctx.get_state(s, c).vec() for s in range(NSTREAMS) for c in range(NCH)], ctx.stats().fast_chan_launches)


def _same(a, b):
    assert a[0] == b[0]
    assert np.array_equal(a[1], b[1])
    assert a[2] == b[2]
    assert a[3] == b[3]


# (kind, flags, taps relative to K): each flag at a shape where it applies
FORMS = []
for _kind in ("real", "cs16", "planar"):
    _real = _kind == "real"
    FORMS += [(_kind, 0, "lt"), (_kind, 0, "eq"), (_kind, FAST_CHANNELIZER, "eq"),
              (_kind, FAST_WIDEBAND_REAL if _real else FAST_WIDEBAND, "eq"), (_kind, 0, "gt"),
              (_kind, FAST_FILTER_REAL if _real else FAST_FILTER, "gt"), (_kind, FAST_WIDEBAND_REAL if _real else FAST_WIDEBAND, "gt")]


def _taps(K, rel):
    return {"lt": K // 2 + 3, "eq": 0, "gt": 2 * K + 3}[rel]


@pytest.mark.parametrize("kind,flags,rel", FORMS, ids=[f"{k}-{f}-{r}" for k, f, r in FORMS])
def test_device_submits_equal_host_submits(native, kind, flags, rel):
    K = _kind_K(kind)
    taps = _taps(K, rel)
    counts = _counts(K)
    fd, fc, x = _signal(kind, 11 + flags + len(rel), sum(counts))
    keep = []
    with _make(kind, flags, taps, fd, fc) as host, _make(kind, flags, taps, fd, fc) as dev:
        at = 0
        for i, n in enumerate(counts):
            part = x[:, at:at + n]
            a, b = _host_submit(host, kind, part), _device_submit(dev, kind, part, keep)
            assert a == b, (i, n)
            at += n
            if i % 3 == 2:
                host.collect()
                dev.collect()
        assert 0 in [(sum(counts[:i + 1]) // K) - (sum(counts[:i]) // K) for i in range(len(counts))]
        want, got = _finish(host, a), _finish(dev, b)
    _same(got, want)
    if flags:
        assert want[3] > 0
    if rel != "lt":
        assert want[0]


MIXED = [("real", FAST_WIDEBAND_REAL, "gt"), ("cs16", 0, "eq"), ("planar", FAST_FILTER, "gt"), ("cs16", FAST_WIDEBAND, "eq")]


@pytest.mark.parametrize("kind,flags,rel", MIXED, ids=[f"{k}-{f}-{r}" for k, f, r in MIXED])
def test_mixed_host_and_device_submits(native, kind, flags, rel):
    """Host and device submits alternating in one context: the all-host result, across an acb_reset too."""
    K = _kind_K(kind)
    taps = _taps(K, rel)
    counts = _counts(K)
    fd, fc, x = _signal(kind, 40 + flags, 2 * sum(counts))
    keep = []
    with _make(kind, flags, taps, fd, fc) as host, _make(kind, flags, taps, fd, fc) as mixed:
        res = []
        for ctx, alternate in ((host, False), (mixed, True)):
            out, at = [], 0
            for rnd in range(2):
                for i, n in enumerate(counts):
                    part = x[:, at:at + n]
                    dev = alternate and (i + rnd) % 2 == 1
                    out.append(_device_submit(ctx, kind, part, keep) if dev else _host_submit(ctx, kind, part))
                    at += n
                if rnd == 0:
                    ctx.sync()
                    out.append(_msgs(ctx))
                    ctx.reset()
            res.append((out, _finish(ctx, out[-1])))
    assert res[1][0] == res[0][0]
    _same(res[1][1], res[0][1])


@pytest.mark.parametrize("kind", ["real", "cs16", "planar"])
def test_wait_event_orders_the_device_read(native, kind):
    """The device buffer is filled on a torch side stream behind a long sleep; acb_wait_event on an event recorded there,
    then the device submit, with no host synchronisation in between: the result is the host context's.  The device
    context is created with ACB_FLAG_NO_INPUT_STAGING, which does not concern the streaming kinds."""
    import torch
    K = _kind_K(kind)
    counts = [3 * K + 1, 1024 * K + 7, K // 2, 2 * 1024 * K - 5]
    fd, fc, x = _signal(kind, 77, sum(counts))
    side = torch.cuda.Stream()
    bufs = []
    at = 0
    for n in counts:                                  # the device buffers start out as noise, the samples are in pinned memory
        part = np.ascontiguousarray(x[:, at:at + n])
        if kind == "planar":                          # (2, S, n): the I plane, then the Q plane
            part = np.ascontiguousarray(np.moveaxis(part, 2, 0))
        at += n
        src = torch.from_numpy(part).pin_memory()
        dst = torch.randint(-30000, 30000, src.shape, dtype=torch.int16, device="cuda") if src.dtype == torch.int16 \
            else torch.randn(src.shape, device="cuda") * 1e4
        bufs.append((src, dst))
    torch.cuda.synchronize()
    with _make(kind, 0, 0, fd, fc) as host, _make(kind, NO_INPUT_STAGING, 0, fd, fc) as dev:
        want, got = [], []
        at = 0
        for n, (src, dst) in zip(counts, bufs):
            want.append(_host_submit(host, kind, x[:, at:at + n]))
            at += n
            ev = torch.cuda.Event()
            with torch.cuda.stream(side):
                torch.cuda._sleep(100_000_000)            # ~50 ms of GPU time before the samples land
                dst.copy_(src, non_blocking=True)
                ev.record(side)
            dev.wait_event(ev.cuda_event)
            got.append(dev.submit_tensor(dst[0], dst[1]) if kind == "planar" else dev.submit_tensor(dst))
        assert got == want
        _same(_finish(dev, got[-1]), _finish(host, want[-1]))


@pytest.mark.parametrize("kind", ["real", "cs16", "planar"])
def test_device_input_may_be_overwritten_once_covered(native, kind):
    """Each device buffer is overwritten with noise on a torch stream as soon as the lifetime rule frees it: by the
    acb_collect that covers its submit, or, for a submit that produced no row, by the next acb_sync."""
    import torch
    K = _kind_K(kind)
    counts = [5 * K + 3, 1024 * K + 1, K // 3, 3 * K, 2 * 1024 * K - K, 17]
    fd, fc, x = _signal(kind, 91, sum(counts))
    side = torch.cuda.Stream()
    keep, live = [], []

    def scribble(t):
        with torch.cuda.stream(side):
            t.copy_(torch.randint(-20000, 20000, t.shape, device="cuda").to(t.dtype))
    with _make(kind, 0, 0, fd, fc) as host, _make(kind, 0, 0, fd, fc) as dev:
        want, got, at = [], [], 0
        for n in counts:
            part = x[:, at:at + n]
            at += n
            want.append(_host_submit(host, kind, part))
            got.append(_device_submit(dev, kind, part, keep))
            live.append((keep[-1], got[-1]))
            if len(live) == 2:
                # the older one: produced rows -> covered by this collect; produced none -> only by the sync
                if live[0][1] > 0:
                    host.collect()
                    dev.collect()
                else:
                    host.sync()
                    dev.sync()
                scribble(live[0][0])
                live.pop(0)
        assert 0 in got and got == want
        _same(_finish(dev, got[-1]), _finish(host, want[-1]))


def _raw_submit(lib, ctx, kind, p, q, stride, n):
    if kind == "real":
        return lib.acb_submit_real_device(ctx.h, p, stride, n)
    if kind == "cs16":
        return lib.acb_submit_cs16_device(ctx.h, p, stride, n)
    return lib.acb_submit_cs16_planar_device(ctx.h, p, q, stride, n)


@pytest.mark.parametrize("kind", ["real", "cs16", "planar"])
def test_device_submit_refusals_leave_the_carry(native, kind):
    """Host memory (pageable and pinned), misaligned pointers, the wrong context kind, nsamples 0 or too large and a
    stride below nsamples are refused with ACB_ERR_ARG; the next valid submit then gives exactly the host result."""
    import torch
    lib = api.load()
    K = _kind_K(kind)
    counts = [K + 5, 1024 * K + 9, 3 * K]
    fd, fc, x = _signal(kind, 5, sum(counts))
    keep = []
    el = 2 if kind == "planar" else 4
    with _make(kind, 0, 0, fd, fc) as host, _make(kind, 0, 0, fd, fc) as dev:
        want, got, at = [], [], 0
        for j, n in enumerate(counts):
            part = x[:, at:at + n]
            at += n
            want.append(_host_submit(host, kind, part))
            d, dq = _to_device(kind, part, keep)
            p, q = d.data_ptr(), (dq.data_ptr() if dq is not None else None)
            stride = n + PAD
            if j == 1:
                pageable = np.zeros(NSTREAMS * stride * 2, dtype=np.float32)
                pinned = api.PinnedBuffer(NSTREAMS * stride * 8)
                for hp in (pageable.ctypes.data, pinned.ptr):
                    assert _raw_submit(lib, dev, kind, hp, hp, stride, n) == ERR_ARG
                    if kind == "planar":                # either plane on the host is refused
                        assert _raw_submit(lib, dev, kind, p, hp, stride, n) == ERR_ARG
                assert _raw_submit(lib, dev, kind, p + el // 2 if el == 4 else p + 1, q, stride, n) == ERR_ARG
                if kind == "planar":
                    assert _raw_submit(lib, dev, kind, p, q + 1, stride, n) == ERR_ARG
                assert _raw_submit(lib, dev, kind, p, q, stride, 0) == ERR_ARG
                assert _raw_submit(lib, dev, kind, p, q, stride + 10 ** 7, MAXBLK * 1024 * K + K) == ERR_ARG
                assert _raw_submit(lib, dev, kind, p, q, n - 1, n) == ERR_ARG
                # the wrong kind: a real call on a CS16 context and the CS16 calls on a real one
                if kind == "real":
                    assert lib.acb_submit_cs16_device(dev.h, p, stride, n) == ERR_ARG
                    assert lib.acb_submit_cs16_planar_device(dev.h, p, p, stride, n) == ERR_ARG
                else:
                    assert lib.acb_submit_real_device(dev.h, p, stride, n) == ERR_ARG
                with api.Context(K, NSTREAMS, NCH, 1) as u8:
                    assert _raw_submit(lib, u8, kind, p, q if q else p, stride, n) == ERR_ARG
                if torch.cuda.device_count() > 1:       # another device's memory
                    other = torch.zeros(NSTREAMS * stride * 2, dtype=torch.float32, device="cuda:1")
                    assert _raw_submit(lib, dev, kind, other.data_ptr(), other.data_ptr(), stride, n) == ERR_ARG
                with pytest.raises(TypeError):
                    dev.submit_tensor(torch.from_numpy(np.ascontiguousarray(part if kind != "planar" else part[..., 0])))
                pinned.close()
            got.append(dev.submit_tensor(d, dq))
        assert got == want
        _same(_finish(dev, got[-1]), _finish(host, want[-1]))


def test_managed_memory_is_accepted(native):
    """Managed memory (cudaMallocManaged) is device-accessible input: the same result as the host call."""
    cudart = None
    for name in ("libcudart.so", "libcudart.so.12"):
        try:
            cudart = C.CDLL(name)
            break
        except OSError:
            continue
    if cudart is None:
        pytest.skip("libcudart not loadable by name")
    K = _kind_K("cs16")
    n = 1024 * K + 77
    fd, fc, x = _signal("cs16", 3, n)
    p = C.c_void_p()
    assert cudart.cudaMallocManaged(C.byref(p), C.c_size_t(x.nbytes), 1) == 0
    try:
        C.memmove(p.value, np.ascontiguousarray(x).ctypes.data, x.nbytes)
        with _make("cs16", 0, 0, fd, fc) as host, _make("cs16", 0, 0, fd, fc) as dev:
            a = _host_submit(host, "cs16", x)
            b = dev.submit_cs16_device(p.value, n, n)
            assert a == b
            _same(_finish(dev, b), _finish(host, a))
    finally:
        cudart.cudaDeviceSynchronize()
        cudart.cudaFree(p)


def test_wide_stream_of_every_streaming_kind(native):
    """WideStream(kind="cs16" / "real"): one stream, channels split over the visible GPUs (two at most; world size 1 when
    only one is visible), one broadcast per submit, device submits on every rank; the merged messages equal one
    context's in order, and at taps = K without fast flags the CPU oracle's."""
    import json
    import subprocess
    import sys
    from pathlib import Path
    import torch
    n = min(torch.cuda.device_count(), 2)
    worker = str(Path(__file__).resolve().parent / "wide_stream_kinds_worker.py")
    if n >= 2:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
               "--master-addr", "127.0.0.1", "--master-port", "29547", worker]
    else:
        cmd = [sys.executable, worker]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads([line for line in r.stdout.splitlines() if line.startswith("{")][-1])
    assert res["match"] and res["world"] == max(n, 1) and len(res["cases"]) == 6
