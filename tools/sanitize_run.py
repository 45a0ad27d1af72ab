"""Small end-to-end run for compute-sanitizer (memcheck / racecheck): u8 path with 11 channels
(two groups), real-input path with an awkward length, envelope path; checks frames against the oracle."""
import sys
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import numpy as np
from acarsdec_b200 import api, synth
import refs
from common import msg_tuple, load_testwav

orc = refs.OracleLib()
K, fm, nblk = 160, synth.DEFAULT_FREQS_MHZ, 3
fd, _, fc = api.plan(K, fm)
plan = synth.make_plan(K, fm, fc, seconds=0.24, seed=5, text_len=(5, 20))
iq = synth.render_blocks(plan, 0, nblk).reshape(1, -1)
with api.Context(K, 2, 8, nblk) as ctx:
    for s in range(2): ctx.set_plan(s, fd)
    ctx.submit_host(np.concatenate([iq, iq]), nblk); ctx.submit_host(np.concatenate([iq, iq]), nblk); ctx.sync()
    n1 = len(ctx.drain())
rate, fma = 2500000, (131.525, 131.725, 131.825)
fda, fca, Ka = api.air_plan(rate, fma)
x = (np.random.default_rng(1).standard_normal((1, 1024 * Ka + 777)) * 0.01).astype(np.float32)
with api.Context(Ka, 1, 3, 3, flags=2) as ctx:
    ctx.set_plan_air(0, fda); ctx.submit_real(x); ctx.submit_real(x[:, :5000]); ctx.sync()
xw, exp = load_testwav()
with api.Context(160, 1, 4, 4, flags=1) as ctx:
    ctx.submit_dm(xw[None, :4096]); ctx.submit_dm(xw[None, 4096:8000]); ctx.sync()
    n3 = len(ctx.drain())
# fast channelizer (bulk copies + mbarrier), K=160 and K=192, partial channel group
for Kf, fmf in ((160, fm), (192, (131.525, 131.725, 131.825))):
    fdf, _, fcf = api.plan(Kf, fmf)
    pf = synth.make_plan(Kf, fmf, fcf, seconds=0.24, seed=6, text_len=(5, 20))
    iqf = synth.render_blocks(pf, 0, 2).reshape(1, -1)
    with api.Context(Kf, 2, len(fmf), 2, flags=8) as ctx:
        for s in range(2): ctx.set_plan(s, fdf)
        ctx.submit_host(np.concatenate([iqf, iqf]), 2); ctx.submit_host(np.concatenate([iqf, iqf]), 2); ctx.sync()
        assert ctx.stats().fast_chan_launches == 2
        n4 = len(ctx.drain())
# CS16 front-end with a ragged length, and the batched device FEC
iqc = synth.render_cs16(plan, 0, 1024 * K + 333)[None]
with api.Context(K, 1, 8, 2, flags=4) as ctx:
    ctx.set_plan_cs16(0, fd, 0); ctx.submit_cs16(iqc); ctx.submit_cs16(iqc[:, :4000]); ctx.sync()
    m = api.Msg(); fr = synth.frame_bytes(b"SANITIZER", prekey=0)[5:-1]
    m.len = len(fr) - 2; m.txt[:m.len] = fr[:-2]; m.crc[:] = fr[-2:]
    m.txt[3] ^= 0x04
    out = ctx.block_fec_batch([m] * 70)
    assert all(o is not None and o.err == 1 for o in out)
# the fast forms of the streaming front-ends (partial blocks, tiles past the end, the 32 rows of slack), four submits so that
# every one of the three pipeline slots is reused
with api.Context(K, 1, 8, 2, flags=4 | 8) as ctx:
    ctx.set_plan_cs16(0, fd, 1)
    for part in (iqc, iqc[:, :4000], iqc[:, :33 * K + 5], iqc):
        ctx.submit_cs16(part)
    ctx.sync()
    assert ctx.stats().fast_chan_launches >= 3
    n5 = len(ctx.drain())
xr = synth.render_real(synth.StreamPlan(K=Ka, freqs_hz=tuple(fda), fc_hz=fca, seed=2, noise_sigma=1.0), 0, 1024 * Ka + 777)[None]
with api.Context(Ka, 1, 3, 3, flags=2 | 8) as ctx:
    ctx.set_plan_air(0, fda)
    for part in (xr, xr[:, :5000], xr[:, :17 * Ka + 3], xr):
        ctx.submit_real(part)
    ctx.sync()
    assert ctx.stats().fast_chan_launches >= 3
# the wideband fast form at its largest shared-memory configuration (K = 1808: 12-row tiles, 115704 bytes per CTA),
# taps > K, ragged CS16 submits
Kw = 1808
fw = [120_000_000 + 25_000 * (i // 2 + 1) * (1 if i % 2 == 0 else -1) for i in range(13)]
xw = np.random.default_rng(1).integers(-32768, 32768, size=(1, 40 * Kw + 77, 2), dtype=np.int16)
with api.Context(Kw, 1, 13, 1, flags=4 | api.FLAG_FAST_WIDEBAND, taps=2 * Kw + 3) as ctx:
    ctx.set_plan_cs16(0, fw, 0, 120_000_000)
    for part in (xw, xw[:, :1000], xw[:, :17 * Kw + 3]):
        ctx.submit_cs16(part)
    ctx.sync()
    assert ctx.stats().fast_chan_launches == 2          # the 1000-sample submit completes no row
# the real-input wideband fast form at its largest shared-memory configuration (K = 1112: 24-row tiles, 115648 bytes per
# CTA), taps > K (the history in front of the rows), ragged real submits, every residue k mod 4
Kr = 1112
fr = [131_500_000 + 12_500 * d for d in (-200, -151, -150, -149, -100, -3, -2, -1, 0, 1, 50, 101, 150)]
xr = (np.random.default_rng(2).standard_normal((1, 40 * Kr + 77)) * 100).astype(np.float32)
with api.Context(Kr, 1, 13, 1, flags=2 | api.FLAG_FAST_WIDEBAND_REAL, taps=2 * Kr + 3) as ctx:
    ctx.set_plan_air(0, fr)
    for part in (xr, xr[:, :1000], xr[:, :17 * Kr + 3]):
        ctx.submit_real(part)
    ctx.sync()
    assert ctx.stats().fast_chan_launches == 2          # the 1000-sample submit completes no row
# the streaming kinds' device submits: one of each kind behind a carry of 77 samples (a destination offset that is not on
# 16 bytes), the source rows 5 samples wider than the input, taps > K (the history in front of the rows)
import torch  # noqa: E402
for kind, Kd, fl in (("real", Ka, 2), ("cs16", K, 4), ("planar", K, 4)):
    with api.Context(Kd, 2, 3, 1, flags=fl, taps=2 * Kd + 3) as ctx:
        for s in range(2):
            ctx.set_plan_air(s, fda) if kind == "real" else ctx.set_plan_cs16(s, fd[:3], 0)
        n = 3 * Kd + 7
        if kind == "real":
            dev = torch.randn((2, n + 5), device="cuda") * 100
            assert ctx.submit_real((dev[:, :77].cpu().numpy()).copy()) == 0
            assert ctx.submit_tensor(dev[:, :n]) == 3
        else:
            dev = torch.randint(-3000, 3000, (2, n + 5, 2), dtype=torch.int16, device="cuda")
            assert ctx.submit_cs16(dev[:, :77].cpu().numpy().copy()) == 0
            if kind == "cs16":
                assert ctx.submit_tensor(dev[:, :n]) == 3
            else:
                planes = dev.permute(2, 0, 1).contiguous()
                assert ctx.submit_tensor(planes[0, :, :n], planes[1, :, :n]) == 3
        ctx.sync()
# ragged submits: u8 device input with unequal nblk (the channelizer reads every stream, the last included, for the
# largest nblk: the buffer ends there) and the taps > K history gather; the streaming kinds' ragged device submits
# (k_append4_ragged behind unequal carries, k_move_tail), a stream at count 0 among them
with api.Context(K, 3, 3, 2, flags=1, taps=2 * K + 3) as ctx:
    for s in range(3):
        ctx.set_plan(s, fd[:3])
    bb = 1024 * K * 2
    dev = torch.randint(0, 256, (3, 2 * bb), dtype=torch.uint8, device="cuda")
    for counts in ([2, 0, 1], [1, 2, 0], [0, 1, 2]):
        ctx.submit_device(dev.data_ptr(), 0, 2 * bb, counts=counts)
    ctx.sync()
for kind, Kd, fl in (("real", Ka, 2), ("cs16", K, 4), ("planar", K, 4)):
    with api.Context(Kd, 3, 3, 1, flags=fl, taps=2 * Kd + 3) as ctx:
        for s in range(3):
            ctx.set_plan_air(s, fda) if kind == "real" else ctx.set_plan_cs16(s, fd[:3], 0)
        n = 3 * Kd + 7
        dev = (torch.randn((3, n), device="cuda") * 100 if kind == "real"
               else torch.randint(-3000, 3000, (3, n, 2), dtype=torch.int16, device="cuda"))
        for counts in ([77, 0, n], [n, 5, 0], [0, n, Kd + 1]):
            if kind == "planar":
                planes = dev.permute(2, 0, 1).contiguous()
                ctx.submit_tensor(planes[0], planes[1], counts=counts)
            else:
                ctx.submit_tensor(dev, counts=counts)
        ctx.sync()
# ACB_FLAG_LEVEL_STATS: k_level_in on each input kind (a ragged u8 device submit, a CS16 length that is no whole number
# of 16-byte loads), k_level_dm on the channelizer's envelope and on envelope input
with api.Context(K, 3, 3, 2, flags=1 | api.FLAG_LEVEL_STATS, taps=2 * K + 3) as ctx:
    for s in range(3):
        ctx.set_plan(s, fd[:3])
    bb = 1024 * K * 2
    dev = torch.randint(0, 256, (3, 2 * bb), dtype=torch.uint8, device="cuda")
    ctx.submit_device(dev.data_ptr(), 0, 2 * bb, counts=[2, 0, 1])
    ctx.submit_dm(np.ones((3, 1500, 3), np.float32))
    ctx.sync()
    ctx.level_stats()
# K = 161 and 162: stream 0's 3 rows and stream 2's 1 row are 3 * K * 4 and K * 4 bytes, which end 12 and 4 bytes (K = 161)
# or 8 bytes (K = 162) past a 16-byte load, so k_level_in's scalar tail reads them
for kind, Kd, fl in (("real", 162, 2), ("cs16", 161, 4), ("planar", 162, 4)):
    with api.Context(Kd, 3, 3, 1, flags=fl | api.FLAG_LEVEL_STATS) as ctx:
        for s in range(3):
            ctx.set_plan_air(s, fda) if kind == "real" else ctx.set_plan_cs16(s, fd[:3], 0)
        n = 3 * Kd + 7
        assert {3 * Kd * 4 % 16, Kd * 4 % 16} & {4, 8, 12}
        dev = (torch.randn((3, n), device="cuda") * 0.5 if kind == "real"
               else torch.randint(-32768, 32767, (3, n, 2), dtype=torch.int16, device="cuda"))
        if kind == "planar":
            planes = dev.permute(2, 0, 1).contiguous()
            ctx.submit_tensor(planes[0], planes[1], counts=[n, 5, Kd + 1])
        else:
            ctx.submit_tensor(dev, counts=[n, 5, Kd + 1])
        ctx.sync()
        ctx.level_stats()
# moving streams: k_stream_pack / k_stream_unpack over every region kind (chain states, the u8 history, the streaming
# carry, exact tables, the fast plans' 4-byte-strided metadata, the open level windows), two streams to two other slots
for kind, Kd, fl, tp in (("u8", K, 1 | 16 | api.FLAG_LEVEL_STATS, 2 * K + 3), ("cs16", K, 4 | 64, 0), ("real", Ka, 2 | 8, 0)):
    with api.Context(Kd, 3, 3, 1, flags=fl, taps=tp) as a, api.Context(Kd, 4, 3, 1, flags=fl, taps=tp) as b:
        for ctx in (a, b):
            for s in range(ctx.nstreams):
                (ctx.set_plan(s, fd[:3]) if kind == "u8" else ctx.set_plan_air(s, fda) if kind == "real"
                 else ctx.set_plan_cs16(s, fd[:3], 0))
        if kind == "u8":
            dev = torch.randint(0, 256, (3, 1024 * Kd * 2), dtype=torch.uint8, device="cuda")
            a.submit_device(dev.data_ptr(), 1, dev.stride(0))
        else:
            n = 3 * Kd + 7
            dev = torch.randn((3, n), device="cuda") if kind == "real" else torch.randint(-3000, 3000, (3, n, 2), dtype=torch.int16, device="cuda")
            a.submit_tensor(dev)
        b.load_streams([3, 0], a.save_streams([2, 0]))
        b.sync()
print("sanitize run ok", n1, n3, n4, n5)
