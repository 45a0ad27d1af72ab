"""Which channelizer (K1) kernels one submit launches, for every form a context can take: the fast forms each input kind
has, what selects one over another when several flags apply, the exact block kernel and the generic kernel, and the
launches that go with them (the generic kernel for the rows after the last whole block, the recompute of a u8 context's
leading rows at taps > K).  A stream planned with acb_set_wf has no raster structure, so a fast context with one runs the
exact form.  The launch counters alone cannot say which fast kernel ran: the kernels' names come from torch.profiler."""
import collections
import re

import numpy as np
import pytest

from acarsdec_b200 import api

pytestmark = pytest.mark.gpu

FLAG_REAL, FLAG_CS16 = 2, 4
FAST, FILTER, FILTER_REAL, WB, WB_REAL = 8, 16, 32, 64, 128
KIND_FLAG = {"u8": 0, "cs16": FLAG_CS16, "real": FLAG_REAL}
FREQS_MHZ = (131.450, 131.525, 131.550, 131.725)    # 25 kHz apart: on the fast forms' raster around every planner's Fc
S, MAXBLK = 2, 2
K1_NAME = re.compile(r"\b(k_channelize\w*)\s*[<(]")

DFT1, DFT, RDFT = "k_channelize_dft1", "k_channelize_dft", "k_channelize_rdft"
OVL_FAST, OVL_RDFT = "k_channelize_ovl_fast", "k_channelize_ovl_rdft"
WBK, WBK_REAL = "k_channelize_wb", "k_channelize_wb_real"
IQ4, REAL4, REAL2 = "k_channelize_iq4", "k_channelize_real4", "k_channelize"
GEN, GEN_OVL = "k_channelize_generic", "k_channelize_generic_ovl"

# (id, kind, K, taps, flags, rows of the profiled submit, K1 kernels it launches, fast form?, options)
# options: "unplanned" = stream 1 takes acb_set_wf tables; "second" = one submit before the profiled one; "env" = switches
CASES = [
    # u8 IQ
    ("u8-dft", "u8", 160, 0, FAST, 1024, {DFT1: 1}, True, {}),
    ("u8-dft-fold4", "u8", 192, 0, FAST, 1024, {DFT: 1}, True, {"env": {"ACB_FAST_FOLD8": "0"}}),
    ("u8-dft-before-wb", "u8", 160, 0, FAST | WB, 1024, {DFT1: 1}, True, {}),
    ("u8-ovl-fast", "u8", 160, 2 * 160, FILTER, 1024, {OVL_FAST: 1}, True, {}),
    ("u8-ovl-fast-before-wb", "u8", 192, 2 * 192 + 3, FILTER | WB, 1024, {OVL_FAST: 1}, True, {}),
    ("u8-wb", "u8", 96, 0, WB, 1024, {WBK: 1}, True, {}),
    ("u8-wb-ovl", "u8", 96, 200, WB, 1024, {WBK: 1}, True, {}),
    ("u8-wb-not-below-K", "u8", 96, 90, WB, 1024, {IQ4: 1}, False, {"unplanned": "all"}),
    ("u8-fast-K-unsupported", "u8", 96, 0, FAST, 1024, {IQ4: 1}, False, {}),
    ("u8-fast-taps-over-K", "u8", 160, 2 * 160, FAST, 1024, {IQ4: 1, GEN_OVL: 1}, False, {}),
    ("u8-generic", "u8", 100, 0, 0, 1024, {GEN: 1}, False, {}),
    ("u8-generic-ovl", "u8", 100, 250, 0, 1024, {GEN_OVL: 1}, False, {}),
    ("u8-generic-flags", "u8", 100, 0, FAST | WB, 1024, {GEN: 1}, False, {}),
    ("u8-exact", "u8", 160, 0, 0, 2048, {IQ4: 1}, False, {}),
    ("u8-exact-ovl-first", "u8", 160, 2 * 160, 0, 1024, {IQ4: 1, GEN_OVL: 1}, False, {}),
    ("u8-exact-ovl-second", "u8", 160, 2 * 160, 0, 1024, {IQ4: 1}, False, {"second": True}),
    ("u8-dft-unplanned", "u8", 160, 0, FAST, 1024, {IQ4: 1}, False, {"unplanned": "one"}),
    ("u8-ovl-fast-unplanned", "u8", 160, 2 * 160, FILTER, 1024, {IQ4: 1, GEN_OVL: 1}, False, {"unplanned": "one"}),
    ("u8-wb-ovl-unplanned", "u8", 96, 200, WB, 1024, {IQ4: 1, GEN_OVL: 1}, False, {"unplanned": "one"}),
    # CS16 IQ: every fast form takes partial blocks
    ("cs16-dft", "cs16", 160, 0, FAST, 1500, {DFT1: 1}, True, {}),
    ("cs16-ovl-fast", "cs16", 160, 2 * 160, FILTER, 1500, {OVL_FAST: 1}, True, {}),
    ("cs16-wb", "cs16", 96, 0, WB, 1500, {WBK: 1}, True, {}),
    ("cs16-wb-ovl", "cs16", 96, 3 * 96, WB, 1500, {WBK: 1}, True, {}),
    ("cs16-generic", "cs16", 90, 0, 0, 1500, {GEN: 1}, False, {}),
    ("cs16-exact", "cs16", 160, 0, 0, 1024, {IQ4: 1}, False, {}),
    ("cs16-exact-tail", "cs16", 160, 0, 0, 1500, {IQ4: 1, GEN: 1}, False, {}),
    ("cs16-exact-ovl-tail", "cs16", 160, 2 * 160, 0, 1500, {IQ4: 1, GEN_OVL: 1}, False, {}),
    ("cs16-exact-short", "cs16", 160, 0, 0, 500, {GEN: 1}, False, {}),
    ("cs16-dft-unplanned", "cs16", 160, 0, FAST, 1500, {IQ4: 1, GEN: 1}, False, {"unplanned": "one"}),
    # real input
    ("real-rdft", "real", 200, 0, FAST, 1500, {RDFT: 1}, True, {}),
    ("real-rdft-before-wb", "real", 200, 0, FAST | WB_REAL, 1500, {RDFT: 1}, True, {}),
    ("real-ovl-rdft", "real", 200, 2 * 200, FILTER_REAL, 1500, {OVL_RDFT: 1}, True, {}),
    ("real-u8-filter-flag", "real", 200, 2 * 200, FILTER, 1500, {REAL4: 1, GEN_OVL: 1}, False, {}),
    ("real-wb", "real", 200, 0, WB_REAL, 1500, {WBK_REAL: 1}, True, {}),
    ("real-wb-ovl", "real", 200, 2 * 200, WB_REAL, 1500, {WBK_REAL: 1}, True, {}),
    ("real-u8-wb-flag", "real", 200, 0, WB, 1500, {REAL4: 1, GEN: 1}, False, {}),
    ("real-generic", "real", 202, 0, 0, 1500, {GEN: 1}, False, {}),
    ("real-exact", "real", 200, 0, 0, 1024, {REAL4: 1}, False, {}),
    ("real-exact-rows2", "real", 200, 0, 0, 1024, {REAL2: 1}, False, {"env": {"ACB_REAL_ROWS": "2"}}),
    ("real-exact-tail", "real", 200, 0, 0, 1500, {REAL4: 1, GEN: 1}, False, {}),
    ("real-exact-short", "real", 200, 0, 0, 500, {GEN: 1}, False, {}),
    ("real-wb-unplanned", "real", 200, 0, WB_REAL, 1500, {REAL4: 1, GEN: 1}, False, {"unplanned": "one"}),
]


def _context(kind, K, taps, flags, unplanned):
    ctx = api.Context(K, S, len(FREQS_MHZ), MAXBLK, flags=flags | KIND_FLAG[kind], taps=taps)
    T = taps or K
    tables = (np.random.default_rng(K + T).standard_normal((len(FREQS_MHZ), 2 * T)) / T).astype(np.float32)
    for s in range(S):
        if unplanned == "all" or (unplanned == "one" and s == 1):
            ctx.set_wf(s, tables)
        elif kind == "u8":
            ctx.set_plan(s, api.plan(K, FREQS_MHZ)[0])
        elif kind == "cs16":
            ctx.set_plan_cs16(s, api.plan(K, FREQS_MHZ)[0], 0)
        else:
            ctx.set_plan_air(s, api.air_plan(K * 12500, FREQS_MHZ)[0])
    return ctx


def _submit(ctx, kind, K, rows, rng):
    if kind == "u8":
        ctx.submit_host(rng.integers(0, 256, size=(S, rows * 2 * K), dtype=np.uint8), rows // 1024)
    elif kind == "cs16":
        assert ctx.submit_cs16(rng.integers(-2000, 2000, size=(S, rows * K, 2), dtype=np.int16)) == rows
    else:
        assert ctx.submit_real((rng.standard_normal((S, rows * K)) * 100).astype(np.float32)) == rows


@pytest.mark.parametrize("kind,K,taps,flags,rows,want,fast,opts", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_k1_kernels(native, monkeypatch, kind, K, taps, flags, rows, want, fast, opts):
    from torch.profiler import ProfilerActivity, profile
    for name, value in opts.get("env", {}).items():
        monkeypatch.setenv(name, value)
    rng = np.random.default_rng(K + taps + rows)
    with _context(kind, K, taps, flags, opts.get("unplanned")) as ctx:
        if opts.get("second"):
            _submit(ctx, kind, K, rows, rng)
        ctx.sync()
        ctx.stats(reset=True)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _submit(ctx, kind, K, rows, rng)
            ctx.sync()
        st = ctx.stats()
    ran = collections.Counter(m.group(1) for e in prof.events() if e.device_type.name == "CUDA"
                              for m in [K1_NAME.search(e.name)] if m)
    assert dict(ran) == want
    # every K1 launch counts once beside the demodulator and the block FEC; one channelizer step per submit
    assert (st.kernel_launches, st.chan_launches, st.fast_chan_launches) == (sum(want.values()) + 2, 1, int(fast))
