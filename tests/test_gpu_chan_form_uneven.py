"""Which channelizer (K1) kernels one submit launches while a context's streams sit at different positions (taps > K).

The launch runs at the furthest stream's position, and a stream whose window still reaches before its own start is
redone alone at its own position where the form needs it: u8 EXACT and GENERIC through the generic kernel over its
leading rows, u8 / CS16 OVL_FAST and WB with their own kernel.  The forms that read zero history from in front of the
rows (CS16 / real EXACT, OVL_RDFT, WB_REAL) need no second launch.  Contexts and names as in test_gpu_chan_form."""
import collections

import numpy as np
import pytest

from test_gpu_chan_form import (FILTER, FILTER_REAL, GEN_OVL, IQ4, K1_NAME, OVL_FAST, OVL_RDFT, REAL4, S, WB, WB_REAL,
                                WBK, WBK_REAL, _context)

pytestmark = pytest.mark.gpu

# (id, kind, K, taps, flags, rows, K1 kernels, (kernel_launches, chan_launches, fast_chan_launches), how stream 1 falls
# behind).  "reset": one submit, then reset_stream(1); "ragged": stream 1 brings 0 to the first submit; "idle": as "reset",
# and stream 1 brings 0 to the profiled submit (its rows are not redone; the ragged path's own kernels count too).
CASES = [
    ("u8-exact", "u8", 160, 2 * 160, 0, 1024, {IQ4: 1, GEN_OVL: 1}, (4, 1, 0), "reset"),
    ("u8-exact-ragged", "u8", 160, 2 * 160, 0, 1024, {IQ4: 1, GEN_OVL: 1}, (4, 1, 0), "ragged"),
    ("u8-exact-idle", "u8", 160, 2 * 160, 0, 1024, {IQ4: 1}, (4, 1, 0), "idle"),
    ("u8-generic", "u8", 100, 250, 0, 1024, {GEN_OVL: 2}, (4, 1, 0), "reset"),
    ("u8-ovl-fast", "u8", 160, 2 * 160, FILTER, 1024, {OVL_FAST: 2}, (4, 1, 1), "reset"),
    ("u8-wb", "u8", 96, 200, WB, 1024, {WBK: 2}, (4, 1, 1), "reset"),
    ("cs16-exact", "cs16", 160, 2 * 160, 0, 1500, {IQ4: 1, GEN_OVL: 1}, (4, 1, 0), "reset"),
    ("cs16-ovl-fast", "cs16", 160, 2 * 160, FILTER, 1500, {OVL_FAST: 2}, (4, 1, 1), "reset"),
    ("cs16-ovl-fast-idle", "cs16", 160, 2 * 160, FILTER, 1500, {OVL_FAST: 1}, (5, 1, 1), "idle"),
    ("cs16-wb", "cs16", 96, 3 * 96, WB, 1500, {WBK: 2}, (4, 1, 1), "reset"),
    ("real-exact", "real", 200, 2 * 200, 0, 1500, {REAL4: 1, GEN_OVL: 1}, (4, 1, 0), "reset"),
    ("real-ovl-rdft", "real", 200, 2 * 200, FILTER_REAL, 1500, {OVL_RDFT: 1}, (3, 1, 1), "reset"),
    ("real-wb", "real", 200, 2 * 200, WB_REAL, 1500, {WBK_REAL: 1}, (3, 1, 1), "reset"),
]


def _submit(ctx, kind, K, rows, rng, counts=None):
    """One submit of `rows` rows per stream, or (counts, rows per stream) the ragged call"""
    if kind == "u8":
        iq = rng.integers(0, 256, size=(S, rows * 2 * K), dtype=np.uint8)
        if counts is None:
            ctx.submit_host(iq, rows // 1024)
        else:
            ctx.submit_host(iq, counts=[c // 1024 for c in counts])
    elif kind == "cs16":
        iq = rng.integers(-2000, 2000, size=(S, rows * K, 2), dtype=np.int16)
        if counts is None:
            assert ctx.submit_cs16(iq) == rows
        else:
            assert list(ctx.submit_cs16(iq, counts=[c * K for c in counts])) == list(counts)
    else:
        assert ctx.submit_real((rng.standard_normal((S, rows * K)) * 100).astype(np.float32)) == rows


@pytest.mark.parametrize("kind,K,taps,flags,rows,want,counters,behind", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_k1_kernels_uneven(native, kind, K, taps, flags, rows, want, counters, behind):
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(K + taps + rows)
    with _context(kind, K, taps, flags, None) as ctx:
        _submit(ctx, kind, K, rows, rng, counts=(rows, 0) if behind == "ragged" else None)
        if behind != "ragged":
            ctx.reset_stream(1)
        ctx.sync()
        ctx.stats(reset=True)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _submit(ctx, kind, K, rows, rng, counts=(rows, 0) if behind == "idle" else None)
            ctx.sync()
        st = ctx.stats()
    ran = collections.Counter(m.group(1) for e in prof.events() if e.device_type.name == "CUDA"
                              for m in [K1_NAME.search(e.name)] if m)
    got = (st.kernel_launches, st.chan_launches, st.fast_chan_launches)
    assert (dict(ran), got) == (want, counters)
