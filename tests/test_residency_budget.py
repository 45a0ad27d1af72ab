"""The demodulator's residency budget beside the exact IQ channelizer, checked on the compiled library (no GPU).

k_demod2 of submit i runs underneath k_channelize_iq4 of submit i+1.  At bench.py's shape (4224 streams x 8 channels on
132 SMs) an SM's share of the demodulator is eight one-warp CTAs, and the launch rules in kernels.cu are built so that
all eight become resident as soon as ONE of the SM's three channelizer CTAs has retired.  That rests on what ptxas makes
of both kernels (registers per thread, static shared memory), so a change to either that breaks it fails here instead of
costing a few per cent of the step on an H100."""
import shutil
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))

FLAGSHIP_CHAINS, H100_SMS = 4224 * 8, 132
K2_WARPS_PER_SM = 8


def _have_nvcc() -> bool:
    from acarsdec_b200 import build
    try:
        build.nvcc()
    except RuntimeError:
        return False
    return bool(shutil.which("cuobjdump") or Path("/usr/local/cuda/bin/cuobjdump").exists())


@pytest.fixture(scope="module")
def budget():
    if not _have_nvcc():
        pytest.skip("nvcc / cuobjdump not found")
    from acarsdec_b200 import build
    import residency_budget
    return residency_budget.budget(str(build.build()), FLAGSHIP_CHAINS, H100_SMS)


def test_default_kernels_are_all_found_and_spill_free(budget):
    k1s, k2s, _ = budget
    assert sorted((k["input"], k["ovl"]) for k in k1s) == [("cs16", False), ("cs16", True), ("u8", False), ("u8", True)]
    # one lane: plain and register-capped; 2, 4, 8 lanes pinned: wide and lean schedule
    assert sorted((k["lanes"], k["minb"]) for k in k2s) == [(1, 1), (1, 20), (2, 0), (2, 1), (4, 0), (4, 1), (8, 0), (8, 1)]
    for k in k1s + k2s:
        assert k["local"] == 0, f"{k}: local memory (spills)"


def test_flagship_pair_is_the_capped_one_lane_form(budget):
    _, _, pairs = budget
    sel = [p for p in pairs if p["selected_by_default"]]
    assert sel and all(p["k2"] == {"lanes": 1, "pinned": 0, "minb": 20} for p in sel)
    assert all(p["k2_warps_per_sm"] == K2_WARPS_PER_SM and p["k1_ctas_per_sm"] == 3 for p in sel)


def test_one_retired_channelizer_cta_makes_room_for_an_sms_demodulator(budget):
    _, _, pairs = budget
    flagship = [p for p in pairs if p["selected_by_default"] and p["k1"] == {"input": "u8", "ovl": False}]
    assert len(flagship) == 1
    for p in flagship:
        fits = p["k2_ctas_that_fit"]
        # registers: one K1 CTA's allocation plus what three leave spare
        assert fits["beside_2_k1"]["registers"] >= K2_WARPS_PER_SM, p
        # shared memory: the configuration the demodulator asks for holds them even beside all three K1 CTAs
        assert fits["beside_3_k1"]["smem_k2_config"] >= K2_WARPS_PER_SM, p
        # and something always runs beside a full set of K1 CTAs
        assert fits["beside_3_k1"]["registers"] >= 1, p
