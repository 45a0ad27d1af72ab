"""Residency budget of the demodulator (K2) beside the exact IQ channelizer (K1), read from the compiled library with
cuobjdump (no GPU needed).

K2 of submit i runs underneath K1 of submit i+1, on a stream of greater priority: whether its one-warp CTAs become
resident as soon as one K1 CTA of an SM retires is a matter of registers and shared memory per CTA, which the compiler
decides.  For the default K1 forms (k_channelize_iq4, u8 and CS16, taps <= K and taps > K) and every k_demod2 instance a
default launch can select, this prints registers per thread, registers per CTA as the hardware allocates them, shared
memory per CTA, and for every pair how many K2 CTAs fit beside 3, 2 and 1 K1 CTAs: in registers, in the shared-memory
configuration K1 asks for and in the one K2 asks for at `--chains` chains on `--sms` SMs.  The launch rules (K1's CTAs
per SM and carve-out, K2's register cap and carve-out) are read from csrc/kernels.cu.

  python tools/residency_budget.py [library] [--chains N] [--sms N]      (one JSON line per kernel, then per pair)
"""
import argparse
import json
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
from sass_mix import cuobjdump  # noqa: E402

SM_REGISTERS = 65536                     # sm_90: 64 K 32-bit registers per SM,
REG_UNIT = 8                             # allocated per warp in units of 256 = 8 per thread
SMEM_CONFIGS_KB = [0, 8, 16, 32, 64, 100, 132, 164, 196, 228]     # sm_90 shared-memory configurations of the 256 KB array
SMEM_PER_SM = 228 * 1024

K1 = re.compile(r"_ZN3acb16k_channelize_iq4ILi(\d)ELb(\d)EEE")
K2 = re.compile(r"_ZN3acb8k_demod2ILi(\d)ELb(\d)ELb(\d)ELi(\d+)EEE")


def launch_rules(src: str) -> dict:
    """The numbers the launchers in kernels.cu use, so that a change there shows here."""
    def one(pattern):
        m = re.search(pattern, src)
        if not m:
            raise RuntimeError(f"kernels.cu: no match for {pattern!r}")
        return int(m.group(1))
    return {
        "k1_threads": one(r"IQ4_THREADS = (\d+)"),
        "k1_ctas_per_sm": one(r"__launch_bounds__\(IQ4_THREADS, (\d+)\)"),
        "k1_carveout_pct": one(r"k_channelize_iq4<MODE, OVL>, cudaFuncAttributePreferredSharedMemoryCarveout, (\d+)\)"),
        "smem_reserved": one(r"DEMOD_SMEM_RESERVED = (\d+)"),
        "k2_max_warps_per_sm": one(r"DEMOD_MAX_WARPS_PER_SM = (\d+)"),
        "k2_min_warps_sharing": one(r"DEMOD_MIN_WARPS_SHARING = (\d+)"),
        "k2_capped_minb": one(r"DEMOD_MINB_96REG = (\d+)"),
        "k2_warps_per_k1_cta": one(r"DEMOD_WARPS_PER_K1_CTA = (\d+)"),
    }


def resources(lib: str) -> dict:
    out = subprocess.run([cuobjdump(), "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    # SHARED is the CTA's whole allocation: the kernel's static shared memory plus the 1 KB the system reserves per CTA
    return {m.group(1): {"registers": int(m.group(2)), "shared_per_cta": int(m.group(3)), "local": int(m.group(4))}
            for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:\d+ SHARED:(\d+) LOCAL:(\d+)", out)}


def cta_registers(regs_per_thread: int, threads: int) -> int:
    return (regs_per_thread + REG_UNIT - 1) // REG_UNIT * REG_UNIT * threads


def smem_config(request_bytes: int) -> int:
    """the smallest configuration that holds a request, in bytes"""
    return next(kb for kb in SMEM_CONFIGS_KB if kb * 1024 >= request_bytes) * 1024


def default_k2(lanes: int, pinned: int, minb: int, rules: dict) -> bool:
    """launch_demod's default arms: one lane unpinned (plain or register-capped), 2 / 4 / 8 lanes pinned (wide or lean)"""
    return (lanes == 1 and not pinned and minb in (1, rules["k2_capped_minb"])) or (lanes > 1 and pinned and minb in (0, 1))


def selected_k2(chains: int, sms: int, rules: dict):
    """(lanes, pinned, minb) of the instance a default launch of `chains` chains on `sms` SMs runs: demod_pick_lanes,
    launch_demod_one_lane and launch_demod_pinned of kernels.cu restated"""
    lanes = next((l for l in (1, 2, 4) if chains * l >= 32 * 4 * sms), 8)
    warps = (chains * lanes + 31) // 32
    if lanes == 1:
        return 1, 0, 1 if warps <= rules["k2_warps_per_k1_cta"] * sms else rules["k2_capped_minb"]
    return lanes, 1, 1 if warps <= 8 * sms else 0


def budget(lib: str, chains: int, sms: int):
    rules = launch_rules((ROOT / "acarsdec_b200" / "csrc" / "kernels.cu").read_text())
    res = resources(lib)
    k1s, k2s = [], []
    for name, r in sorted(res.items()):
        m = K1.match(name)
        if m:
            k1s.append({"kernel": "k_channelize_iq4", "input": "cs16" if m.group(1) == "2" else "u8", "ovl": m.group(2) == "1",
                        "threads": rules["k1_threads"], **r,
                        "cta_registers": cta_registers(r["registers"], rules["k1_threads"])})
        m = K2.match(name)
        if m and m.group(2) == "0" and default_k2(int(m.group(1)), int(m.group(3)), int(m.group(4)), rules):
            k2s.append({"kernel": "k_demod2", "lanes": int(m.group(1)), "pinned": int(m.group(3)), "minb": int(m.group(4)),
                        "threads": 32, **r, "cta_registers": cta_registers(r["registers"], 32)})
    sel = selected_k2(chains, sms, rules)
    pairs = []
    for a in k1s:
        for b in k2s:
            warps = (chains * b["lanes"] + 31) // 32
            per_sm = min((warps + sms - 1) // sms, rules["k2_max_warps_per_sm"])
            k1_smem, k2_smem = a["shared_per_cta"], b["shared_per_cta"]
            # launch_demod_t's request: its CTAs of one SM beside three u8 K1 CTAs, as a whole percentage of the SM's maximum;
            # the maximum itself for launches of less than a warp per scheduler
            need = per_sm * k2_smem + 3 * (4096 + rules["smem_reserved"])
            pct = 100 if per_sm < rules["k2_min_warps_sharing"] else min(100, (need * 100 + SMEM_PER_SM - 1) // SMEM_PER_SM)
            cfg = {"k1": smem_config(SMEM_PER_SM * rules["k1_carveout_pct"] // 100), "k2": smem_config(SMEM_PER_SM * pct // 100)}
            fits = {}
            for n in (3, 2, 1):
                fits[f"beside_{n}_k1"] = {
                    "registers": max(0, SM_REGISTERS - n * a["cta_registers"]) // b["cta_registers"],
                    "smem_k1_config": max(0, cfg["k1"] - n * k1_smem) // k2_smem,
                    "smem_k2_config": max(0, cfg["k2"] - n * k1_smem) // k2_smem}
            pairs.append({"k1": {k: a[k] for k in ("input", "ovl")}, "k2": {k: b[k] for k in ("lanes", "pinned", "minb")},
                          "selected_by_default": (b["lanes"], b["pinned"], b["minb"]) == sel,
                          "chains": chains, "sms": sms, "k2_warps_per_sm": per_sm,
                          "k1_ctas_per_sm": min(rules["k1_ctas_per_sm"], SM_REGISTERS // a["cta_registers"]),
                          "smem_config_bytes": cfg, "k2_ctas_that_fit": fits})
    return k1s, k2s, pairs


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("library", nargs="?", default=str(ROOT / "acarsdec_b200" / "libacars_b200.so"))
    ap.add_argument("--chains", type=int, default=4224 * 8, help="streams x channels of the launch (default: bench.py's 4224 x 8)")
    ap.add_argument("--sms", type=int, default=132, help="SMs of the device (default: H100 SXM)")
    args = ap.parse_args()
    k1s, k2s, pairs = budget(args.library, args.chains, args.sms)
    for row in k1s + k2s + pairs:
        print(json.dumps(row))


if __name__ == "__main__":
    main()
