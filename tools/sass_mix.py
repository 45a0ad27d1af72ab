"""Instruction mix of the exact channelizer kernels, read from the compiled library with cuobjdump (no GPU needed).

For each exact channelizer kernel (k_channelize*, not the fast forms and not the generic fall-backs) it finds the
innermost loop that does the MACs — of the loops closed by a backward branch, the one with the most FMUL, the shortest
on a tie — and reports its instruction mix, instructions per MAC, registers and local memory (spills).  A complex MAC
(u8 / CS16) is 4 FMUL, a real one (float32 input) 2 FMUL; the MACs of a trip are counted from its FMUL.

  python tools/sass_mix.py [library]          (default: acarsdec_b200/libacars_b200.so; prints one JSON line per kernel)
"""
import json
import os
import re
import shutil
import subprocess
import sys
from collections import Counter
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
KERNEL = re.compile(r"_ZN3acb\d+k_channelize(?:_iq4|_real4)?I")     # exact kernels only
LINE = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)([^;]*);")


def cuobjdump() -> str:
    for cand in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("cuobjdump not found")


def functions(sass: str):
    """{mangled name: [(address, opcode, operands)]}"""
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
            continue
        m = LINE.search(line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(3), m.group(4)))
    return out


def mac_loop(ins):
    """(first, last) index of the innermost loop holding the most FMUL"""
    index = {a: i for i, (a, _, _) in enumerate(ins)}
    best = None
    for i, (a, op, args) in enumerate(ins):
        m = re.match(r"\s*(0x[0-9a-f]+)", args)
        if op.startswith("BRA") and m and int(m.group(1), 16) < a and int(m.group(1), 16) in index:
            j = index[int(m.group(1), 16)]
            fmul = sum(1 for _, o, _ in ins[j:i + 1] if o.split(".")[0] == "FMUL")
            key = (fmul, -(i - j))
            if best is None or key > best[0]:
                best = (key, j, i)
    return None if best is None else (best[1], best[2])


def kind(name: str) -> str:
    if "real4" in name or re.search(r"k_channelizeILb", name) or "ILi1E" in name:
        return "real"
    return "cs16" if "ILi2E" in name else "u8"


def resources(lib: str):
    r = subprocess.run([cuobjdump(), "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    out = {}
    for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", r):
        out[m.group(1)] = {"registers": int(m.group(2)), "stack": int(m.group(3)), "shared_static": int(m.group(4)),
                           "local": int(m.group(5))}
    return out


def main() -> None:
    lib = sys.argv[1] if len(sys.argv) > 1 else str(ROOT / "acarsdec_b200" / "libacars_b200.so")
    sass = subprocess.run([cuobjdump(), "-sass", lib], capture_output=True, text=True, check=True).stdout
    res = resources(lib)
    for name, ins in sorted(functions(sass).items()):
        if not KERNEL.match(name):
            continue
        loop = mac_loop(ins)
        if loop is None:
            continue
        body = ins[loop[0]:loop[1] + 1]
        mix = Counter(op.split(".")[0] for _, op, _ in body)
        k = kind(name)
        macs = mix["FMUL"] / (2 if k == "real" else 4)
        spills = sum(mix[o] for o in ("LDL", "STL"))
        print(json.dumps({"kernel": name, "input": k, "loop_instructions": len(body), "macs_per_trip": macs,
                          "instructions_per_mac": round(len(body) / macs, 3) if macs else None,
                          "mix": dict(mix.most_common()), "spill_instructions_in_loop": spills,
                          **res.get(name, {}), "library": os.path.relpath(lib, ROOT)}))


if __name__ == "__main__":
    main()
