"""Check that two builds of libacars_b200.so carry the same machine code for every kernel of the first.

    python tools/sass_same.py OLD.so NEW.so

Dumps both with `cuobjdump -sass`, splits the listings per function and compares, for every function of OLD, its
listing in NEW instruction for instruction (the per-file `identifier = <source path>` trailer is not code and is
skipped).  Prints each function that is missing or differs and exits 1 if there is one; prints nothing and exits 0
otherwise.  Functions only NEW has (new kernels) are not compared.
"""
from __future__ import annotations

import re
import shutil
import subprocess
import sys


def functions(lib: str) -> dict[str, list[str]]:
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([tool, "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs: dict[str, list[str]] = {}
    cur = None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None and not line.lstrip().startswith("identifier ="):
            funcs[cur].append(line)
    return funcs


def main() -> int:
    if len(sys.argv) != 3:
        print(__doc__, file=sys.stderr)
        return 2
    old, new = functions(sys.argv[1]), functions(sys.argv[2])
    bad = [name for name in old if old[name] != new.get(name)]
    for name in bad:
        print(("differs: " if name in new else "missing: ") + name)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
