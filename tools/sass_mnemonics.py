#!/usr/bin/env python
"""Per-kernel counts of the Hopper-specific SASS mnemonics in the shipped library (cuobjdump -sass, no GPU needed):
    python tools/sass_mnemonics.py
HGMMA/IGMMA = wgmma (f16 / s8), UTMALDG = TMA tensor load, UBLKCP = TMA bulk copy, UTMAPF = TMA prefetch,
IMMA/HMMA = mma.sync, LDSM = ldmatrix, SYNCS = mbarrier ops, USETMAXREG = setmaxnreg, UCGABAR = cluster barrier."""
import collections
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
LIB = ROOT / "tinychatengine_b200" / "lib" / "libtce_b200.so"
COLS = ["HGMMA", "IGMMA", "UTMALDG", "UBLKCP", "UTMAPF", "IMMA", "HMMA", "LDSM", "SYNCS", "USETMAXREG", "REDUX", "UCGABAR"]


def short_name(demangled: str) -> str:
    """'void tce::(anonymous namespace)::k<A, B>(tce::Args)' -> 'k<A, B>': drop namespaces' noise and the parameter list (the last top-level parenthesis)."""
    n = demangled.replace("(anonymous namespace)::", "").replace("tce::", "").replace("void ", "")
    depth, cut = 0, len(n)
    for i in range(len(n) - 1, -1, -1):
        if n[i] == ")":
            depth += 1
        elif n[i] == "(":
            depth -= 1
            if depth == 0:
                cut = i
                break
    return n[:cut]


def main():
    lib = Path(sys.argv[1]) if len(sys.argv) > 1 else LIB
    sass = subprocess.run(["cuobjdump", "-sass", str(lib)], capture_output=True, text=True, check=True).stdout
    names = subprocess.run(["c++filt"], input="\n".join(re.findall(r"Function : (\S+)", sass)), capture_output=True, text=True).stdout.splitlines()
    counts, order, cur, it = collections.defaultdict(collections.Counter), [], None, iter(names)
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = short_name(next(it))
            order.append(cur)
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
        if m and cur:
            op = m.group(1)
            for c in COLS:
                if op == c or op.startswith(c + "_") or (c in ("IMMA", "HMMA", "HGMMA", "IGMMA", "LDSM", "SYNCS", "REDUX", "UCGABAR") and op.startswith(c)):
                    counts[cur][c] += 1
    print(f"SASS mnemonic counts per kernel of {lib.relative_to(ROOT) if lib.is_relative_to(ROOT) else lib} (cuobjdump -sass; sm_90a), kernels that use any of them.")
    print(__doc__.split("tools/sass_mnemonics.py\n", 1)[1].strip())
    print()
    print(f"{'kernel':<78}" + "".join(f"{c[:7]:>8}" for c in COLS))
    for k in sorted(set(order), key=lambda k: (-sum(counts[k].values()), k)):
        if sum(counts[k].values()):
            print(f"{k[:77]:<78}" + "".join(f"{counts[k][c]:>8}" for c in COLS))
    tot = collections.Counter()
    for k in counts:
        tot.update(counts[k])
    print(f"{'TOTAL':<78}" + "".join(f"{tot[c]:>8}" for c in COLS))


if __name__ == "__main__":
    main()
