"""Per-kernel SASS evidence of libsugar_b200.so, printed:
    python scripts/sass_summary.py [tag] > sass_summary.txt
Counts, per kernel, the mnemonics that prove the hardware paths DESIGN.md claims: UBLKCP (1-D TMA bulk copies,
both directions), SYNCS (mbarrier transaction waits), LDGSTS (cp.async), REDG...F32x4 / F32x2 (vector
reductions), ATOMG (returning atomics), MUFU.* (special-function unit), plus registers and static shared memory
from `cuobjdump -res-usage`."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "sugar_b200", "lib", "libsugar_b200.so")
PAT = [("UBLKCP", r"\bUBLKCP"), ("SYNCS", r"\bSYNCS"), ("LDGSTS", r"\bLDGSTS"), ("LDGDEPBAR", r"\bLDGDEPBAR"),
       ("REDG.F32x4", r"\bREDG\S*F32x4"), ("REDG.F32x2", r"\bREDG\S*F32x2"), ("REDG.F32", r"\bREDG\S*\.F32\."),
       ("RED(int)", r"\bREDG\.E\.ADD\.STRONG|\bRED\.E\.ADD\b"), ("ATOMG", r"\bATOMG"), ("ATOMS", r"\bATOMS"),
       ("MUFU.EX2", r"MUFU\.EX2"), ("MUFU.RCP", r"MUFU\.RCP"), ("MUFU.SQRT/RSQ", r"MUFU\.(SQRT|RSQ)"), ("MUFU.LG2", r"MUFU\.LG2"),
       ("LDS.128", r"\bLDS\.128"), ("STS.128", r"\bSTS\.128"), ("BAR.SYNC", r"\bBAR\."), ("VOTE", r"\bVOTE"), ("SHFL", r"\bSHFL"),
       ("STL/LDL", r"\b(STL|LDL)")]


def main(tag):
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    usage = {}
    for m in re.finditer(r"Function (\S+):\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", res):
        usage[m.group(1)] = (int(m.group(2)), int(m.group(3)), int(m.group(4)))
    counts, n_inst, cur = collections.OrderedDict(), {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = collections.Counter()
            n_inst[cur] = 0
            continue
        if cur and re.match(r"\s*/\*[0-9a-f]{4}\*/", line):
            n_inst[cur] += 1
            for name, pat in PAT:
                if re.search(pat, line):
                    counts[cur][name] += 1
    demangle = lambda n: subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip().split("(")[0]
    out = [f"# SASS summary of {os.path.relpath(LIB, ROOT)} ({tag}); made by scripts/sass_summary.py",
           "# instructions = static count; REG / STACK (spill bytes) / static SHARED from cuobjdump -res-usage", ""]
    for k in counts:
        name = demangle(k).replace("sgr::", "")
        if not name or name.startswith("_"):
            continue
        reg, stack, sh = usage.get(k, (0, 0, 0))
        hits = "  ".join(f"{n}={c}" for n, c in counts[k].items() if c)
        out.append(f"{name:48s} inst={n_inst[k]:5d} REG={reg:3d} STACK={stack:3d} SHARED={sh:6d}  {hits}")
    print("\n".join(out))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "r02")
