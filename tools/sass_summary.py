#!/usr/bin/env python
"""Static evidence from the build itself (no GPU needed): per kernel, the ptxas resource line
(registers, spills, static shared memory) and the SASS mnemonic counts that show which hardware
paths the code uses (UBLKCP = cp.async.bulk / TMA bulk copy, SYNCS = mbarrier, ATOMS / ATOMG =
shared / global atomics, POPC, REDUX, ...).

    python tools/sass_summary.py > sass_summary.txt

Rebuilds the product with `-Xptxas -v` and disassembles the objects with cuobjdump."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from croaring_b200 import build as b  # noqa: E402

KEYS = ["UBLKCP", "SYNCS", "LDG", "STG", "LDS", "STS", "ATOMS", "ATOMG", "RED", "POPC", "REDUX", "SHFL", "VOTE",
        "MATCH", "BAR", "LDL", "STL", "FLO", "BREV", "LOP3"]


def demangle(name):
    out = subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip()
    return re.sub(r"\(.*", "", out).replace("void ", "").replace("rb200::", "")


def main():
    log = subprocess.run([sys.executable, "-m", "croaring_b200.build", "--force", "--verbose"], cwd=ROOT,
                         capture_output=True, text=True)
    text = log.stdout + log.stderr
    res = {}
    pat = re.compile(r"Compiling entry function '([^']+)' for 'sm_90a'\n(?:ptxas info\s*:\s*Function properties for [^\n]+\n)?"
                     r"\s*(?:ptxas info\s*:\s*)?(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                     r"ptxas info\s*:\s*Used (\d+) registers(?:, used (\d+) barriers)?(?:, (\d+) bytes smem)?")
    for name, stack, ss, sl, regs, _bars, smem in pat.findall(text):
        res[demangle(name)] = dict(regs=int(regs), stack=int(stack), spill_st=int(ss), spill_ld=int(sl), smem=int(smem or 0))
    counts = {}
    for s in b.SOURCES:
        obj = os.path.join(b.CSRC, s.replace(".cu", ".o"))
        sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
        cur = None
        for line in sass.splitlines():
            m = re.match(r"\s*Function : (\S+)", line)
            if m:
                cur = demangle(m.group(1))
                counts[cur] = collections.Counter()
                continue
            m = re.match(r"\s*/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_]*)", line)
            if m and cur:
                counts[cur][m.group(1)] += 1
                counts[cur]["_total"] += 1
    print("# kernel: registers / stack / spill st+ld bytes / static smem | SASS instructions | mnemonic counts")
    print("# (sm_90a, nvcc " + subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-2].strip() + ")")
    for k in sorted(counts):
        r = res.get(k, {})
        c = counts[k]
        mn = " ".join(f"{x}={c[x]}" for x in KEYS if c[x])
        print(f"{k}: regs={r.get('regs', '?')} stack={r.get('stack', '?')} spill={r.get('spill_st', '?')}+{r.get('spill_ld', '?')} "
              f"smem={r.get('smem', '?')} | sass={c['_total']} | {mn}")


if __name__ == "__main__":
    main()
