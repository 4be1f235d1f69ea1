"""profiles/r2_sass_summary.txt: per kernel of the shipped libian_b200.so, the SASS mnemonics that prove the Hopper
paths (wgmma.mma_async -> HGMMA, wgmma.fence / wait_group -> WARPGROUP.ARRIVE / WARPGROUP.DEPBAR, TMA -> UTMALDG / UTMASTG /
UBLKCP) plus registers / shared memory from --dump-resource-usage.

usage: python tools/sass_summary.py > profiles/r2_sass_summary.txt      (no GPU needed)
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "neural-photo-editor_b200", "libian_b200.so")
PAT = re.compile(r"\b(HGMMA\.[0-9x]+\.F32\.BF16|WARPGROUP\.ARRIVE|WARPGROUP\.DEPBAR|UTMALDG(?:\.[0-9]D)?|UTMASTG|UBLKCP|"
                 r"SYNCS\.[A-Z]+|HMMA|FFMA|MUFU\.[A-Z0-9]+|LDGSTS|RED|ATOM[GS]?|"
                 r"PREEXIT|ACQBULK)\b")   # griddepcontrol.launch_dependents / .wait (PDL)


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    out = [d.replace("ian::(anonymous namespace)::", "").replace("(anonymous namespace)::", "").replace("void ", "") for d in out]
    return [d[:d.index("(")] if "(" in d else d for d in out]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    res = subprocess.run(["cuobjdump", "--dump-resource-usage", LIB], capture_output=True, text=True, check=True).stdout
    usage = {}
    cur = None
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = m.group(1)
        m = re.search(r"REG:(\d+).*SHARED:(\d+)", line)
        if m and cur:
            usage[cur] = (int(m.group(1)), int(m.group(2)))
    counts, order = collections.OrderedDict(), []
    cur = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.x]+)", line)   # x: HGMMA.64x128x16
        if m:
            op = m.group(1)
            counts[cur]["_total"] += 1
            k = PAT.match(op)
            if k:
                counts[cur][k.group(1)] += 1
    names = list(counts)
    pretty = demangle(names)
    print("# SASS summary of %s (cuobjdump -sass; CUDA 12.9, sm_90a)" % os.path.relpath(LIB, ROOT))
    print("# kernel | regs | static smem | instructions | Hopper / tensor mnemonics (count)")
    for n, p in sorted(zip(names, pretty), key=lambda t: t[1]):
        c = counts[n]
        key = {k: v for k, v in c.items() if k != "_total" and not k.startswith(("FFMA", "MUFU", "SYNCS", "RED", "ATOM"))}
        other = {k: v for k, v in c.items() if k.startswith(("FFMA", "MUFU", "ATOM", "RED"))}
        r = usage.get(n, ("?", "?"))
        print("%s | %s | %s | %d | %s | %s" % (p, r[0], r[1], c["_total"],
                                             ", ".join("%s x%d" % kv for kv in sorted(key.items())) or "-",
                                             ", ".join("%s x%d" % kv for kv in sorted(other.items())) or "-"))
    tot = collections.Counter()
    for c in counts.values():
        tot.update({k: v for k, v in c.items() if k.startswith(("HGMMA", "UTMA", "HMMA"))})
    print("# totals: " + ", ".join("%s x%d" % kv for kv in sorted(tot.items())))
    print("# HMMA (legacy mma.sync) x%d: none expected" % tot.get("HMMA", 0))


if __name__ == "__main__":
    main()
