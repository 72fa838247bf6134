#!/usr/bin/env python
"""SASS evidence of the built library: per kernel, how many warpgroup-MMA / TMA / FP32 instructions it contains.

  python tools/sass_opcodes.py

(PTX names never appear in SASS: wgmma.mma_async -> HGMMA (f16 / bf16 / tf32) or IGMMA (s8), cp.async.bulk.tensor -> UTMALDG;
HMMA / IMMA would be the warp-level tensor paths — none is expected.)"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "seekstorm_b200", "libseekstorm_b200.so")
PAT = ["HGMMA", "IGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UBLKCP", "UTMAPF", "SYNCS", "FFMA",
       "HMMA", "IMMA", "LDL", "STL", "LDG", "LDS", "STS", "ATOM", "RED", "SHFL", "VOTE", "POPC", "F2F", "HADD2", "MUFU", "BAR"]


def main():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    fn = None
    counts = collections.OrderedDict()
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            counts[fn] = collections.Counter()
            continue
        if fn is None:
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_.]+)", line)
        if m:
            op = m.group(1).split(".")[0]
            counts[fn][op] += 1
            counts[fn]["_total"] += 1
    demangled = subprocess.run(["c++filt"], input="\n".join(counts.keys()), capture_output=True, text=True).stdout.splitlines()
    print(f"# {os.path.relpath(LIB, ROOT)}: SASS opcode counts per kernel (cuobjdump -sass, sm_90a)")
    print("# kernel | total | " + " ".join(PAT))
    for (fn, c), dn in zip(counts.items(), demangled):
        name = re.sub(r"\(.*", "", dn)[:70]
        if not any(k in name for k in ("scan_tc", "scan_ffma", "lex_", "merge_lists", "kth", "prep_", "split_", "quantize", "fill_bounds", "build_")):
            continue
        cols = " ".join(f"{p}={c[p]}" for p in PAT if c[p])
        print(f"{name:72s} total={c['_total']:6d}  {cols}")
    tot = collections.Counter()
    for c in counts.values():
        tot.update(c)
    print("# library totals: " + " ".join(f"{p}={tot[p]}" for p in PAT if tot[p]))


if __name__ == "__main__":
    sys.exit(main())
