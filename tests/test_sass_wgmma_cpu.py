"""CPU: the warpgroup-MMA chains of every scan_tc instantiation in the built library stay pipelined.

When ptxas serialises a wgmma chain (remarks C7514 / C7520: accumulator registers read, or a compiler-inserted
warpgroup.arrive in a divergent path, between an MMA and its wait) it puts a WARPGROUP.ARRIVE before and a
WARPGROUP.DEPBAR after EVERY HGMMA / IGMMA, so each MMA waits for the previous one to finish.  A pipelined stage
loop has one ARRIVE per stage and one DEPBAR for the wait that keeps one commit group in flight.  Reads the SASS
with cuobjdump; no GPU needed."""
import collections
import os
import re
import shutil
import subprocess

import pytest

from seekstorm_b200 import _lib


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe:
        return exe
    exe = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not found")
    return exe


def _scan_tc_counts():
    out = subprocess.run([_cuobjdump(), "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    counts, fn = collections.OrderedDict(), None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1) if "scan_tc" in m.group(1) else None
            if fn:
                counts[fn] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)", line) if fn else None
        if m:
            op = m.group(1)
            if op.startswith(("HGMMA", "IGMMA")):
                counts[fn]["mma"] += 1
            elif op.startswith("WARPGROUP.DEPBAR"):
                counts[fn]["depbar"] += 1
            elif op.startswith("WARPGROUP.ARRIVE"):
                counts[fn]["arrive"] += 1
    return counts


def test_scan_tc_wgmma_chains_are_not_serialised():
    counts = _scan_tc_counts()
    # 64/128/256 queries x tf32/bf16/fp16 filter/int8 (+ scaled, resident), and the CTA-pair filter scan
    assert len(counts) >= 16, sorted(counts)
    assert any(f.startswith("_ZN3ssb3vec2tc7scan_tcILi256E") for f in counts)
    for fn, c in counts.items():
        assert c["mma"] >= 16, (fn, dict(c))
        # serialised: one DEPBAR (and one ARRIVE) per MMA; pipelined: one per stage-loop copy plus the final wait
        assert c["depbar"] * 4 <= c["mma"], (fn, dict(c))
        assert c["arrive"] * 4 <= c["mma"], (fn, dict(c))
