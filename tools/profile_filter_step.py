"""Per-kernel device times of one C2 vector step: 1M x 768 f32 cosine, top-10, 256 queries through search_vector_keys under AUTO.

    python tools/profile_filter_step.py [--lib path/to/libseekstorm_b200.so] [--steps 50] [--json out.json]

The step time comes from CUDA events around `--steps` back-to-back steps with the profiler off.  A separate run of the same steps under
torch.profiler (CUDA activities) gives every kernel's device time; the table lists each launch of a step in launch order with its median
over the steps, and the step time minus the sum of the kernel times (launch gaps).  --lib selects another build of the library
(SSB_LIB), so that two builds can be profiled one after the other in one session.  The card's name, power limit and clocks are read
with nvidia-smi in the same run: a time means little without them.
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def parse():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--lib", default=None, help="library to load instead of the in-tree build (sets SSB_LIB)")
    p.add_argument("--rows", type=int, default=1_000_000)
    p.add_argument("--dims", type=int, default=768)
    p.add_argument("--batch", type=int, default=256)
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--json", default=None, help="also write the result as JSON to this path")
    return p.parse_args()


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    except (OSError, subprocess.SubprocessError) as e:
        return {"error": str(e)}
    line = out.strip().splitlines()[0] if out.strip() else ""
    return dict(zip(q.split(","), [x.strip() for x in line.split(",")]))


def short_name(name):
    """`void ssb::vec::tc::scan_tc<256, 3, false, 0, false, true>(...)` -> `scan_tc<256, 3, false, 0, false, true>`"""
    name = re.sub(r"\(.*$", "", name)
    name = re.sub(r"^void\s+", "", name)
    return re.sub(r"^[\w:]*::", "", name)


def main():
    a = parse()
    if a.lib:
        os.environ["SSB_LIB"] = os.path.abspath(a.lib)
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    from seekstorm_b200 import Index, VectorSimilarity, synth

    assert torch.cuda.is_available(), "profile_filter_step.py measures on the GPU"
    dev = torch.device("cuda", 0)
    ix = Index(0, vector_dims=a.dims, vector_similarity=VectorSimilarity.Cosine, max_batch=max(a.batch, 16))
    ix.set_stream(torch.cuda.current_stream().cuda_stream)
    ix.reserve_vectors(a.rows)
    for lv in range((a.rows + 65535) // 65536):   # the corpus bench.py builds for C2
        ix.add_vector_level(lv, synth.gen_vectors(min(65536, a.rows - lv * 65536), a.dims, 1002 * 1000 + lv, dev))
    q = synth.gen_vectors(a.batch, a.dims, 2002, "cpu").to(dev)
    keys = torch.zeros((a.batch, 32), dtype=torch.int64, device=dev)
    ix.set_vector_kernel(0)   # AUTO

    def step():
        ix.search_vector_keys(q, 10, keys)

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    launches = ix.last_stats()["kernel_launches"]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / a.steps
    clocks_after = card()

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            step()
        torch.cuda.synchronize()
    dev_events = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    dev_events.sort(key=lambda e: e.time_range.start)
    if len(dev_events) % a.steps:
        raise SystemExit(f"{len(dev_events)} device activities over {a.steps} steps: not one sequence per step")
    per = len(dev_events) // a.steps
    names = [short_name(e.name) for e in dev_events[:per]]
    for s in range(a.steps):
        got = [short_name(e.name) for e in dev_events[s * per:(s + 1) * per]]
        if got != names:
            raise SystemExit(f"step {s} ran {got}, step 0 ran {names}")
    dur = np.array([[dev_events[s * per + i].time_range.elapsed_us() for i in range(per)] for s in range(a.steps)]) / 1e3   # ms
    med = np.median(dur, axis=0)
    kernel_sum = float(np.median(dur.sum(axis=1)))

    rows = [{"launch": i, "name": n, "median_ms": float(m)} for i, (n, m) in enumerate(zip(names, med))]
    scan = max(rows, key=lambda r: r["median_ms"])
    res = {"card": card(), "card_after_timed_steps": clocks_after, "lib": os.environ.get("SSB_LIB", "in-tree"),
           "workload": f"{a.rows} x {a.dims} f32 cosine, top-10, {a.batch} queries per step, AUTO", "steps": a.steps,
           "kernel_launches": int(launches), "step_ms": step_ms, "kernel_sum_ms": kernel_sum, "gaps_ms": step_ms - kernel_sum,
           "scan_kernel_ms": scan["median_ms"], "chain_ms": step_ms - scan["median_ms"], "kernels": rows}
    print(f"card: {res['card']}")
    print(f"lib: {res['lib']}   kernel_launches: {launches}")
    print(f"{'#':>2}  {'kernel':<60} {'median ms':>10}")
    for r in rows:
        print(f"{r['launch']:>2}  {r['name'][:60]:<60} {r['median_ms']:>10.4f}")
    print(f"    {'sum of kernels':<60} {kernel_sum:>10.4f}")
    print(f"    {'step (CUDA events, profiler off)':<60} {step_ms:>10.4f}")
    print(f"    {'gaps (step - sum of kernels)':<60} {step_ms - kernel_sum:>10.4f}")
    print(f"    {'chain (step - scan kernel)':<60} {step_ms - scan['median_ms']:>10.4f}")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
