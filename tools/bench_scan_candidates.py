#!/usr/bin/env python
"""Times the unseeded 256-query filter scan (kernel 8) on the C2 corpus (1M x 768 cosine, top-10, 256 queries per step).

A delete set turns the threshold seed off (vec_scan.h, with_threshold_seed), so every CTA starts with empty lists and the first tiles
are an insert storm.  bench.py only measures the seeded scan; this script covers the other case.  One doc is deleted so that the
results stay those of the full corpus minus that doc.  Prints one JSON line: device ms per step and the scan kernel's ms (CUDA events
the library records around it), with the GPU's name, its power limit and the SM clocks sampled during the timed steps.

usage: python tools/bench_scan_candidates.py [--steps K] [--warmup W] [--rows N] [--kernel 8]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import C2_DIMS, C2_ROWS, TOPK, ClockSampler, gen_vector_level, timed_steps  # noqa: E402


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=10).stdout.strip().split(", ")
        return out[0], float(out[1])
    except Exception:  # pragma: no cover
        return None, None


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--rows", type=int, default=C2_ROWS)
    p.add_argument("--batch", type=int, default=256)
    p.add_argument("--kernel", type=int, default=8)
    a = p.parse_args()
    from seekstorm_b200 import Index, VectorSimilarity, synth
    dev = torch.device("cuda", torch.cuda.current_device())
    ix = Index(dev.index, vector_dims=C2_DIMS, vector_similarity=VectorSimilarity.Cosine, max_batch=a.batch, vector_kernel=a.kernel)
    ix.set_stream(torch.cuda.current_stream().cuda_stream)
    n_levels = (a.rows + 65535) // 65536
    ix.reserve_vectors(a.rows)
    for lv in range(n_levels):
        r = gen_vector_level(lv, a.rows, C2_DIMS, dev)
        ix.add_vector_level(lv, r)
        del r
    ix.set_deleted([a.rows - 1])
    q = synth.gen_vectors(a.batch, C2_DIMS, 2002, "cpu").to(dev)
    keys = torch.zeros((a.batch, 32), dtype=torch.int64, device=dev)

    def step():
        ix.search_vector_keys(q, TOPK, keys)
    sampler = ClockSampler(dev.index)
    ms = timed_steps(step, a.steps, a.warmup, 1, sampler) / a.steps
    clocks = sampler.stop()
    kern_ns = []
    for _ in range(5):
        step()
        torch.cuda.synchronize()
        kern_ns.append(ix.last_stats()["dominant_kernel_ns"])
    name, plimit = power_limit()
    print(json.dumps({"kernel": a.kernel, "rows": a.rows, "batch": a.batch, "deleted_docs": 1, "ms_per_step": ms,
                      "kernel_ms": float(np.median(kern_ns)) / 1e6, "gpu": name, "power_limit_w": plimit, "clocks": clocks,
                      "filter_fallbacks": ix.last_stats().get("filter_fallbacks")}))
    ix.close()


if __name__ == "__main__":
    main()
