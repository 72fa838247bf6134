"""Facet counts (ssb_search_lexical_facets) next to a lexical search on the C3 corpus, host-facing throughput.

Builds bench.py's C3 law on the GPU from a seed (10 M docs Zipf(1) over 1 M terms, 64K-doc levels) with three facets: `price` a random U32,
`brand` a String16 facet of 1 000 values (Zipf-like ids) and `loc` a Point facet of uniform positions in [40, 60] deg N x [5, 25] deg E.
Each step searches 1024 OR queries of bench.bm25_queries' law with k = 10, TopkCount, and then counts facets of the same batch:
  search            the search alone
  search_u32        + one U32 range facet with 10 ranges                                    (a)
  search_string     + one String16 facet, length 10                                         (b)
  search_all        + (a) + (b) + a Point facet with 5 distance ranges from a per-query base (c)
The variants run alternated, R rounds of W warm-up and K timed steps each (a host clock; every call ends in a device synchronise); per
variant the median queries/s over the rounds, the facet call's kernel time (lex_facets, ssb_last_stats) and its algorithmic bytes.  The
card's name and power limit are read in the same run.  One JSON line on stdout; --out also writes it to a file.

    python tools/bench_facets.py --steps 10 --warmup 2 --rounds 3
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import C3_DOCS, C3_VOCAB, bm25_queries  # noqa: E402
from bench_phrase_multifield import gpu_name_and_power_limit  # noqa: E402
from seekstorm_b200 import DistanceUnit, Index, QueryFacet, QueryType, ResultType, synth  # noqa: E402
from seekstorm_b200._lib import check, lib  # noqa: E402
from seekstorm_b200.index import _hits_array  # noqa: E402

TOPK = 10


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--docs", type=int, default=C3_DOCS)
    p.add_argument("--queries", type=int, default=1024, help="queries per step")
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--seed", type=int, default=1007)
    p.add_argument("--out", default=None, help="also write the JSON result here")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_facets: needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    card, power = gpu_name_and_power_limit(dev.index)
    ix = Index(dev.index, max_batch=a.queries)
    t0 = time.perf_counter()
    len_sum = 0
    for lv in synth.gen_lexical_corpus(a.docs, C3_VOCAB, a.seed, dev):
        ix.add_synth_level(lv)
        len_sum += int(lv.len_sum_normalized)
    ix.commit(a.docs, len_sum)
    rng = np.random.default_rng(a.seed + 1)
    loc = np.stack([rng.uniform(40.0, 60.0, a.docs), rng.uniform(5.0, 25.0, a.docs)], axis=1)
    brand = np.minimum(rng.zipf(1.3, a.docs) - 1, 999).astype(np.uint16)
    ix.set_facets({"price": rng.integers(0, 2**32, a.docs, dtype=np.uint32), "brand": brand, "loc": loc}, string_facets=("brand",),
                  point_facets=("loc",), string_values={"brand": [f"brand{i:04d}" for i in range(1000)]})
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    qk = bm25_queries(a.queries)
    nq = len(qk)
    b, keep = ix._lex_batch(qk, QueryType.Union)
    hits = _hits_array(nq * TOPK); nh = np.zeros(nq, dtype=np.uint32); cnt = np.zeros(nq, dtype=np.uint64)
    base = np.ascontiguousarray(np.stack([rng.uniform(45.0, 55.0, nq), rng.uniform(10.0, 20.0, nq)], axis=1))
    fa = QueryFacet("price", ranges=[(f"p{i}", i * (2**32 // 10)) for i in range(10)])
    fb = QueryFacet("brand", length=10)
    fc = QueryFacet("loc", ranges=[(f"d{i}", s) for i, s in enumerate((0.0, 50.0, 100.0, 250.0, 500.0))], base=(50.0, 15.0),
                    unit=DistanceUnit.Kilometers)
    sets = {"search": None, "search_u32": [fa], "search_string": [fb], "search_all": [fa, fb, fc]}
    calls = {}
    for name, qfs in sets.items():
        if qfs is None:
            calls[name] = None
            continue
        arr, n_req, kept, meta = ix._facet_requests(qfs)
        stride = sum(qf.length if qf.field == "brand" else len(qf.ranges) for _, _, qf in meta)
        out = np.zeros(nq * stride, dtype=[("value", np.uint32), ("pad", np.uint32), ("count", np.uint64)])
        n_out = np.zeros(nq * n_req, dtype=np.uint32)
        has_point = any(qf.field == "loc" for _, _, qf in meta)
        calls[name] = (arr, n_req, kept, out, n_out, base if has_point else None)
    res = {"metric": "facet_counts_qps", "card": card, "power_limit": power,
           "config": {"docs": a.docs, "vocab": C3_VOCAB, "queries_per_step": nq, "query_law": "bench.bm25_queries (OR, 2-4 terms)", "k": TOPK,
                      "result_type": "TopkCount", "facets": "price random U32 (10 ranges); brand String16, 1000 values, length 10; "
                      "loc Point uniform in [40, 60] N x [5, 25] E, 5 distance ranges from a per-query base",
                      "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds, "index_build_s": round(build_s, 2)}}
    qps = {n: [] for n in sets}
    stats = {}
    for _ in range(a.rounds):
        for name in sets:
            fcall = calls[name]

            def step(fcall=fcall):
                check(lib().ssb_search_lexical(ix._h, C.byref(b), TOPK, int(ResultType.TopkCount), hits.ctypes.data, nh.ctypes.data,
                                               cnt.ctypes.data))
                if fcall is not None:
                    arr, n_req, _, out, n_out, bs = fcall
                    check(lib().ssb_search_lexical_facets(ix._h, C.byref(b), C.addressof(arr), n_req, bs.ctypes.data if bs is not None else None,
                                                          out.ctypes.data, n_out.ctypes.data))
            for _ in range(a.warmup):
                step()
            t = time.perf_counter()
            for _ in range(a.steps):
                step()
            s = time.perf_counter() - t
            qps[name].append(nq * a.steps / s)
            sv = ix.last_stats()
            stats[name] = sv
    for name in sets:
        sv = stats[name]
        r = {"queries_per_s": round(statistics.median(qps[name]), 1), "queries_per_s_rounds": [round(x, 1) for x in qps[name]]}
        if calls[name] is not None:
            r.update(facet_kernel_ms=round(sv["dominant_kernel_ns"] / 1e6, 3), facet_algorithmic_bytes=sv["algorithmic_bytes"],
                     facet_launches=sv["kernel_launches"])
        else:
            r.update(scoring_kernel_ms=round(sv["dominant_kernel_ns"] / 1e6, 3), mean_count=round(float(cnt.mean()), 1))
        res[name] = r
    ix.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
