"""Geo search on a Point facet (SSB_FILTER_POINT filters, nearest-first sorting) on the C3 corpus, host-facing throughput.

Builds bench.py's C3 law on the GPU from a seed (10 M docs Zipf(1) over 1 M terms, 64K-doc levels) with two facets: `loc` a Point facet
of uniform positions in [40, 60] deg N x [5, 25] deg E (one side of 0 deg latitude / longitude, so the Morton intervals are proper) and
`price` a random U32.  Each step searches 1024 OR queries of bench.bm25_queries' law with k = 10:
  unfiltered                 Topk / TopkCount
  u32_filter                 price < 10 % of the U32 range                                  Topk / TopkCount
  point_filter               within 320 km of a per-query base drawn in [45, 55] x [10, 20]  (about 10 % of the docs)  Topk / TopkCount
  u32_filter_one_point       the u32 filter on every query, plus a Point filter on query 0 only: a batch with a Point filter plans
                             every filtered query off the lex_score record path — this variant shows what that costs the others (Topk)
  price_asc                  sorted by the U32 facet, Topk / TopkCount
  nearest                    sorted by the distance to the per-query base, ascending, Topk / TopkCount
W warm-up steps, then K steps timed with a host clock (every call ends in a device synchronise).  Per variant: queries/s, ms per step, the
dominant kernel's time (ssb_last_stats), items processed / skipped, mean hits and counts; the card's name and power limit are read in the
same run.  One JSON line on stdout; --out also writes it to a file.

    python tools/bench_geo.py --steps 20 --warmup 3
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import C3_DOCS, C3_VOCAB, bm25_queries  # noqa: E402
from bench_phrase_multifield import gpu_name_and_power_limit  # noqa: E402
from seekstorm_b200 import DistanceUnit, FacetFilter, Index, QueryType, ResultSort, ResultType, SortOrder, synth  # noqa: E402
from seekstorm_b200._lib import check, lib  # noqa: E402
from seekstorm_b200.index import _hits_array  # noqa: E402

TOPK = 10
RADIUS_KM = 320.0


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--docs", type=int, default=C3_DOCS)
    p.add_argument("--queries", type=int, default=1024, help="queries per step")
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--seed", type=int, default=1005)
    p.add_argument("--out", default=None, help="also write the JSON result here")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_geo: needs a CUDA device")
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
    ix.set_facets({"loc": loc, "price": rng.integers(0, 2**32, a.docs, dtype=np.uint32)}, point_facets=("loc",))
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    qk = bm25_queries(a.queries)
    nq = len(qk)
    bases = np.ascontiguousarray(np.stack([rng.uniform(45.0, 55.0, nq), rng.uniform(10.0, 20.0, nq)], axis=1))
    u32 = [FacetFilter("price", 0, 2**32 // 10)]
    geo = [[FacetFilter("loc", 0.0, RADIUS_KM, base=(float(la), float(lo)), unit=DistanceUnit.Kilometers)] for la, lo in bases]
    batches = {"none": ix._lex_batch(qk, QueryType.Union), "u32": ix._lex_batch(qk, QueryType.Union, None, [u32] * nq),
               "point": ix._lex_batch(qk, QueryType.Union, None, geo),
               "u32_one_point": ix._lex_batch(qk, QueryType.Union, None, [u32 + geo[0]] + [u32] * (nq - 1))}
    hits = _hits_array(nq * TOPK); nh = np.zeros(nq, dtype=np.uint32); cnt = np.zeros(nq, dtype=np.uint64)
    res = {"metric": "geo_lexical_qps", "card": card, "power_limit": power,
           "config": {"docs": a.docs, "vocab": C3_VOCAB, "queries_per_step": nq, "query_law": "bench.bm25_queries (OR, 2-4 terms)", "k": TOPK,
                      "facets": "loc Point uniform in [40, 60] N x [5, 25] E, price random U32",
                      "filters": f"price < 2^32 / 10; loc within {RADIUS_KM} km of a per-query base in [45, 55] x [10, 20]",
                      "steps": a.steps, "warmup": a.warmup, "index_build_s": round(build_s, 2)}}
    price_asc, _ = ix._sort_criteria([ResultSort("price", SortOrder.Ascending)])
    nearest, _ = ix._sort_criteria([ResultSort("loc", SortOrder.Ascending)])
    variants = [("unfiltered_topk", "none", None, ResultType.Topk), ("unfiltered_topkcount", "none", None, ResultType.TopkCount),
                ("u32_filter_topk", "u32", None, ResultType.Topk), ("u32_filter_topkcount", "u32", None, ResultType.TopkCount),
                ("point_filter_topk", "point", None, ResultType.Topk), ("point_filter_topkcount", "point", None, ResultType.TopkCount),
                ("u32_filter_one_point_topk", "u32_one_point", None, ResultType.Topk),
                ("price_asc_topk", "none", price_asc, ResultType.Topk), ("price_asc_topkcount", "none", price_asc, ResultType.TopkCount),
                ("nearest_topk", "none", nearest, ResultType.Topk), ("nearest_topkcount", "none", nearest, ResultType.TopkCount)]
    for name, batch, crit, rt in variants:
        b = batches[batch][0]
        if crit is None:
            def step(b=b, rt=rt):
                check(lib().ssb_search_lexical(ix._h, C.byref(b), TOPK, int(rt), hits.ctypes.data, nh.ctypes.data, cnt.ctypes.data))
        else:
            def step(b=b, rt=rt, crit=crit):
                check(lib().ssb_search_lexical_sorted_ex(ix._h, C.byref(b), C.addressof(crit), 1, bases.ctypes.data, TOPK, int(rt), hits.ctypes.data,
                                                         nh.ctypes.data, cnt.ctypes.data))
        for _ in range(a.warmup):
            step()
        t = time.perf_counter()
        for _ in range(a.steps):
            step()
        s = time.perf_counter() - t
        sv = ix.last_stats()
        res[name] = {"queries_per_s": round(nq * a.steps / s, 1), "ms_per_step": round(s * 1e3 / a.steps, 3),
                     "scoring_kernel_ms": round(sv["dominant_kernel_ns"] / 1e6, 3), "items_processed": sv["items_processed"],
                     "items_skipped": sv["items_skipped"], "mean_hits": round(float(nh.mean()), 2),
                     "mean_count": round(float(cnt.mean()), 1) if rt == ResultType.TopkCount else None}
    ix.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
