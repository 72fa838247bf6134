"""The empty query (ssb_search_empty): filter-only batches over every doc of a C3-sized index, host-facing throughput.

The index holds bench.py's C3 doc count (10 M docs in 153 levels of 64K docs); the empty query reads no postings, so each level carries a
single one-posting term.  Facets, drawn from a seed: `price` a random U32 (0 .. 99 999), `brand` a String16 facet of 1 000 Zipf-like ids,
`ts` a Timestamp rising with the doc id (time-ordered ingest) and `loc` a Point facet uniform in [40, 60] deg N x [5, 25] deg E.
Each step is one batch of Q queries (default 1024), k = 10:
  a_newest          no filter, Topk, doc id descending (newest first): only the top tiles are read
  b_brand_price     TopkCount, a 3-brand set and a price range of 20 %
  c_ts_window       TopkCount, a 5 % window of `ts` (the level zones skip or accept whole levels)
  d_price_asc       TopkCount, price ascending under a 1-brand filter
  e_geo_nearest     TopkCount, a 50 km Point filter around a per-query base, nearest first
The variants run alternated, R rounds of W warm-up and K timed steps each (a host clock around calls that end in a device synchronise);
per variant the median queries/s, the scan's kernel time and algorithmic bytes (ssb_last_stats), the kernel's share of the HBM data-sheet
bandwidth (3.35 TB/s, H100 SXM) and the (query, tile) pairs skipped.  The card's name and power limit are read in the same run, and
--check // 5 queries of each variant (60 in all by default) are checked against a numpy restatement: the doc universe, the typed filters,
the sort, ties by doc id descending.  One JSON line on stdout; --out also writes it to a file.

    python tools/bench_empty_query.py --steps 10 --warmup 2 --rounds 3
"""
import argparse
import json
import math
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import C3_DOCS  # noqa: E402
from bench_phrase_multifield import gpu_name_and_power_limit  # noqa: E402
from seekstorm_b200 import DistanceUnit, FacetFilter, Index, ResultSort, ResultType, SortOrder  # noqa: E402
from seekstorm_b200.index import decode_morton_2d, encode_morton_2d, point_column  # noqa: E402

TOPK = 10
HBM_BPS = 3.35e12
DEG2RAD = 0.017453292519943295
RADIUS_KM = 6371.0087714


def build(docs, seed):
    ix = Index(0, max_batch=4096)
    n_levels = (docs + 65535) // 65536
    for lv in range(n_levels):
        n = min(65536, docs - lv * 65536)
        ix.add_lexical_level(lv, n, np.array([8], dtype=np.uint64), np.array([0, 1], dtype=np.uint32), np.array([0], dtype=np.uint16),
                             np.array([1], dtype=np.uint16), np.ones(n, dtype=np.uint8))
    ix.commit(docs, docs)
    r = np.random.default_rng(seed)
    cols = {"price": r.integers(0, 100_000, docs, dtype=np.uint32),
            "brand": np.minimum(r.zipf(1.3, docs) - 1, 999).astype(np.uint16),
            "ts": 1_600_000_000 + np.arange(docs, dtype=np.int64) * 3,
            "loc": np.stack([r.uniform(40.0, 60.0, docs), r.uniform(5.0, 25.0, docs)], axis=1)}
    ix.set_facets(cols, string_facets=("brand",), timestamp_facets=("ts",), point_facets=("loc",))
    return ix, cols, n_levels


def variants(cols, nq, seed):
    """name -> (result_type, filters per query, sort, per-query sort bases or None)"""
    r = np.random.default_rng(seed)
    docs = len(cols["price"])
    b = []
    for _ in range(nq):
        lo = int(r.integers(0, 80_000))
        b.append([FacetFilter("brand", values=[int(x) for x in r.choice(50, 3, replace=False)]), FacetFilter("price", lo, lo + 20_000)])
    c = []
    for _ in range(nq):
        s = int(r.integers(0, docs - docs // 20))
        c.append([FacetFilter("ts", int(cols["ts"][s]), int(cols["ts"][s + docs // 20]))])
    d = [[FacetFilter("brand", values=[int(r.integers(0, 20))])] for _ in range(nq)]
    bases = np.stack([r.uniform(45.0, 55.0, nq), r.uniform(10.0, 20.0, nq)], axis=1)
    e = [[FacetFilter("loc", 0.0, 50.0, base=(float(la), float(lo)), unit=DistanceUnit.Kilometers)] for la, lo in bases]
    return {"a_newest": (ResultType.Topk, None, None, None),
            "b_brand_price": (ResultType.TopkCount, b, None, None),
            "c_ts_window": (ResultType.TopkCount, c, None, None),
            "d_price_asc": (ResultType.TopkCount, d, [ResultSort("price", SortOrder.Ascending)], None),
            "e_geo_nearest": (ResultType.TopkCount, e, [ResultSort("loc", SortOrder.Ascending, base=tuple(bases[0]))], bases)}


def expected(cols, plat, plon, fl, sort, base):
    """one query restated in numpy: (top-k doc ids, count)"""
    n = len(cols["price"])
    m = np.ones(n, dtype=bool)
    for f in fl or ():
        if f.base is not None:
            (lat, lon), (lo, hi) = f.base, (int(encode_morton_2d(f.base[0] - f.end / (DEG2RAD * RADIUS_KM),
                                                                  f.base[1] - f.end / (DEG2RAD * RADIUS_KM * math.cos(DEG2RAD * f.base[0])))),
                                             int(encode_morton_2d(f.base[0] + f.end / (DEG2RAD * RADIUS_KM),
                                                                  f.base[1] + f.end / (DEG2RAD * RADIUS_KM * math.cos(DEG2RAD * f.base[0])))))
            codes = cols["_codes"]
            x = DEG2RAD * (plon - lon) * np.cos(DEG2RAD * (lat + plat) / 2.0)
            y = DEG2RAD * (plat - lat)
            dist = RADIUS_KM * np.sqrt(x * x + y * y)
            m &= (codes >= np.uint64(lo)) & (codes < np.uint64(hi)) & (f.start <= dist) & (dist < f.end)
        elif f.values is not None:
            m &= np.isin(cols[f.field], np.asarray(f.values, dtype=cols[f.field].dtype))
        else:
            m &= (f.start <= cols[f.field]) & (cols[f.field] < f.end)
    d = np.nonzero(m)[0]
    if not sort:
        top = d[::-1][:TOPK]
    elif sort[0].field == "price":
        top = d[np.lexsort((-d, cols["price"][d]))][:TOPK]
    else:
        x = (base[1] - plon[d]) * np.cos(DEG2RAD * (plat[d] + base[0]) / 2.0)
        y = base[0] - plat[d]
        top = d[np.lexsort((-d, x * x + y * y))][:TOPK]
    return [int(v) for v in top], int(m.sum())


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--docs", type=int, default=C3_DOCS)
    p.add_argument("--queries", type=int, default=1024, help="queries per step")
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--check", type=int, default=64, help="queries checked against the numpy restatement, spread over the variants")
    p.add_argument("--seed", type=int, default=2024)
    p.add_argument("--out", default=None, help="also write the JSON result here")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_empty_query: needs a CUDA device")
    card, power = gpu_name_and_power_limit(torch.cuda.current_device())
    t0 = time.perf_counter()
    ix, cols, n_levels = build(a.docs, a.seed)
    build_s = time.perf_counter() - t0
    vs = variants(cols, a.queries, a.seed + 1)
    res = {"metric": "empty_query_qps", "card": card, "power_limit": power,
           "config": {"docs": a.docs, "levels": n_levels, "queries_per_step": a.queries, "k": TOPK, "steps": a.steps, "warmup": a.warmup,
                      "rounds": a.rounds, "index_build_s": round(build_s, 2),
                      "facets": "price U32 0..99999; brand String16 1000 Zipf-like ids; ts Timestamp rising with the doc id; loc Point uniform"}}
    qps = {n: [] for n in vs}
    stats, out = {}, {}
    for _ in range(a.rounds):
        for name, (rt, fl, sort, bases) in vs.items():
            def step():
                return ix.search_empty_batch(a.queries, TOPK, rt, filters=fl, sort=sort, sort_bases=bases)
            for _ in range(a.warmup):
                step()
            t = time.perf_counter()
            for _ in range(a.steps):
                out[name] = step()
            qps[name].append(a.queries * a.steps / (time.perf_counter() - t))
            stats[name] = ix.last_stats()
    cols["_codes"] = point_column(cols["loc"])
    plat, plon = decode_morton_2d(cols["_codes"])
    mismatches, checked = 0, 0
    per = max(1, a.check // len(vs))
    for name, (rt, fl, sort, bases) in vs.items():
        got, counts = out[name]
        for q in np.linspace(0, a.queries - 1, per).astype(int):
            top, cnt = expected(cols, plat, plon, fl[q] if fl else None, sort, bases[q] if bases is not None else None)
            ok = [d for d, _ in got[q]] == top and (rt == ResultType.Topk or int(counts[q]) == cnt)
            mismatches += 0 if ok else 1
            checked += 1
    for name in vs:
        sv = stats[name]
        kern_s = sv["dominant_kernel_ns"] / 1e9
        res[name] = {"queries_per_s": round(statistics.median(qps[name]), 1), "queries_per_s_rounds": [round(x, 1) for x in qps[name]],
                     "kernel_ms": round(kern_s * 1e3, 3), "algorithmic_bytes": sv["algorithmic_bytes"],
                     "hbm_fraction": round(sv["algorithmic_bytes"] / kern_s / HBM_BPS, 4) if kern_s > 0 else None,
                     "items_processed": sv["items_processed"], "items_skipped": sv["items_skipped"]}
    res["check"] = {"queries": checked, "mismatches": mismatches}
    ix.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
