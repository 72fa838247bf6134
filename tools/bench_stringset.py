"""Multi-value string facets (StringSet32) on the C3 corpus: member filters, member counts and the empty query, next to String16.

Builds bench.py's C3 law on the GPU from a seed (10 M docs Zipf(1) over 1 M terms, 64K-doc levels) with two facets:
  tags  StringSet32: 1..5 distinct tags per doc out of --tags (5,000) drawn Zipf(1) by rank; member id = tag rank (the strings
        "tag0000".. sort like their ranks), combinations numbered by np.unique of the sorted tag lists
  cat   String16: 1,000 values, Zipf(1.3) ids (bench_facets' `brand`)
The tag filter is one tag (member --tag, Zipf rank 10 by default); the String16 filter is the one cat id whose share of the docs is
closest to the tag's, so both one-value filters pass about the same docs (both shares are reported).
Each step runs 1024 OR queries of bench.bm25_queries' law with k = 10:
  topk_tag / topk_cat                 Topk behind the tag / the cat filter
  topkcount_tag / topkcount_cat       TopkCount behind the tag / the cat filter
  count_tags / count_cat              TopkCount, then ssb_search_lexical_facets of the batch: tags length 10 / cat length 10
  empty_tag                           ssb_search_empty, --empty-queries queries with the tag filter, k = 10, TopkCount
  empty_tag_counts                    ssb_search_empty_facets, tags length 10 (index-wide)
The variants run alternated, R rounds of W warm-up and K timed steps each (a host clock; every call ends in a device synchronise); per
variant the median queries/s (calls/s for empty_tag_counts), and the last call's kernel time and algorithmic bytes (ssb_last_stats).
The card's name and power limit are read in the same run.  One JSON line on stdout; --out also writes it to a file.

    python tools/bench_stringset.py --steps 10 --warmup 2 --rounds 3
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
from seekstorm_b200 import Index, QueryType, ResultType, _lib, synth  # noqa: E402
from seekstorm_b200._lib import SsbFacetField, SsbFacetFilter, SsbFacetRequest, check, lib  # noqa: E402
from seekstorm_b200.index import _hits_array  # noqa: E402

TOPK = 10
COUNT_T = np.dtype([("value", np.uint32), ("pad", np.uint32), ("count", np.uint64)])


def tag_column(n_docs, n_tags, seed):
    """(combination id per doc u32, CSR offsets u64, member ids u32): 1..5 distinct Zipf(1) tags per doc, sorted"""
    r = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, n_tags + 1)
    p /= p.sum()
    k = r.integers(1, 6, n_docs)
    draw = r.choice(n_tags, (n_docs, 5), p=p).astype(np.uint16)
    draw[np.arange(5)[None, :] >= k[:, None]] = 0xFFFF                        # unused slots sort last
    draw.sort(axis=1)
    dup = np.zeros_like(draw, dtype=bool)
    dup[:, 1:] = draw[:, 1:] == draw[:, :-1]
    draw[dup] = 0xFFFF                                                        # distinct tags per doc
    draw.sort(axis=1)
    rows = np.ascontiguousarray(draw).view(np.dtype((np.void, 10))).reshape(-1)
    uniq, inv = np.unique(rows, return_inverse=True)
    combos = uniq.view(np.uint16).reshape(-1, 5)
    sizes = (combos != 0xFFFF).sum(axis=1)
    offs = np.zeros(len(combos) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(sizes)
    members = combos[combos != 0xFFFF].astype(np.uint32)                     # row-major: each combination's tags, ascending
    return inv.astype(np.uint32).reshape(-1), offs, members


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--docs", type=int, default=C3_DOCS)
    p.add_argument("--queries", type=int, default=1024, help="queries per step")
    p.add_argument("--empty-queries", type=int, default=64, help="filter-only queries per empty-query step")
    p.add_argument("--tags", type=int, default=5000)
    p.add_argument("--tag", type=int, default=10, help="member id (Zipf rank) of the filter tag")
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--seed", type=int, default=1011)
    p.add_argument("--out", default=None, help="also write the JSON result here")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_stringset: needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    card, power = gpu_name_and_power_limit(dev.index)
    ix = Index(dev.index, max_batch=max(a.queries, a.empty_queries))
    t0 = time.perf_counter()
    len_sum = 0
    for lv in synth.gen_lexical_corpus(a.docs, C3_VOCAB, a.seed, dev):
        ix.add_synth_level(lv)
        len_sum += int(lv.len_sum_normalized)
    ix.commit(a.docs, len_sum)
    tags, offs, members = tag_column(a.docs, a.tags, a.seed + 1)
    rng = np.random.default_rng(a.seed + 2)
    cat = np.minimum(rng.zipf(1.3, a.docs) - 1, 999).astype(np.uint16)
    rows = np.zeros((a.docs, 6), dtype=np.uint8)
    rows[:, 0:4] = tags.view(np.uint8).reshape(-1, 4)
    rows[:, 4:6] = cat.view(np.uint8).reshape(-1, 2)
    fields = (SsbFacetField * 2)(SsbFacetField(_lib.FACET_STRINGSET32, 0), SsbFacetField(_lib.FACET_STRING16, 4))
    check(lib().ssb_set_facets(ix._h, rows.ctypes.data, 0, a.docs, 6, fields, 2))
    check(lib().ssb_set_facet_string_sets(ix._h, 0, offs.ctypes.data, members.ctypes.data, len(offs) - 1, a.tags))
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    # selectivity: the tag's share of the docs, and the cat id closest to it
    in_set = np.zeros(len(offs) - 1, dtype=bool)
    owner = np.repeat(np.arange(len(offs) - 1), np.diff(offs.astype(np.int64)))
    in_set[owner[members == a.tag]] = True
    tag_share = float(in_set[tags].mean())
    cat_freq = np.bincount(cat, minlength=1000) / a.docs
    cat_set = [int(np.argmin(np.abs(cat_freq - tag_share)))]
    cat_share = float(cat_freq[cat_set].sum())

    qk = bm25_queries(a.queries)
    nq = len(qk)
    hits = _hits_array(max(nq, a.empty_queries) * TOPK)
    nh = np.zeros(max(nq, a.empty_queries), dtype=np.uint32)
    cnt = np.zeros(max(nq, a.empty_queries), dtype=np.uint64)

    def filtered(batch_n, facet, values, terms=True):
        b, keep = ix._lex_batch(qk if terms else [[] for _ in range(batch_n)], QueryType.Union)
        if not terms:
            b.term_offsets = None
        fo = np.arange(batch_n + 1, dtype=np.uint32)
        sv = np.asarray(values, dtype=np.uint64)
        fl = (SsbFacetFilter * batch_n)(*[SsbFacetFilter(facet, _lib.FILTER_SET, 0, 0, 0, len(values)) for _ in range(batch_n)])
        b.filter_offsets, b.filters, b.filter_set_values = fo.ctypes.data, C.addressof(fl), sv.ctypes.data
        return b, (keep, fo, sv, fl)

    plain, keep_plain = ix._lex_batch(qk, QueryType.Union)
    b_tag, keep_tag = filtered(nq, 0, [a.tag])
    b_cat, keep_cat = filtered(nq, 1, cat_set)
    b_etag, keep_etag = filtered(a.empty_queries, 0, [a.tag], terms=False)

    def request(facet):
        arr = (SsbFacetRequest * 1)(SsbFacetRequest(facet, _lib.FACET_COUNT_VALUES, 10, 0, 0, 0, 0, 0, None))
        return arr, np.zeros(nq * 10, dtype=COUNT_T), np.zeros(nq, dtype=np.uint32)
    r_tags, r_cat = request(0), request(1)

    def search(b, rt):
        return lambda: check(lib().ssb_search_lexical(ix._h, C.byref(b), TOPK, int(rt), hits.ctypes.data, nh.ctypes.data, cnt.ctypes.data))

    def counts(r):
        def f():
            search(plain, ResultType.TopkCount)()
            check(lib().ssb_search_lexical_facets(ix._h, C.byref(plain), C.addressof(r[0]), 1, None, r[1].ctypes.data, r[2].ctypes.data))
        return f

    def empty():
        check(lib().ssb_search_empty(ix._h, C.byref(b_etag), None, 0, None, TOPK, int(ResultType.TopkCount), hits.ctypes.data, nh.ctypes.data,
                                     cnt.ctypes.data))

    def empty_counts():
        check(lib().ssb_search_empty_facets(ix._h, C.addressof(r_tags[0]), 1, r_tags[1].ctypes.data, r_tags[2].ctypes.data))

    variants = {"topk_tag": (search(b_tag, ResultType.Topk), nq), "topk_cat": (search(b_cat, ResultType.Topk), nq),
                "topkcount_tag": (search(b_tag, ResultType.TopkCount), nq), "topkcount_cat": (search(b_cat, ResultType.TopkCount), nq),
                "count_tags": (counts(r_tags), nq), "count_cat": (counts(r_cat), nq),
                "empty_tag": (empty, a.empty_queries), "empty_tag_counts": (empty_counts, 1)}
    res = {"metric": "stringset_qps", "card": card, "power_limit": power,
           "config": {"docs": a.docs, "vocab": C3_VOCAB, "queries_per_step": nq, "query_law": "bench.bm25_queries (OR, 2-4 terms)", "k": TOPK,
                      "tags": a.tags, "combinations": len(offs) - 1, "member_occurrences": int(offs[-1]), "filter_tag": a.tag,
                      "tag_filter_share": round(tag_share, 5), "cat_filter_id": cat_set[0], "cat_filter_share": round(cat_share, 5),
                      "empty_queries": a.empty_queries, "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds,
                      "index_build_s": round(build_s, 2)}}
    qps = {n: [] for n in variants}
    stats = {}
    for _ in range(a.rounds):
        for name, (step, per_step) in variants.items():
            for _ in range(a.warmup):
                step()
            t = time.perf_counter()
            for _ in range(a.steps):
                step()
            s = time.perf_counter() - t
            qps[name].append(per_step * a.steps / s)
            stats[name] = ix.last_stats()
    for name in variants:
        sv = stats[name]
        res[name] = {"per_s": round(statistics.median(qps[name]), 1), "per_s_rounds": [round(x, 1) for x in qps[name]],
                     "kernel_ms": round(sv["dominant_kernel_ns"] / 1e6, 3), "algorithmic_bytes": sv["algorithmic_bytes"],
                     "launches": sv["kernel_launches"]}
    ix.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
