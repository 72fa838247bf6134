"""Sorted lexical search (`result_sort`, ssb_search_lexical_sorted) on the C3 corpus, host-facing throughput.

Builds bench.py's C3 law on the GPU from a seed (10 M docs Zipf(1) over 1 M terms, 64K-doc levels) with three facets: `ts` a Timestamp
rising with the doc id plus jitter, `price` a random U32 and `lang` a String16 of 40 language codes (sorted by their strings).  Each step
searches 1024 OR queries of bench.bm25_queries' law with k = 10: unsorted first for context, then `ts` desc (Topk and TopkCount),
`price` asc, `price` desc + `lang` asc, and `_id` desc.  W warm-up steps, then K steps timed with a host clock (every call ends in a
device synchronise: the hits are copied to host buffers).  Per variant: queries/s, ms per step, the dominant kernel's time (the scoring
kernel, ssb_last_stats), items processed / skipped and postings visited; the card's name and power limit are read in the same run.
One JSON line on stdout; --out also writes it to a file.

    python tools/bench_sorted.py --steps 20 --warmup 3
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
from seekstorm_b200 import Index, QueryType, ResultSort, ResultType, SortOrder, synth  # noqa: E402
from seekstorm_b200._lib import check, lib  # noqa: E402
from seekstorm_b200.index import _hits_array  # noqa: E402

TOPK = 10
LANGS = ["ar", "bg", "ca", "cs", "da", "de", "el", "en", "es", "et", "fa", "fi", "fr", "he", "hi", "hr", "hu", "id", "it", "ja",
         "ko", "lt", "lv", "ms", "nb", "nl", "pl", "pt", "ro", "ru", "sk", "sl", "sr", "sv", "th", "tr", "uk", "vi", "zh-Hans", "zh-Hant"]


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--docs", type=int, default=C3_DOCS)
    p.add_argument("--queries", type=int, default=1024, help="queries per step")
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--seed", type=int, default=1003)
    p.add_argument("--out", default=None, help="also write the JSON result here")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_sorted: needs a CUDA device")
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
    ts = 1_500_000_000_000 + np.arange(a.docs, dtype=np.int64) * 1000 + rng.integers(0, 5000, a.docs)
    cols = {"ts": ts, "price": rng.integers(0, 2**32, a.docs, dtype=np.uint32), "lang": rng.integers(0, len(LANGS), a.docs, dtype=np.uint16)}
    ix.set_facets(cols, string_facets=("lang",), timestamp_facets=("ts",), string_values={"lang": LANGS})
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    qk = bm25_queries(a.queries)
    b, keep = ix._lex_batch(qk, QueryType.Union)
    nq = len(qk)
    hits = _hits_array(nq * TOPK); nh = np.zeros(nq, dtype=np.uint32); cnt = np.zeros(nq, dtype=np.uint64)
    res = {"metric": "sorted_lexical_qps", "card": card, "power_limit": power,
           "config": {"docs": a.docs, "vocab": C3_VOCAB, "queries_per_step": nq, "query_law": "bench.bm25_queries (OR, 2-4 terms)", "k": TOPK,
                      "facets": "ts Timestamp rising with the doc id + jitter, price random U32, lang String16 of 40 values",
                      "steps": a.steps, "warmup": a.warmup, "index_build_s": round(build_s, 2)}}
    variants = [("unsorted_topk", None, ResultType.Topk), ("ts_desc_topk", [ResultSort("ts", SortOrder.Descending)], ResultType.Topk),
                ("ts_desc_topkcount", [ResultSort("ts", SortOrder.Descending)], ResultType.TopkCount),
                ("price_asc_topk", [ResultSort("price", SortOrder.Ascending)], ResultType.Topk),
                ("price_desc_lang_asc_topk", [ResultSort("price", SortOrder.Descending), ResultSort("lang", SortOrder.Ascending)], ResultType.Topk),
                ("id_desc_topk", [ResultSort("_id", SortOrder.Descending)], ResultType.Topk)]
    for name, sort, rt in variants:
        if sort is None:
            def step():
                check(lib().ssb_search_lexical(ix._h, C.byref(b), TOPK, int(rt), hits.ctypes.data, nh.ctypes.data, cnt.ctypes.data))
        else:
            crit, n_crit = ix._sort_criteria(sort)

            def step(crit=crit, n_crit=n_crit):
                check(lib().ssb_search_lexical_sorted(ix._h, C.byref(b), C.addressof(crit), n_crit, TOPK, int(rt), hits.ctypes.data, nh.ctypes.data,
                                                      cnt.ctypes.data))
        for _ in range(a.warmup):
            step()
        t = time.perf_counter()
        for _ in range(a.steps):
            step()
        s = time.perf_counter() - t
        sv = ix.last_stats()
        res[name] = {"queries_per_s": round(nq * a.steps / s, 1), "ms_per_step": round(s * 1e3 / a.steps, 3),
                     "scoring_kernel_ms": round(sv["dominant_kernel_ns"] / 1e6, 3), "items_processed": sv["items_processed"],
                     "items_skipped": sv["items_skipped"], "postings_visited": sv["postings_visited"],
                     "mean_hits": round(float(nh.mean()), 2)}
    ix.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
