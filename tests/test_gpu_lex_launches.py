"""GPU: the kernel launches of each lexical call kind (last_stats()["kernel_launches"]), with and without a delete set, on a small
synthetic corpus.  Unsorted: lex_plan, lex_score (unless Count), lex_count (unless Topk), lex_generic, lex_not_count (unless Topk),
lex_del_count (with a delete set, unless Topk), copy_out.  Sorted: lex_plan, lex_generic, then the same count corrections (a sorted Count
search is an unsorted one).  Facet counts: lex_plan, then lex_facets + facet_select per query chunk.  Every call also reports a kernel
time."""
import numpy as np
import pytest

from helpers import gpu_index, query_keys, synth_levels
from seekstorm_b200 import QueryFacet, QueryType, ResultSort, ResultType, SortOrder

pytestmark = pytest.mark.gpu

N = 20000
UNSORTED = {ResultType.Topk: (4, 4), ResultType.TopkCount: (6, 7), ResultType.Count: (5, 6)}   # (no delete set, delete set)
SORTED = {ResultType.Topk: (2, 2), ResultType.TopkCount: (3, 4), ResultType.Count: UNSORTED[ResultType.Count]}   # Count: no sort


@pytest.fixture(scope="module")
def ix():
    lvs, ls = synth_levels(N, 2000, 21)
    ix = gpu_index([l.to_numpy() for l in lvs], N, ls)
    rng = np.random.default_rng(22)
    big = rng.integers(0, 1 << 24, N, dtype=np.uint32)
    big[0] = (1 << 24) - 1                     # 2^24 value ids: a query's histogram takes 64 MiB, so 4 queries fill one chunk
    ix.set_facets({"price": rng.integers(0, 1000, N, dtype=np.uint32), "big": big}, string_facets=("big",))
    yield ix
    ix.close()


QUERIES = query_keys([[3, 17], [5, 40, 41], [8], [2, 9, 30, 31, 32, 33], [12, 13], [7, 60, 61, 62]])


def _launches(ix):
    s = ix.last_stats()
    assert s["dominant_kernel_ns"] > 0, s
    return s["kernel_launches"]


@pytest.mark.parametrize("deleted", [False, True])
@pytest.mark.parametrize("qt", [QueryType.Union, QueryType.Intersection])
def test_search_launches(ix, qt, deleted):
    ix.set_deleted(range(0, N, 7) if deleted else [])
    try:
        for rt, want in UNSORTED.items():
            ix.search_lexical_batch(QUERIES, qt, 10, rt)
            assert _launches(ix) == want[deleted], (rt, "unsorted")
        for rt, want in SORTED.items():
            ix.search_lexical_batch(QUERIES, qt, 10, rt, sort=[ResultSort("price", SortOrder.Ascending)])
            assert _launches(ix) == want[deleted], (rt, "sorted")
    finally:
        ix.set_deleted([])


def test_facet_count_launches(ix):
    ix.search_lexical_facets(QUERIES, QueryType.Union, [QueryFacet("price", ranges=[("lo", 0), ("hi", 500)])])
    assert _launches(ix) == 1 + 2
    ix.search_lexical_facets(QUERIES, QueryType.Union, [QueryFacet("big", length=3)])      # 6 queries: chunks of 4 and 2
    assert _launches(ix) == 1 + 2 * 2
