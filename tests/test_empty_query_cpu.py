"""CPU: the empty query's restatement (helpers_empty) and the Python mirror's routing (Index.search("", enable_empty_query=True)).

- the literal shard route (docs in id order, delete set, is_facet_filter, add_topk with the empty query's comparator) against an independent
  numpy restatement (np.lexsort over typed ranks, ties to the larger doc id), filters of every type, deletes, sort criteria;
- the reference's test_05_empty_query on its 4-doc fixture (tests/golden/golden.json, ref_fixture_lexical);
- which route Index.search takes (search.rs:1413-1432 index route, search.rs:3374-3386 shard route), with a fake index;
- enable_empty_query=False keeps its behaviour."""
import numpy as np
import pytest

from helpers_empty import live_docs, numpy_route, shard_route, top_values, value_fn
from helpers_facets import facet_columns, numpy_pass, random_filters
from helpers_sort import FacetRows
from seekstorm_b200 import FacetFilter, Index, QueryFacet, ResultSort, ResultType, SortOrder, _lib

LEVELS = [(0, 300), (2, 250), (5, 77)]


def _world(seed):
    n_rows = (5 << 16) + 77
    cols, kw = facet_columns(n_rows, seed)
    strings = {"s16": [f"v{i:02d}" for i in range(12)][::-1], "s32": [f"w{(i * 7) % 300:03d}" for i in range(300)]}
    facets = FacetRows.pack(cols, 0, kw["string_facets"], kw["timestamp_facets"], strings)
    r = np.random.default_rng(seed)
    deleted = set(int(x) for x in r.choice(live_docs(LEVELS), 40, replace=False))
    return cols, facets, live_docs(LEVELS, deleted)


CRITERIA = [[], [("_id", True)], [("_id", False)], [("_score", False)], [("_score", True)], [("u8", False)], [("f32", True)],
            [("s16", True), ("i8", False)], [("s32", False), ("_score", False)], [("u16", True), ("_id", False)], [("ts", False)]]


@pytest.mark.parametrize("rt", [_lib.RESULT_COUNT, _lib.RESULT_TOPK, _lib.RESULT_TOPKCOUNT])
def test_literal_route_matches_numpy(rt):
    cols, facets, docs = _world(3)
    fls = random_filters(cols, 9, 24)
    value = value_fn(facets)
    for i, fl in enumerate(fls):
        crit = CRITERIA[i % len(CRITERIA)]
        mask = np.array([numpy_pass(cols, fl, d) for d in docs])
        got, cnt = shard_route(docs, lambda d: numpy_pass(cols, fl, d), 17, rt, crit, value)
        if rt == _lib.RESULT_COUNT:
            assert got == []
        else:
            assert got == numpy_route(docs, mask, 17, crit, lambda n, d: facets.rank(n)[d]), (i, crit)
        assert cnt == (0 if rt == _lib.RESULT_TOPK else int(mask.sum()))


def test_tie_rule_larger_doc_first():
    """every doc has the same value: the larger doc id ranks first, both sort directions"""
    docs = list(range(50))
    value = lambda name, d: 7                                                # noqa: E731
    for desc in (False, True):
        got, _ = shard_route(docs, lambda d: d % 3 == 0, 5, _lib.RESULT_TOPKCOUNT, [("c", desc)], value)
        assert got == [48, 45, 42, 39, 36]


def test_top_values():
    col = np.array([3, 1, 1, 2, 2, 3, 0, 5], dtype=np.uint16)
    assert top_values(col, 3) == [(1, 2), (2, 2), (3, 2)]
    assert top_values(col, 2, lambda i: i >= 2) == [(2, 2), (3, 2)]


class _Fake(Index):
    """an Index without a device: search_empty_batch / search_empty_facets answered by the restatement over `docs`"""

    def __init__(self, docs, facets=None, cols=None):
        self.docs, self.facets, self.cols, self.calls = docs, facets, cols, []
        self._facet_schema = {} if facets is None else {n: (i, t) for i, (n, (t, _)) in enumerate(facets.fields.items())}
        self._string_values = {} if facets is None else dict(facets.strings)
        self._string_order = {n: sorted(set(s.encode() for s in v)) for n, v in self._string_values.items()}

    def __del__(self):
        pass

    def search_empty_batch(self, n_queries, k, result_type=ResultType.TopkCount, filters=None, sort=None, sort_bases=None):
        self.calls.append(("batch", k, ResultType(result_type), filters, sort))
        crit = [(s.field, SortOrder(s.order) == SortOrder.Descending) for s in sort or []]
        fl = filters[0] if filters else []
        got, cnt = shard_route(self.docs, lambda d: numpy_pass(self.cols, fl, d) if fl else True, k, int(result_type), crit,
                               value_fn(self.facets) if self.facets else None)
        return [[(d, 0.0) for d in got]], np.array([cnt], dtype=np.uint64)

    def search_empty_facets(self, query_facets):
        self.calls.append(("facets", list(query_facets)))
        return {qf.field: top_values(self.cols[qf.field], qf.length) for qf in query_facets if qf.field in ("s16", "s32")}


def test_reference_fixture_test_05(golden):
    """test_05_empty_query (tests/test.rs:215-335) on the reference's 4-doc fixture: default and _id descending start at doc 3, _id
    ascending at doc 0; 4 results, result_count 4, result_count_total 4"""
    n = golden["ref_fixture_lexical"]["n_docs"]
    ix = _Fake(list(range(n)))
    for sort, first in ((None, 3), ([ResultSort("_id", SortOrder.Descending)], 3), ([ResultSort("_id", SortOrder.Ascending)], 0)):
        ro = ix.search("", enable_empty_query=True, result_sort=sort or ())
        assert ro.results[0].doc_id == first and len(ro.results) == 4
        assert ro.result_count == 4 and ro.result_count_total == 4
        assert all(r.score == 0.0 for r in ro.results)


def test_routes():
    cols, facets, docs = _world(5)
    ix = _Fake(docs, facets, cols)
    # index route: no filter, no query facets, at most one _id / _score criterion; total = the live docs for every result type
    for rt in ResultType:
        ix.calls.clear()
        ro = ix.search("", enable_empty_query=True, result_type=rt, offset=2, length=3)
        assert ro.result_count_total == len(docs)
        assert [r.doc_id for r in ro.results] == ([] if rt == ResultType.Count else docs[::-1][2:5])
        assert ix.calls[0][1:3] == (0, ResultType.Count)
    ro = ix.search("", enable_empty_query=True, result_sort=[ResultSort("_score", SortOrder.Ascending)])
    assert [r.doc_id for r in ro.results] == docs[:10]
    # shard route: a filter; Topk counts nothing, Count returns no hits
    fl = [FacetFilter("u8", 10, 100)]
    want = [d for d in docs if numpy_pass(cols, fl, d)]
    ro = ix.search("", enable_empty_query=True, facet_filter=fl, result_type=ResultType.Topk)
    assert [r.doc_id for r in ro.results] == want[::-1][:10] and ro.result_count_total == 0
    ro = ix.search("", enable_empty_query=True, facet_filter=fl, result_type=ResultType.TopkCount, offset=4, length=2)
    assert [r.doc_id for r in ro.results] == want[::-1][4:6] and ro.result_count_total == len(want) and ro.result_count == 2
    ix.calls.clear()
    ro = ix.search("", enable_empty_query=True, facet_filter=fl, result_type=ResultType.Count, result_sort=[ResultSort("u16")])
    assert ro.results == [] and ro.result_count_total == len(want)
    assert ix.calls[0][4] is None                                            # Count ignores the sort
    # shard route: two criteria; query facets (index-wide, every result type, ranges left out)
    ro = ix.search("", enable_empty_query=True, result_sort=[ResultSort("s16"), ResultSort("_id", SortOrder.Ascending)])
    assert [r.doc_id for r in ro.results] == numpy_route(docs, np.ones(len(docs), bool), 10, [("s16", True), ("_id", False)],
                                                          lambda n, d: facets.rank(n)[d])
    qfs = [QueryFacet("s16", length=2), QueryFacet("u8", ranges=[("a", 0), ("b", 50)])]
    for rt in ResultType:
        ro = ix.search("", enable_empty_query=True, result_type=rt, query_facets=qfs)
        top = top_values(cols["s16"], 2)
        assert ro.facets == {"s16": [(facets.strings["s16"][i], c) for i, c in top]}, rt
        assert ro.result_count_total == (0 if rt == ResultType.Topk else len(docs))
    assert ix.search("", enable_empty_query=True, result_type=ResultType.Topk, length=0, query_facets=qfs).facets == {}


def test_disabled_keeps_behaviour():
    ix = _Fake([0, 1, 2])
    ro = ix.search("")
    assert ro.results == [] and ro.result_count_total == 0 and ix.calls == []
    with pytest.raises(NotImplementedError):
        ix.search("", query_facets=[QueryFacet("s16", length=2)])
