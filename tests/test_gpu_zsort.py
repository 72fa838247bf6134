"""GPU: sorted lexical search (`result_sort`, search.rs:1004-1013; result_ordering_shard min_heap.rs:574-1051) through
ssb_search_lexical_sorted — OR / AND / phrase / 2-4-field BM25F, 1-9 terms, NOT terms, the delete set, a facet filter on one facet with a
sort on another, Topk / TopkCount / Count, k 1 / 10 / 32 / 100 (paging): ids, scores and counts == the oracle's exhaustive matches
ordered by helpers_sort.  Level skipping by the per-level facet bounds, the refusals, and the mirrored Search::search."""
import numpy as np
import pytest

from oracle import oracle as O
from seekstorm_b200 import synth
from helpers import gpu_index, oracle_index, query_keys, synth_levels
from helpers_facets import abi_filters, facet_columns
from helpers_mf import multifield_levels
from helpers_phrase import phrase_queries, sequence_corpus
from helpers_sort import FacetRows, all_matches, sort_criteria, sort_hits

pytestmark = pytest.mark.gpu
E_INVALID, E_STATE, E_UNSUPPORTED = -1, -4, -5          # SSB_E_*


def _strings(n_ids, seed):
    r = np.random.default_rng(seed)
    return ["".join(r.choice(list("abzAZ0é "), int(r.integers(0, 6)))) for _ in range(n_ids)]


def _facets(ix, orc, n, seed):
    cols, kinds = facet_columns(n, seed)
    strings = {"s16": _strings(12, seed + 1), "s32": _strings(300, seed + 2)}
    ix.set_facets(cols, string_values=strings, **kinds)
    rows, fields, first, nd, rb = ix._facet_rows
    orc.set_facets(rows, [(fields[i].type, fields[i].offset) for i in range(len(cols))], first, nd, rb)
    return FacetRows.of_index(ix, strings)


_ALL = {}      # the oracle's exhaustive match lists, shared by every sort of the same search


def _compare(ix, orc, n, qk, qt, oqt, criteria, facets, k, rt, ort, not_keys=None, filters=None, phrase=False, state=""):
    """one batch through the GPU, every query against the oracle; returns the list of mismatches.  state: names the index state (delete
    set, corpus) for the match-list cache"""
    got, cnt = ix.search_lexical_batch(qk, qt, k, rt, not_keys=not_keys, filters=filters, sort=sort_criteria(criteria))
    errs = []
    for i, q in enumerate(qk):
        kw = {}
        if not_keys and not_keys[i]:
            kw["not_keys"] = not_keys[i]
        if filters and filters[i]:
            kw["filters"], kw["set_values"] = abi_filters(ix, filters[i])
        key = (state, phrase, oqt, tuple(q), tuple(kw.get("not_keys", ())), repr(filters[i] if filters else None))
        if key not in _ALL:
            _ALL[key] = all_matches(orc, n, q, oqt, phrase, **kw)
        allh, tot = _ALL[key]
        want = [] if ort == O.RESULT_COUNT or k == 0 else sort_hits(allh, criteria, facets, k)
        if got[i] != want or (ort != O.RESULT_TOPK and int(cnt[i]) != tot):
            errs.append((criteria, int(qt), int(rt), k, i, got[i][:3], want[:3], int(cnt[i]), tot))
    return errs


CRITERIA = [
    [("ts", True)], [("f32", False)], [("f64", True)], [("u64", False)], [("i8", True), ("u16", False)],
    [("s16", True), ("u32", False)], [("s32", False)], [("i64", False)], [("u8", True), ("_score", False)],
    [("_id", True)], [("_id", False), ("f32", True)], [("_score", False)], [("i32", True), ("i16", False), ("u8", True)],
]


def test_sorted_parity_or_and():
    from seekstorm_b200 import FacetFilter, QueryType, ResultType
    n = 140000
    lvs, ls = synth_levels(n, 2000, 601)
    levels = [l.to_numpy() for l in lvs]
    orc = oracle_index(levels, n, ls)
    ix = gpu_index(levels, n, ls)
    fr = _facets(ix, orc, n, 602)
    qk = query_keys(synth.gen_queries(32, 603, 20, 1500, (1, 2, 3, 4, 6, 9), (0.15, 0.3, 0.2, 0.15, 0.1, 0.1)))
    rng = np.random.default_rng(604)
    nots = [[int(x) for x in rng.integers(0, 40, int(rng.integers(0, 2)))] for _ in qk]
    nk = [query_keys([ns])[0] if ns else [] for ns in nots]
    nk = [[t for t in ns if t not in q] for ns, q in zip(nk, qk)]
    shapes = [(10, ResultType.TopkCount, O.RESULT_TOPKCOUNT), (1, ResultType.Topk, O.RESULT_TOPK), (32, ResultType.TopkCount, O.RESULT_TOPKCOUNT),
              (100, ResultType.Topk, O.RESULT_TOPK), (0, ResultType.Count, O.RESULT_COUNT)]
    errs = []
    for ci, crit in enumerate(CRITERIA):
        k, rt, ort = shapes[ci % len(shapes)]
        for qt, oqt in ((QueryType.Union, O.QUERY_UNION), (QueryType.Intersection, O.QUERY_INTERSECTION)):
            errs += _compare(ix, orc, n, qk, qt, oqt, crit, fr, k, rt, ort, state="plain")
    # NOT terms + the delete set + a facet filter on one facet, sorted by another; every result type and paging
    deleted = [int(x) for x in rng.integers(0, n, 3000)]
    ix.set_deleted(deleted); orc.set_deleted(deleted)
    flt = [[FacetFilter("u8", 40, 220)] if i % 3 else [] for i in range(len(qk))]
    for crit in ([("f32", True)], [("s16", False), ("i32", True)], [("_id", False)]):
        for k, rt, ort in shapes:
            for qt, oqt in ((QueryType.Union, O.QUERY_UNION), (QueryType.Intersection, O.QUERY_INTERSECTION)):
                errs += _compare(ix, orc, n, qk, qt, oqt, crit, fr, k, rt, ort, not_keys=nk, filters=flt, state="deleted")
    assert not errs, (len(errs), errs[:4])
    ix.close()


def test_sorted_phrase_and_multifield():
    from seekstorm_b200 import Index, QueryType, ResultType
    n, vocab = 90000, 250
    docs, levels, ls = sequence_corpus(n, vocab, 611)
    orc = oracle_index(levels, n, ls)
    ix = Index(0)
    for lv in levels:
        ix.add_lexical_level(lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"], lv["doc_len_bytes"],
                             lv["positions"])
    ix.commit(n, ls)
    fr = _facets(ix, orc, n, 612)
    qk = query_keys(phrase_queries(docs, 613, 60, vocab))
    errs = []
    for crit, (k, rt, ort) in (([("u32", True)], (10, ResultType.TopkCount, O.RESULT_TOPKCOUNT)), ([("s32", False)], (32, ResultType.Topk, O.RESULT_TOPK)),
                               ([("_id", True)], (100, ResultType.TopkCount, O.RESULT_TOPKCOUNT))):
        errs += _compare(ix, orc, n, qk, QueryType.Phrase, None, crit, fr, k, rt, ort, phrase=True, state="phrase")
    assert not errs, (len(errs), errs[:4])
    ix.close()
    for n_fields, boosts in ((2, (2.0, 1.0)), (3, (3.0, 1.0, 0.5)), (4, (1.0, 1.0, 1.0, 1.0))):
        n = 70000
        levels, ls = multifield_levels(n, 300, n_fields, seed=620 + n_fields)
        ix = Index(0); ix.set_field_boosts(boosts)
        orc = O.OracleIndex(); orc.set_fields(boosts)
        for lv in levels:
            ix.add_lexical_level(lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"], lv["doc_len_bytes"])
            orc.add_level(lv)
        ix.commit(n, ls); orc.commit(n, ls)
        fr = _facets(ix, orc, n, 630 + n_fields)
        rng = np.random.default_rng(640 + n_fields)
        qk = [[int(x) for x in synth.term_keys_np(rng.choice(np.arange(2, 300), size=nt, replace=False).astype(np.int64))] for nt in (1, 2, 3, 5, 9) * 3]
        for qt, oqt in ((QueryType.Union, O.QUERY_UNION), (QueryType.Intersection, O.QUERY_INTERSECTION)):
            errs += _compare(ix, orc, n, qk, qt, oqt, [("f32", False), ("u16", True)], fr, 10, ResultType.TopkCount, O.RESULT_TOPKCOUNT, state=f"mf{n_fields}")
            errs += _compare(ix, orc, n, qk, qt, oqt, [("_score", False)], fr, 32, ResultType.Topk, O.RESULT_TOPK, state=f"mf{n_fields}")
        ix.close()
    assert not errs, (len(errs), errs[:4])


def test_level_skipping_by_facet_bounds():
    from seekstorm_b200 import QueryType, ResultType
    n = 200000
    lvs, ls = synth_levels(n, 3000, 651)
    levels = [l.to_numpy() for l in lvs]
    orc = oracle_index(levels, n, ls)
    ix = gpu_index(levels, n, ls)
    rng = np.random.default_rng(652)
    ts = (1_600_000_000 + np.arange(n, dtype=np.int64) * 10 + rng.integers(0, 50, n)).astype(np.int64)   # rises with the doc id
    shuffled = rng.permutation(ts)
    cols = {"ts": ts, "sh": shuffled}
    ix.set_facets(cols, timestamp_facets=("ts", "sh"))
    rows, fields, first, nd, rb = ix._facet_rows
    orc.set_facets(rows, [(fields[i].type, fields[i].offset) for i in range(2)], first, nd, rb)
    fr = FacetRows.of_index(ix)
    qk = query_keys(synth.gen_queries(24, 653, 30, 600, (1, 2, 3), (0.4, 0.4, 0.2)))
    errs = []
    for name in ("ts", "sh"):
        for qt, oqt in ((QueryType.Union, O.QUERY_UNION), (QueryType.Intersection, O.QUERY_INTERSECTION)):
            errs += _compare(ix, orc, n, qk, qt, oqt, [(name, True)], fr, 10, ResultType.Topk, O.RESULT_TOPK, state="skip")
            st = ix.last_stats()
            if name == "ts" and qt == QueryType.Union:
                assert st["items_skipped"] > 0, st
    errs += _compare(ix, orc, n, qk, QueryType.Union, O.QUERY_UNION, [("ts", True)], fr, 10, ResultType.TopkCount, O.RESULT_TOPKCOUNT, state="skip")
    errs += _compare(ix, orc, n, qk, QueryType.Union, O.QUERY_UNION, [("_id", True)], fr, 10, ResultType.Topk, O.RESULT_TOPK, state="skip")
    assert not errs, (len(errs), errs[:4])
    ix.close()


def test_sorted_refusals():
    import ctypes as C
    from seekstorm_b200 import QueryType, ResultType, SsbError, _lib
    from seekstorm_b200._lib import SsbSortCriterion, lib
    from seekstorm_b200.index import _hits_array
    n = 140000
    lvs, ls = synth_levels(n, 800, 661)
    levels = [l.to_numpy() for l in lvs]
    ix = gpu_index(levels, n, ls)
    qk = query_keys([[5, 60], [7]])
    b, keep = ix._lex_batch(qk, QueryType.Union)
    hits = _hits_array(2 * 10); nh = np.zeros(2, dtype=np.uint32); cnt = np.zeros(2, dtype=np.uint64)

    def call(crits, rt=ResultType.TopkCount, k=10):
        arr = (SsbSortCriterion * max(len(crits), 1))(*[SsbSortCriterion(*c, 0) for c in crits])
        return lib().ssb_search_lexical_sorted(ix._h, C.byref(b), C.addressof(arr), len(crits), k, int(rt), hits.ctypes.data, nh.ctypes.data, cnt.ctypes.data)

    F, I, S, A, D = _lib.SORT_FACET, _lib.SORT_ID, _lib.SORT_SCORE, _lib.SORT_ASCENDING, _lib.SORT_DESCENDING
    assert call([(F, 0, D)]) == E_STATE                       # no facets
    assert call([(I, 0, D)]) == 0 and call([(S, 0, A)]) == 0 and call([]) == 0
    cols = {"a": np.arange(n, dtype=np.uint64), "b": np.arange(n, dtype=np.int64), "c": np.arange(n, dtype=np.float32), "s": np.zeros(n, dtype=np.uint16)}
    ix.set_facets(cols, string_facets=("s",))
    assert call([(F, 4, D)]) == E_INVALID                    # facet out of range
    assert call([(3, 0, D)]) == E_INVALID and call([(F, 0, 2)]) == E_INVALID   # bad source / order
    assert call([(F, 0, D), (F, 1, A)]) == E_UNSUPPORTED     # 128 bits
    assert call([(F, 2, D), (F, 1, A)]) == E_UNSUPPORTED     # 96 bits
    assert call([(F, 2, D), (I, 0, A)]) == 0                          # 64 bits
    assert call([(F, 0, D), (S, 0, A), (F, 1, A)]) == 0               # criteria after _score are not compared
    assert call([(F, 3, D)]) == E_STATE                      # String facet without a value order
    rank = np.zeros(1, dtype=np.uint32)
    assert lib().ssb_set_facet_value_order(ix._h, 0, rank.ctypes.data, 1) == E_INVALID   # not a String facet
    assert lib().ssb_set_facet_value_order(ix._h, 3, np.array([1], dtype=np.uint32).ctypes.data, 1) == E_INVALID   # rank >= n_ids
    assert lib().ssb_set_facet_value_order(ix._h, 3, rank.ctypes.data, 1) == 0 and call([(F, 3, D)]) == 0
    ix.set_facets({"s": np.full(n, 2, dtype=np.uint16)}, string_facets=("s",), string_values={"s": ["x", "y"]})
    assert call([(F, 0, D)]) == E_STATE                      # an id >= n_ids
    ix.set_facets({"a": np.arange(70000, dtype=np.uint64)})
    assert call([(F, 0, D)]) == E_STATE                      # rows do not cover every level
    assert call([(F, 0, D)], ResultType.Count, 0) == 0                # Count ignores the sort
    with pytest.raises(SsbError):
        ix.search_lexical_batch(qk, QueryType.Union, 10, sort=sort_criteria([("a", True)]))
    ix.close()


def test_search_mirror_result_sort():
    from seekstorm_b200 import Index, QueryType, ResultSort, ResultType, SearchMode, SortOrder
    n = 100000
    lvs, ls = synth_levels(n, 1500, 671)
    levels = [l.to_numpy() for l in lvs]
    orc = oracle_index(levels, n, ls)
    ix = gpu_index(levels, n, ls, vector_dims=8)
    rng = np.random.default_rng(672)
    langs = ["en", "de", "fr", "zh", "pt-BR", "pt"] + [f"l{i}" for i in range(34)]
    cols = {"price": rng.integers(0, 50, n, dtype=np.uint32).astype(np.float32), "lang": rng.integers(0, len(langs), n, dtype=np.uint16)}
    ix.set_facets(cols, string_facets=("lang",), string_values={"lang": langs})
    rs = [ResultSort("price", SortOrder.Descending), ResultSort("lang", SortOrder.Ascending), ResultSort("nope", SortOrder.Ascending)]
    ro = ix.search("t40 t300 t7", None, QueryType.Union, SearchMode.Lexical(), False, 5, 20, ResultType.TopkCount, result_sort=rs)
    k = query_keys([[40, 300, 7]])[0]
    allh, tot = all_matches(orc, n, k, O.QUERY_UNION)
    want = sort_hits(allh, [("price", True), ("lang", False)], FacetRows.of_index(ix, {"lang": langs}), 25)[5:]
    assert [(r.doc_id, np.float32(r.score)) for r in ro.results] == [(d, np.float32(s)) for d, s in want] and ro.result_count_total == tot
    with pytest.raises(NotImplementedError):
        ix.search("t40", None, result_sort=[ResultSort("price", SortOrder.Descending, base=(52.5, 13.4))])
    with pytest.raises(NotImplementedError):
        ix.search("t40", np.ones(8, dtype=np.float32), search_mode=SearchMode.Vector(), result_sort=[ResultSort("price")])
    with pytest.raises(NotImplementedError):
        ix.search("t40", np.ones(8, dtype=np.float32), search_mode=SearchMode.Hybrid(), result_sort=[ResultSort("price")])
    ix.close()
