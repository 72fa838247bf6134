"""GPU: geo search on Point facets — FacetFilter::Point (distance ranges, FilterSparse::Point add_result.rs:462-478) on every scoring path
and sorting by the distance to a per-query base (morton_ordering, min_heap.rs:510-529).  Ids, scores and counts == the oracle: the C
oracle with the docs a Point filter rejects handed over as deleted docs, the distances restated with math.cos (helpers_geo).  Bounds and
corpora keep every distance more than a relative 1e-12 away from a bound and from its neighbours in sort order (the precision contract:
CUDA's double cos is not bit-equal to the C library's), which the helpers assert."""
import math

import numpy as np
import pytest

from oracle import oracle as O
from seekstorm_b200 import synth
from helpers import gpu_index, oracle_index, query_keys, synth_levels
from helpers_geo import filter_rejects, sort_by_distance, sort_distances
from helpers_phrase import phrase_queries, sequence_corpus
from helpers_phrase_mf import PhraseFieldsOracle, multifield_sequence_corpus, phrase_queries_mf
from helpers_sort import all_matches

pytestmark = pytest.mark.gpu

CITIES = [(52.52, 13.405), (40.7128, -74.006), (-33.8688, 151.2093), (-34.6037, -58.3816), (1.29, 36.82), (51.5072, -0.1276)]


def _points(n, seed):
    """clusters around cities on both sides of 0 deg lat / lon, a cluster near the north pole, docs without a point (NaN: stored as 0)
    and a few exact duplicates"""
    r = np.random.default_rng(seed)
    pts = np.zeros((n, 2))
    centres = CITIES + [(89.95, 20.0)]
    c = r.integers(0, len(centres), n)
    for i, (la, lo) in enumerate(centres):
        m = c == i
        pts[m, 0] = np.clip(la + r.normal(0, 0.6, m.sum()), -90, 90)
        pts[m, 1] = lo + r.normal(0, 0.9, m.sum())
    pts[r.integers(0, n, n // 50)] = np.nan
    dup = r.integers(0, n, 200)
    pts[dup] = pts[r.integers(0, n, 200)]
    return pts


def _setup(n, vocab, seed, **kw):
    lvs, ls = synth_levels(n, vocab, seed)
    levels = [l.to_numpy() for l in lvs]
    orc = oracle_index(levels, n, ls)
    ix = gpu_index(levels, n, ls, **kw)
    rng = np.random.default_rng(seed + 1)
    cols = {"loc": _points(n, seed + 2), "price": rng.integers(0, 1000, n, dtype=np.uint32)}
    ix.set_facets(cols, point_facets=("loc",))
    rows, fields, first, nd, rb = ix._facet_rows
    orc.set_facets(rows, [(fields[i].type, fields[i].offset) for i in range(len(cols))], first, nd, rb)
    codes = rows[:nd, fields[0].offset:fields[0].offset + 8].copy().view(np.uint64).reshape(-1)
    return ix, orc, codes


def _geo_filters(seed, nq):
    """per query a Point filter (km / miles, discs and annuli, end = inf, NaN base / bounds) and sometimes a price range"""
    from seekstorm_b200 import DistanceUnit, FacetFilter
    r = np.random.default_rng(seed)
    out = []
    for i in range(nq):
        la, lo = CITIES[i % len(CITIES)]
        base = (la + float(r.normal(0, 0.3)), lo + float(r.normal(0, 0.3)))
        unit = DistanceUnit.Miles if i % 3 == 1 else DistanceUnit.Kilometers
        end = float(r.choice([20.0, 45.0, 80.0, 150.0]))
        start = 0.0 if i % 4 else end / 3.0
        if i % 11 == 5:
            end = math.inf
        if i % 13 == 7:
            base = (math.nan, base[1])
        if i % 17 == 3:
            start = math.nan
        fl = [FacetFilter("loc", start, end, base=base, unit=unit)]
        if i % 5 == 2:
            fl.append(FacetFilter("price", 100, 700))
        out.append(fl)
    return out


def _oracle_args(ix, codes, fl):
    """(filters, set values, docs rejected by the Point filters) for the oracle"""
    rest = [f for f in fl if f.base is None]
    rej = set()
    for f in fl:
        if f.base is not None:
            rej.update(int(d) for d in filter_rejects(codes, tuple(f.base), float(f.start), float(f.end), int(f.unit)))
    if not rest:
        return None, None, rej
    offs, arr, sv = ix._encode_filters([rest])
    return [(arr[i].facet, arr[i].kind, arr[i].start, arr[i].end, arr[i].set_first, arr[i].set_count) for i in range(int(offs[1]))], \
        [int(x) for x in sv], rej


def test_geo_filter_parity():
    from seekstorm_b200 import QueryType, ResultType
    n = 150000
    ix, orc, codes = _setup(n, 2500, 91)
    qs = synth.gen_queries(40, 93, 2, 2000, (1, 2, 3, 4, 6), (0.15, 0.3, 0.25, 0.15, 0.15))
    qk = query_keys(qs)
    filters = _geo_filters(94, len(qk))
    rng = np.random.default_rng(95)
    nots = [[int(x) for x in rng.integers(0, 50, int(rng.integers(0, 2)))] for _ in qs]
    nots = [[t for t in ns if t not in q] for ns, q in zip(nots, qs)]
    nk = [query_keys([ns])[0] if ns else [] for ns in nots]
    args = [_oracle_args(ix, codes, fl) for fl in filters]
    errs, passed = [], 0
    for deleted in ([], [int(x) for x in rng.integers(0, n, 3000)]):
        ix.set_deleted(deleted)
        for qt, oqt in ((QueryType.Union, O.QUERY_UNION), (QueryType.Intersection, O.QUERY_INTERSECTION)):
            got, cnt = ix.search_lexical_batch(qk, qt, 10, ResultType.TopkCount, not_keys=nk, filters=filters)
            got_t, _ = ix.search_lexical_batch(qk, qt, 10, ResultType.Topk, not_keys=nk, filters=filters)
            _, cnt_c = ix.search_lexical_batch(qk, qt, 0, ResultType.Count, not_keys=nk, filters=filters)
            for i, k in enumerate(qk):
                tup, sv, rej = args[i]
                orc.set_deleted(sorted(set(deleted) | rej))
                kw = dict(filters=tup, set_values=sv) if tup else {}
                want, tot = orc.search(k, oqt, 10, O.RESULT_TOPKCOUNT, not_keys=nk[i], **kw)
                passed += tot > 0
                if got[i] != want or got_t[i] != want or int(cnt[i]) != tot or int(cnt_c[i]) != tot:
                    errs.append((bool(deleted), int(qt), i, filters[i], got[i][:3], want[:3], int(cnt[i]), int(cnt_c[i]), tot))
    assert not errs, (len(errs), errs[:4])
    assert passed > 40                                              # the filters keep hits for many queries
    # paging beyond 32 hits (k = 100)
    ix.set_deleted([])
    got, cnt = ix.search_lexical_batch(qk, QueryType.Union, 100, ResultType.TopkCount, filters=filters)
    for i, k in enumerate(qk):
        tup, sv, rej = args[i]
        orc.set_deleted(sorted(rej))
        kw = dict(filters=tup, set_values=sv) if tup else {}
        want, tot = orc.search(k, O.QUERY_UNION, 100, O.RESULT_TOPKCOUNT, **kw)
        assert got[i] == want and int(cnt[i]) == tot, (i, filters[i])
    ix.close()


def test_geo_sort_parity_and_refusals():
    from seekstorm_b200 import FacetFilter, QueryType, ResultSort, ResultType, SortOrder, SsbError
    n = 150000
    ix, orc, codes = _setup(n, 2500, 101)
    qk = query_keys(synth.gen_queries(24, 103, 2, 2000, (1, 2, 3), (0.3, 0.4, 0.3)))
    rng = np.random.default_rng(104)
    bases = [(CITIES[i % len(CITIES)][0] + float(rng.normal(0, 1)), CITIES[i % len(CITIES)][1] + float(rng.normal(0, 1))) for i in range(len(qk))]
    matches = [all_matches(orc, n, k, O.QUERY_UNION) for k in qk]
    hits = [[(int(d), float(s)) for d, s in zip(m["doc_id"], m["score"])] for m, _ in matches]
    dists = [sort_distances([d for d, _ in h], codes, 0, b) for h, b in zip(hits, bases)]
    errs = []
    for desc in (False, True):
        for score_asc in (None, True):
            sort = [ResultSort("loc", SortOrder.Descending if desc else SortOrder.Ascending)]
            if score_asc is not None:
                sort.append(ResultSort("_score", SortOrder.Ascending))
            for rt in (ResultType.TopkCount, ResultType.Topk):
                for k in (10, 100):
                    got, cnt = ix.search_lexical_batch(qk, QueryType.Union, k, rt, sort=sort, sort_bases=bases)
                    for i in range(len(qk)):
                        tot = matches[i][1]
                        want = sort_by_distance(hits[i], dists[i], desc, bool(score_asc), k)
                        if got[i] != want or (rt == ResultType.TopkCount and int(cnt[i]) != tot):
                            errs.append((desc, score_asc, int(rt), k, i, got[i][:3], want[:3]))
    assert not errs, (len(errs), errs[:4])
    # the base of ResultSort, no base (the criterion is dropped: score order), and a base on a non-Point facet
    near = [ResultSort("loc", SortOrder.Ascending, base=bases[0])]
    got, _ = ix.search_lexical_batch(qk[:1], QueryType.Union, 10, ResultType.Topk, sort=near)
    assert got[0] == sort_by_distance(hits[0], dists[0], False, False, 10)
    plain, _ = ix.search_lexical_batch(qk, QueryType.Union, 10, ResultType.TopkCount)
    dropped, _ = ix.search_lexical_batch(qk, QueryType.Union, 10, ResultType.TopkCount, sort=[ResultSort("loc", SortOrder.Ascending)])
    assert dropped == plain
    with pytest.raises(NotImplementedError):
        ix.search_lexical_batch(qk, QueryType.Union, 10, ResultType.Topk, sort=[ResultSort("price", SortOrder.Ascending, base=(1.0, 2.0))])
    # a Point criterion takes 64 bits: only _score may follow it
    with pytest.raises(SsbError):
        ix.search_lexical_batch(qk, QueryType.Union, 10, ResultType.Topk, sort=[ResultSort("loc"), ResultSort("price")], sort_bases=bases)
    # a Point filter on a non-Point facet, a range filter on a Point facet, a bad unit
    with pytest.raises(SsbError):
        ix.search_lexical_batch(qk[:1], QueryType.Union, 10, ResultType.Topk, filters=[[FacetFilter("price", 0.0, 10.0, base=(1.0, 2.0))]])
    with pytest.raises(SsbError):
        ix.search_lexical_batch(qk[:1], QueryType.Union, 10, ResultType.Topk, filters=[[FacetFilter("loc", 0, 10)]])
    with pytest.raises(ValueError):
        ix.search_lexical_batch(qk[:1], QueryType.Union, 10, ResultType.Topk, filters=[[FacetFilter("loc", 0.0, 10.0, base=(1.0, 2.0), unit=7)]])
    ix.close()


def test_geo_index_search_mirror():
    from seekstorm_b200 import DistanceUnit, FacetFilter, QueryType, ResultSort, ResultType, SearchMode, SortOrder
    n = 100000
    ix, orc, codes = _setup(n, 1500, 111)
    base = (52.6, 13.3)
    ff = [FacetFilter("loc", 0.0, 60.0, base=base, unit=DistanceUnit.Kilometers)]
    rs = [ResultSort("loc", SortOrder.Ascending, base=base)]
    ro = ix.search("t40 t300 t7", None, QueryType.Union, SearchMode.Lexical(), False, 0, 20, ResultType.TopkCount, facet_filter=ff, result_sort=rs)
    k = query_keys([[40, 300, 7]])[0]
    rej = set(int(d) for d in filter_rejects(codes, base, 0.0, 60.0, 0))
    orc.set_deleted(sorted(rej))
    allh, tot = all_matches(orc, n, k, O.QUERY_UNION)
    h = [(int(d), float(s)) for d, s in zip(allh["doc_id"], allh["score"])]
    want = sort_by_distance(h, sort_distances([d for d, _ in h], codes, 0, base), False, False, 20)
    assert tot > 20 and [(r.doc_id, np.float32(r.score)) for r in ro.results] == [(d, np.float32(s)) for d, s in want]
    assert ro.result_count_total == tot
    ix.close()


def _phrase_index(levels, n, ls, boosts=None):
    from seekstorm_b200 import Index
    ix = Index(0)
    if boosts:
        ix.set_field_boosts(boosts)
    for lv in levels:
        ix.add_lexical_level(lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"], lv["doc_len_bytes"],
                             lv["positions"])
    ix.commit(n, ls)
    return ix


def _geo_facets(ix, orc, n, seed):
    """a Point facet on an index built from levels; the facet rows go to the oracle too (when it takes them) -> the column's codes"""
    ix.set_facets({"loc": _points(n, seed)}, point_facets=("loc",))
    rows, fields, first, nd, rb = ix._facet_rows
    if hasattr(orc, "set_facets"):
        orc.set_facets(rows, [(fields[0].type, fields[0].offset)], first, nd, rb)
    return rows[:nd, 0:8].copy().view(np.uint64).reshape(-1)


def test_geo_filter_phrase_batches():
    """Point filters on a phrase batch: single field (lex_generic<false, *, true>) and two indexed fields with per-field position runs
    (lex_generic<true, *, true>), against the oracles' phrase search with the rejected docs deleted"""
    from seekstorm_b200 import QueryType, ResultType
    n, vocab = 60000, 250
    docs, levels, ls = sequence_corpus(n, vocab, 31)
    orc = oracle_index(levels, n, ls)
    ix = _phrase_index(levels, n, ls)
    codes = _geo_facets(ix, orc, n, 32)
    qk = query_keys(phrase_queries(docs, 33, 48, vocab))
    filters = [[f for f in fl if f.base is not None] for fl in _geo_filters(34, len(qk))]
    rej = [_oracle_args(ix, codes, fl)[2] for fl in filters]
    got, cnt = ix.search_lexical_batch(qk, QueryType.Phrase, 10, ResultType.TopkCount, filters=filters)
    got_t, _ = ix.search_lexical_batch(qk, QueryType.Phrase, 10, ResultType.Topk, filters=filters)
    _, cnt_c = ix.search_lexical_batch(qk, QueryType.Phrase, 0, ResultType.Count, filters=filters)
    errs, n_hit = [], 0
    for i, k in enumerate(qk):
        orc.set_deleted(sorted(rej[i]))
        want, tot = orc.search_phrase(k, 10, O.RESULT_TOPKCOUNT)
        n_hit += tot > 0
        if got[i] != want or got_t[i] != want or int(cnt[i]) != tot or int(cnt_c[i]) != tot:
            errs.append((i, got[i][:3], want[:3], int(cnt[i]), int(cnt_c[i]), tot))
    assert not errs and n_hit > 5, (len(errs), errs[:4], n_hit)
    ix.close()
    # two indexed fields
    n2 = 72000
    docs, levels, ls = multifield_sequence_corpus(n2, 200, 2, seed=35)
    boosts = (2.0, 1.0)
    ix = _phrase_index(levels, n2, ls, boosts)
    orc2 = PhraseFieldsOracle(levels, n2, ls, boosts)
    codes = _geo_facets(ix, orc2, n2, 36)
    qk = query_keys(phrase_queries_mf(docs, 37, 40, 200))
    filters = [[f for f in fl if f.base is not None] for fl in _geo_filters(38, len(qk))]
    rej = [_oracle_args(ix, codes, fl)[2] for fl in filters]
    got, cnt = ix.search_lexical_batch(qk, QueryType.Phrase, 10, ResultType.TopkCount, filters=filters)
    got_t, _ = ix.search_lexical_batch(qk, QueryType.Phrase, 10, ResultType.Topk, filters=filters)
    errs, n_hit = [], 0
    for i, k in enumerate(qk):
        orc2.set_deleted(sorted(rej[i]))
        want, tot = orc2.search_phrase(k, 10, O.RESULT_TOPKCOUNT)
        n_hit += tot > 0
        if got[i] != want or got_t[i] != want or int(cnt[i]) != tot:
            errs.append((i, got[i][:3], want[:3], int(cnt[i]), tot))
    assert not errs and n_hit > 5, (len(errs), errs[:4], n_hit)
    ix.close()


def test_geo_filter_hybrid_and_abi_refusals():
    import ctypes as C
    import torch
    from seekstorm_b200 import QueryType, ResultType, VectorSimilarity, _lib
    from seekstorm_b200._lib import check, lib
    from seekstorm_b200.index import _hits_array
    n, dims = 100000, 32
    ix, orc, codes = _setup(n, 1500, 121, vector_dims=dims, vector_similarity=VectorSimilarity.Cosine)
    rows = synth.gen_vectors(n, dims, 123, "cpu").numpy()
    ix.add_vectors(rows)
    qk = query_keys(synth.gen_queries(12, 124, 2, 1000, (2, 3), (0.5, 0.5)))
    filters = _geo_filters(125, len(qk))
    args = [_oracle_args(ix, codes, fl) for fl in filters]
    # hybrid: the Point filter applies to the lexical half (search_vector_shard takes no facet filter, vector.rs:1105-1115)
    qv = synth.gen_vectors(len(qk), dims, 126, "cpu").numpy()
    nq = len(qk)
    b, keep = ix._lex_batch(qk, QueryType.Union, None, filters)
    hits = _hits_array(nq * 10); nh = np.zeros(nq, dtype=np.uint32)
    check(lib().ssb_search_hybrid(ix._h, C.byref(b), qv.ctypes.data, 10, hits.ctypes.data, nh.ctypes.data))
    nrows = np.stack([O.normalize(r) for r in rows])
    for i in range(nq):
        tup, sv, rej = args[i]
        orc.set_deleted(sorted(rej))
        kw = dict(filters=tup, set_values=sv) if tup else {}
        lex, _ = orc.search(qk[i], O.QUERY_UNION, 10, O.RESULT_TOPK, **kw)
        vec = O.search_vector(nrows, O.normalize(qv[i]), 10, O.SIM_COSINE)
        h = hits[i * 10: i * 10 + int(nh[i])]
        assert [int(d) for d in h["doc_id"]] == [d for d, _ in O.rrf(lex, vec)[:10]], i
    # the library's own refusals, past the Python mirror: set_count != 3, a bad unit, a device filter_set_values array
    hits = _hits_array(10); nh = np.zeros(1, dtype=np.uint32); cnt = np.zeros(1, dtype=np.uint64)
    geo = [[f for f in filters[0] if f.base is not None]]

    def call(b):
        return lib().ssb_search_lexical(ix._h, C.byref(b), 10, int(ResultType.TopkCount), hits.ctypes.data, nh.ctypes.data, cnt.ctypes.data)
    b, keep = ix._lex_batch(qk[:1], QueryType.Union, None, geo)
    assert call(b) == 0
    farr, fsets = keep[4], keep[5]
    farr[0].set_count = 2
    assert call(b) == -1 and b"3 filter_set_values" in lib().ssb_last_error()
    farr[0].set_count = 3
    fsets[2] = 7
    assert call(b) == -1 and b"unit" in lib().ssb_last_error()
    fsets[2] = _lib.UNIT_MILES
    assert call(b) == 0
    dev = torch.from_numpy(fsets.astype(np.int64)).cuda()
    b.filter_set_values = dev.data_ptr()
    assert call(b) == -1 and b"host arrays" in lib().ssb_last_error()
    ix.close()
