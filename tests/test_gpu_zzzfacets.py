"""GPU: facet counts of lexical batches (ssb_search_lexical_facets, Index.search(query_facets=...)).  The expected counts are histograms
over the oracle's exhaustive match lists (helpers_sort.all_matches) of the typed numpy columns — np.searchsorted(starts, v, 'right') - 1,
a value below the first start or NaN not counted; Point distances restated with math.cos (helpers_geo) and kept more than a relative
1e-12 away from every start — and, for String facets, the top `length` ids by (count desc, id asc) inside the prefix's rank interval."""
import math

import numpy as np
import pytest

from helpers import gpu_index, oracle_index, query_keys, synth_levels
from helpers_facets import facet_columns, numpy_pass, random_filters
from helpers_geo import decode, euclidian_distance, filter_rejects
from helpers_phrase import phrase_queries, sequence_corpus
from helpers_phrase_mf import PhraseFieldsOracle, multifield_sequence_corpus, phrase_queries_mf
from helpers_sort import all_matches
from seekstorm_b200 import DistanceUnit, FacetFilter, Index, QueryFacet, QueryType, RangeType, ResultType
import seekstorm_b200.index as I

pytestmark = pytest.mark.gpu

S16 = ["apple", "app", "apricot", "b", "banana", "app", "", "ap", "éclair", "apple", "zz", "ab"]
BASES = [(52.52, 13.405), (-33.8688, 151.2093)]
PT_STARTS = [0.0, 60.0, 300.0, 2000.0, 9000.0]


def _points(n, seed):
    r = np.random.default_rng(seed)
    c = r.integers(0, len(BASES), n)
    pts = np.array([BASES[i] for i in c], dtype=np.float64) + r.normal(0, 2.0, (n, 2))
    pts[r.integers(0, n, n // 50)] = np.nan
    return pts


def _starts(col, k, rng):
    """k ascending starts inside the column's range, the type's minimum first (the bins then cover every non-NaN value)"""
    c = np.asarray(col)
    if c.dtype.kind == "f":
        q = np.unique(np.quantile(c[np.isfinite(c)], np.sort(rng.uniform(0.05, 0.95, k - 1))).astype(c.dtype))
        return [-math.inf] + [float(x) for x in q]
    info = np.iinfo(c.dtype)
    q = np.unique(np.quantile(c.astype(np.float64), np.sort(rng.uniform(0.05, 0.95, k - 1))).astype(c.dtype))
    return [int(info.min)] + [int(x) for x in q if int(x) > info.min]


class Corpus:
    def __init__(self, n=70000, vocab=2000, seed=11):
        lvs, ls = synth_levels(n, vocab, seed)
        self.levels = [l.to_numpy() for l in lvs]
        self.n, self.orc = n, oracle_index(self.levels, n, ls)
        self.ix = gpu_index(self.levels, n, ls)
        cols, kw = facet_columns(n, seed + 1)
        rng = np.random.default_rng(seed + 2)
        cols["s16"] = rng.integers(0, len(S16), n, dtype=np.uint16)
        cols["loc"] = _points(n, seed + 3)
        cols["big"] = rng.integers(0, 100000, n, dtype=np.uint32)
        cols["big"][0] = 99999
        self.cols = cols
        self.ix.set_facets(cols, string_facets=kw["string_facets"] + ("big",), timestamp_facets=kw["timestamp_facets"],
                           string_values={"s16": S16, "s32": [f"v{i % 97:03d}" for i in range(300)]}, point_facets=("loc",))
        rows, fields, first, nd, rb = self.ix._facet_rows
        i = self.ix._facet_schema["loc"][0]
        self.codes = rows[:nd, fields[i].offset:fields[i].offset + 8].copy().view(np.uint64).reshape(-1)
        self.dist = {}

    def distances(self, base, unit):
        key = (base, unit)
        if key not in self.dist:
            d = np.array([euclidian_distance(base, decode(int(c)), unit) for c in self.codes])
            for s in PT_STARTS[1:]:
                assert not np.any(np.abs(d - s) <= 1e-12 * s), "a doc lies at a range start"
            self.dist[key] = d
        return self.dist[key]

    def matches(self, keys, qt, not_keys=None, deleted=(), filters=None, phrase=False):
        hits, tot = all_matches(self.orc, self.n, keys, qt, phrase=phrase, not_keys=not_keys)
        docs = hits["doc_id"].astype(np.int64)
        if len(deleted):
            docs = np.setdiff1d(docs, np.asarray(deleted, dtype=np.int64))
        if filters:
            docs = np.array([d for d in docs if numpy_pass(self.cols, [f for f in filters if f.base is None], d)], dtype=np.int64)
            for f in filters:
                if f.base is not None:
                    rej = filter_rejects(self.codes, f.base, f.start, f.end, f.unit)
                    docs = np.setdiff1d(docs, rej)
        return docs

    def expect(self, docs, qf, base=None):
        if qf.ranges:
            if qf.field == "loc":
                v = self.distances(tuple(base), qf.unit)[docs]
                starts = np.asarray([r[1] for r in qf.ranges], dtype=np.float64)
            else:
                c = self.cols[qf.field]
                v = c[docs]
                starts = np.asarray([r[1] for r in qf.ranges], dtype=c.dtype)
            b = np.searchsorted(starts, v, "right") - 1
            ok = b >= 0
            if v.dtype.kind == "f":
                ok &= ~np.isnan(v)
            return np.bincount(b[ok], minlength=len(starts)).astype(int).tolist()
        ids, cnt = np.unique(self.cols[qf.field][docs].astype(np.int64), return_counts=True)
        if qf.prefix:
            order = self.ix._string_order[qf.field]
            lo, hi = I.prefix_rank_interval(order, qf.prefix.encode())
            rank = {s: i for i, s in enumerate(order)}
            strs = self.ix._string_values[qf.field]
            keep = np.array([lo <= rank[strs[i].encode()] < hi for i in ids], dtype=bool)
            ids, cnt = ids[keep], cnt[keep]
        o = np.lexsort((ids, -cnt))
        return [(int(ids[j]), int(cnt[j])) for j in o[:qf.length]]


@pytest.fixture(scope="module")
def corpus():
    c = Corpus()
    yield c
    c.ix.close()


def _queries(seed, nq, lo=1, hi=6):
    r = np.random.default_rng(seed)
    return query_keys([sorted(set(int(x) for x in r.integers(1, 1500, int(r.integers(lo, hi + 1))))) for _ in range(nq)])


def _type_facets(c, seed):
    rng = np.random.default_rng(seed)
    qfs = [QueryFacet(name, ranges=[(f"r{j}", s) for j, s in enumerate(_starts(c.cols[name], int(rng.integers(2, 9)), rng))])
           for name in ("u8", "u16", "u32", "u64", "i8", "i16", "i32", "i64", "ts", "f32", "f64")]
    qfs.append(QueryFacet("loc", ranges=[(f"d{j}", s) for j, s in enumerate(PT_STARTS)], base=BASES[0], unit=DistanceUnit.Kilometers))
    qfs += [QueryFacet("s16", length=50), QueryFacet("s32", length=7)]
    return qfs


def _check(c, qk, qt, qfs, raw, docs_of, bases=None):
    errs = []
    for i, k in enumerate(qk):
        docs = docs_of(i, k)
        for r, qf in enumerate(qfs):
            want = c.expect(docs, qf, bases[i] if bases is not None else qf.base)
            if raw[i][qf.field] != want:
                errs.append((i, qf.field, raw[i][qf.field][:6], want[:6]))
    assert not errs, (len(errs), errs[:4])


@pytest.mark.parametrize("qt", [QueryType.Union, QueryType.Intersection])
def test_every_type_or_and(corpus, qt):
    """every facet type, OR / AND with 1..6 terms and 5..12 terms (the generic path), queries without a match; the u32 bins (first start
    = 0) sum to count_total of a TopkCount search of the same batch"""
    c = corpus
    qk = _queries(5 + int(qt), 48) + _queries(7 + int(qt), 8, 5, 12) + [[123456789]]
    qfs = _type_facets(c, 3 + int(qt))
    raw = c.ix.search_lexical_facets(qk, qt, qfs)
    _check(c, qk, qt, qfs, raw, lambda i, k: c.matches(k, qt))
    _, counts = c.ix.search_lexical_batch(qk, qt, 10, ResultType.TopkCount)
    for i in range(len(qk)):
        assert sum(raw[i]["u32"]) == int(counts[i])
        assert sum(raw[i]["f64"]) == int(counts[i]) - int(np.isnan(c.cols["f64"][c.matches(qk[i], qt)]).sum())
    assert sum(1 for i in range(len(qk)) if counts[i]) > (30 if qt == QueryType.Union else 10) and int(counts[-1]) == 0
    st = c.ix.last_stats()
    assert st["kernel_launches"] >= 3 and st["algorithmic_bytes"] > 0


def test_not_deleted_filters_points(corpus):
    """NOT terms, a delete set, range / set / Point facet filters; Point facets in km and miles with a per-query base"""
    c = corpus
    nq = 40
    qk = _queries(21, nq)
    r = np.random.default_rng(22)
    nots = [[int(x) for x in query_keys([[int(r.integers(1, 60))]])[0]] if i % 3 == 0 else [] for i in range(nq)]
    base_cols = {k: c.cols[k] for k in ("u8", "u32", "i32", "f32", "s16", "s32")}
    filters = random_filters(base_cols, 23, nq, 2)
    for i in range(0, nq, 4):
        filters[i] = filters[i] + [FacetFilter("loc", 0.0, 400.0 if i % 8 else 300.0, base=BASES[(i // 4) % 2], unit=DistanceUnit.Kilometers)]
    deleted = sorted(set(int(x) for x in r.integers(0, c.n, 3000)))
    c.ix.set_deleted(deleted)
    try:
        bases = [[BASES[i % 2], BASES[(i + 1) % 2]] for i in range(nq)]
        qfs = [QueryFacet("u16", ranges=[("a", 0), ("b", 1000), ("c", 30000)]),
               QueryFacet("loc", ranges=[(f"d{j}", s) for j, s in enumerate(PT_STARTS)], base=BASES[0], unit=DistanceUnit.Kilometers),
               QueryFacet("s16", length=4, prefix="ap")]
        qfs_m = qfs[:2] + [QueryFacet("f64", ranges=[("lo", -math.inf), ("mid", 0.0)])]
        # the second Point request is in miles on another facet request set: one base per Point request and query
        raw = c.ix.search_lexical_facets(qk, QueryType.Union, qfs, not_keys=nots, filters=filters, facet_bases=[[b[0]] for b in bases])
        _check(c, qk, QueryType.Union, qfs, raw, lambda i, k: c.matches(k, QueryType.Union, nots[i] or None, deleted, filters[i]),
               bases=[b[0] for b in bases])
        qmi = [QueryFacet("loc", ranges=[(f"d{j}", s) for j, s in enumerate(PT_STARTS)], base=BASES[1], unit=DistanceUnit.Miles)]
        raw = c.ix.search_lexical_facets(qk, QueryType.Intersection, qmi, not_keys=nots, filters=filters, facet_bases=[[b[1]] for b in bases])
        _check(c, qk, QueryType.Intersection, qmi, raw, lambda i, k: c.matches(k, QueryType.Intersection, nots[i] or None, deleted, filters[i]),
               bases=[b[1] for b in bases])
        _, counts = c.ix.search_lexical_batch(qk, QueryType.Union, 10, ResultType.TopkCount, not_keys=nots, filters=filters)
        raw = c.ix.search_lexical_facets(qk, QueryType.Union, qfs_m, not_keys=nots, filters=filters)
        for i in range(nq):
            assert sum(raw[i]["u16"]) == int(counts[i])
    finally:
        c.ix.set_deleted([])


def test_values_selection_batch_invariance_chunks(corpus):
    """String facets: ties in count (id ascending), prefixes (shared prefixes, equal strings), length 0 / 1 / above the distinct values;
    one query alone == the same query in a 1024-query batch; two calls agree; a String32 facet of 100 000 ids runs in several chunks"""
    c = corpus
    qk = _queries(41, 1024)
    for qf_set in ([QueryFacet("s16", length=100, prefix="ap"), QueryFacet("s32", length=3, prefix="v00")], [QueryFacet("s16", length=1)], [QueryFacet("s16", length=0)],
                   [QueryFacet("s16", length=5, prefix="zz")], [QueryFacet("s16", length=5, prefix="q")],
                   [QueryFacet("s32", length=20, prefix="v0"), QueryFacet("big", length=10)]):
        raw = c.ix.search_lexical_facets(qk[:24], QueryType.Union, qf_set)
        _check(c, qk[:24], QueryType.Union, qf_set, raw, lambda i, k: c.matches(k, QueryType.Union))
    big = [QueryFacet("big", length=12), QueryFacet("s16", length=3)]
    raw_a = c.ix.search_lexical_facets(qk, QueryType.Union, big)
    raw_b = c.ix.search_lexical_facets(qk, QueryType.Union, big)
    assert raw_a == raw_b
    assert c.ix.last_stats()["kernel_launches"] >= 5                  # plan + two chunks of (lex_facets, facet_select)
    for i in (0, 511, 700, 1023):
        assert c.ix.search_lexical_facets([qk[i]], QueryType.Union, big)[0] == raw_a[i]
        _check(c, [qk[i]], QueryType.Union, big, [raw_a[i]], lambda j, k: c.matches(k, QueryType.Union))
    ties = [x for x in raw_a[0]["big"] if x[1] == raw_a[0]["big"][-1][1]]
    assert ties == sorted(ties)


def test_phrase_single_and_multifield():
    """a single-field phrase batch, and two indexed fields with a field filter (per-field position runs)"""
    n, vocab = 60000, 250
    docs, levels, ls = sequence_corpus(n, vocab, 31)
    orc = oracle_index(levels, n, ls)
    ix = Index(0)
    for lv in levels:
        ix.add_lexical_level(lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"], lv["doc_len_bytes"],
                             lv["positions"])
    ix.commit(n, ls)
    col = np.random.default_rng(5).integers(0, 40, n).astype(np.uint8)
    ix.set_facets({"c": col})
    qk = query_keys(phrase_queries(docs, 33, 48, vocab))
    qf = [QueryFacet("c", ranges=[("a", 0), ("b", 10), ("c", 30)])]
    raw = ix.search_lexical_facets(qk, QueryType.Phrase, qf)
    _, cnt = ix.search_lexical_batch(qk, QueryType.Phrase, 10, ResultType.TopkCount)
    n_hit = 0
    for i, k in enumerate(qk):
        h, tot = all_matches(orc, n, k, QueryType.Phrase, phrase=True)
        d = h["doc_id"].astype(np.int64)
        want = np.bincount(np.searchsorted([0, 10, 30], col[d], "right") - 1, minlength=3).tolist()
        assert raw[i]["c"] == want and sum(want) == int(cnt[i]) == tot
        n_hit += tot > 0
    assert n_hit > 5
    ix.close()
    n2 = 72000
    docs, levels, ls = multifield_sequence_corpus(n2, 200, 2, seed=35)
    boosts = [1.0, 0.5]
    ix = Index(0)
    ix.set_field_boosts(boosts)
    for lv in levels:
        ix.add_lexical_level(lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"], lv["doc_len_bytes"],
                             lv["positions"])
    ix.commit(n2, ls)
    orc2 = PhraseFieldsOracle(levels, n2, ls, boosts)
    col = np.random.default_rng(6).integers(0, 40, n2).astype(np.uint8)
    ix.set_facets({"c": col})
    qk = query_keys(phrase_queries_mf(docs, 37, 40, 200))
    masks = [(i % 3) for i in range(len(qk))]                           # 0 = no field filter, 1 / 2 = one field
    raw = ix.search_lexical_facets(qk, QueryType.Phrase, qf, field_masks=masks)
    _, cnt = ix.search_lexical_batch(qk, QueryType.Phrase, 10, ResultType.TopkCount, field_masks=masks)
    n_hit = 0
    for i, k in enumerate(qk):
        d = np.array(sorted(orc2.phrase_docs(k, masks[i])), dtype=np.int64)
        want = np.bincount(np.searchsorted([0, 10, 30], col[d], "right") - 1, minlength=3).tolist() if len(d) else [0, 0, 0]
        assert raw[i]["c"] == want and sum(want) == int(cnt[i])
        n_hit += len(d) > 0
    assert n_hit > 5
    ix.close()


def test_search_mirror_and_refusals(corpus):
    """Index.search(query_facets=...) end to end against the restatement; the library's refusals"""
    c = corpus
    qfs = [QueryFacet("u32", range_type=RangeType.CountAboveRange, ranges=[("x", 0), ("y", 2**31), ("z", 3 * 2**30)]),
           QueryFacet("s16", length=3, prefix="a"), QueryFacet("loc", ranges=[("near", 0.0), ("far", 300.0)], base=BASES[1])]
    terms = "t3 t7 t11"
    ro = c.ix.search(terms, query_facets=qfs, length=5)
    keys = [c.ix.term_key_fn(t) for t in terms.split()]
    docs = c.matches(keys, QueryType.Union)
    raw = {qf.field: c.expect(docs, qf, qf.base) for qf in qfs}
    assert ro.result_count_total == len(docs) and ro.facets == c.ix.assemble_facets(raw, qfs) and ro.facets
    assert c.ix.search(terms, query_facets=qfs, result_type=ResultType.Topk).facets == {}
    from seekstorm_b200._lib import SsbFacetRequest, check, lib
    import ctypes as C
    b, keep = c.ix._lex_batch([keys], QueryType.Union)
    out = np.zeros(64, dtype=[("value", np.uint32), ("pad", np.uint32), ("count", np.uint64)])
    n_out = np.zeros(16, dtype=np.uint32)
    s = np.array([5, 5], dtype=np.uint64)
    bad = [SsbFacetRequest(c.ix._facet_schema["u32"][0], 1, 0, 0, 0, 0, 2, 0, s.ctypes.data),            # starts not ascending
           SsbFacetRequest(c.ix._facet_schema["loc"][0], 1, 0, 0, 0, 0, 1, 0, s.ctypes.data),            # Point without bases
           SsbFacetRequest(c.ix._facet_schema["u8"][0], 0, 3, 0, 0, 0, 0, 0, None),                     # VALUES on a number
           SsbFacetRequest(99, 0, 3, 0, 0, 0, 0, 0, None)]                                              # no such facet
    for r in bad:
        arr = (SsbFacetRequest * 1)(r)
        rc = lib().ssb_search_lexical_facets(c.ix._h, C.byref(b), C.addressof(arr), 1, None, out.ctypes.data, n_out.ctypes.data)
        assert rc == -1, rc
