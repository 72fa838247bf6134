"""GPU: multi-value string facets (StringSet16 / StringSet32) — member filters on every scoring path, member counts of lexical matches and
of the empty query, sorting by the first member, and Index.search end to end.  Expected results: the C oracle with the docs a StringSet
filter rejects handed over as deleted docs (the other filters it applies itself), and the numpy formulation of helpers_stringset (pinned
to the literal restatement of the reference by test_stringset_cpu) for member filters, counts and first-member ranks."""
import numpy as np
import pytest

import helpers_stringset as S
from helpers_geo import filter_rejects
from helpers_phrase_mf import PhraseFieldsOracle, multifield_sequence_corpus, phrase_queries_mf
from oracle import oracle as O
from seekstorm_b200 import synth
from helpers import gpu_index, oracle_index, query_keys, synth_levels
from helpers_sort import all_matches

pytestmark = pytest.mark.gpu

N = 150000


def _tag_lists(n, n_tags, seed, hi=5, quirks=True):
    """1..hi Zipf-distributed tags per doc (some docs with none), plus the quirks: a tag spelled like a joined key, repeats, byte-order
    edges"""
    r = np.random.default_rng(seed)
    words = [f"t{i:05d}" for i in range(n_tags)]
    if quirks:
        words += ["t00000_t00001", "Zed", "ä", "é"]
    p = 1.0 / np.arange(1, len(words) + 1)
    p /= p.sum()
    k = r.integers(0 if quirks else 1, hi + 1, n)
    flat = r.choice(len(words), int(k.sum()), p=p)
    out, o = [], 0
    for c in k:
        out.append([words[i] for i in flat[o:o + c]])
        o += c
    if quirks:
        for d in r.integers(0, n, 300):
            out[d] = out[d] + out[d][:1]                                   # a repeated member
    return out


@pytest.fixture(scope="module")
def world():
    lvs, ls = synth_levels(N, 2500, 71)
    levels = [l.to_numpy() for l in lvs]
    orc = oracle_index(levels, N, ls)
    ix = gpu_index(levels, N, ls)
    rng = np.random.default_rng(72)
    cols = {"price": rng.integers(0, 1000, N, dtype=np.uint32), "cat": rng.integers(0, 40, N).astype(np.uint16), "loc": _points(N, 82),
            "tags": _tag_lists(N, 200, 73, hi=2), "tags32": _tag_lists(N, 20000, 74, quirks=False)}
    ix.set_facets(cols, string_facets=("cat",), point_facets=("loc",), string_set_facets=("tags",), string_set32_facets=("tags32",))
    rows, fields, first, nd, rb = ix._facet_rows
    orc.set_facets(rows, [(fields[i].type, fields[i].offset) for i in range(2)], first, nd, rb)   # the oracle takes price and cat
    codes = rows[:nd, fields[2].offset:fields[2].offset + 8].copy().view(np.uint64).reshape(-1)
    ss = ix._string_sets
    assert len(ss["tags"].combos) < 65535 and len(ss["tags32"].combos) > 65536 and len(ss["tags32"].members) > 12288
    qs = synth.gen_queries(48, 75, 2, 2000, (1, 2, 3, 4, 6), (0.15, 0.3, 0.25, 0.15, 0.15))
    return dict(ix=ix, orc=orc, ss=ss, qk=query_keys(qs), codes=codes)


def _points(n, seed):
    """positions around Berlin (52.52 N, 13.405 E): a Point filter there keeps a part of them"""
    r = np.random.default_rng(seed)
    return np.stack([52.52 + r.normal(0, 0.5, n), 13.405 + r.normal(0, 0.8, n)], axis=1)


def _filters(w, seed, nq):
    """per query one or two tag strings (OR inside a filter), sometimes a tags32 filter (AND), a price range or a cat set"""
    from seekstorm_b200 import FacetFilter
    r = np.random.default_rng(seed)
    out = []
    for i in range(nq):
        tags = [f"t{int(x):05d}" for x in r.integers(0, 40, 1 + i % 2)]
        if i % 7 == 3:
            tags = ["t00000_t00001"]                                           # a member and, maybe, a joined key
        if i % 9 == 4:
            tags = ["nope"]
        fl = [FacetFilter("tags", values=tags)]
        if i % 4 == 1:
            fl.append(FacetFilter("tags32", values=[f"t{int(x):05d}" for x in r.integers(0, 30, 3)]))
        if i % 5 == 2:
            fl.append(FacetFilter("price", 100, 800))
        if i % 6 == 5:
            fl.append(FacetFilter("cat", values=[int(x) for x in r.integers(0, 40, 12)]))
        if i % 3 == 2:                                                         # a POINT payload staged next to the MEMBERS payloads
            fl.append(FacetFilter("loc", 0.0, float(r.choice([30.0, 60.0])), base=(52.52, 13.405)))
        out.append(fl)
    return out


def _rejected(w, fl):
    """the docs the StringSet filters of one query reject (numpy formulation) and the oracle's share of the filters"""
    ok = np.ones(N, dtype=bool)
    rest = []
    for f in fl:
        if f.field in w["ss"]:
            s = w["ss"][f.field]
            ok &= S.combination_mask(s.offsets, s.member_ids, s.filter_values(f.values))[s.ids]
        elif f.base is not None:
            ok[filter_rejects(w["codes"], tuple(f.base), float(f.start), float(f.end), int(f.unit))] = False
        else:
            rest.append(f)
    tup, sv = None, None
    if rest:
        offs, arr, v = w["ix"]._encode_filters([rest])
        tup = [(arr[i].facet, arr[i].kind, arr[i].start, arr[i].end, arr[i].set_first, arr[i].set_count) for i in range(int(offs[1]))]
        sv = [int(x) for x in v]
    return set(np.nonzero(~ok)[0].tolist()), tup, sv


def test_filter_parity(world):
    from seekstorm_b200 import QueryType, ResultType
    w = world
    ix, orc, qk = w["ix"], w["orc"], w["qk"]
    filters = _filters(w, 76, len(qk))
    rng = np.random.default_rng(77)
    nk = [query_keys([[int(x)]])[0] if i % 3 == 0 else [] for i, x in enumerate(rng.integers(0, 50, len(qk)))]
    nk = [[t for t in n if t not in q] for n, q in zip(nk, qk)]
    args = [_rejected(w, fl) for fl in filters]
    errs, passed = [], 0
    for deleted in ([], [int(x) for x in rng.integers(0, N, 3000)]):
        ix.set_deleted(deleted)
        for qt, oqt in ((QueryType.Union, O.QUERY_UNION), (QueryType.Intersection, O.QUERY_INTERSECTION)):
            got, cnt = ix.search_lexical_batch(qk, qt, 10, ResultType.TopkCount, not_keys=nk, filters=filters)
            got_t, _ = ix.search_lexical_batch(qk, qt, 10, ResultType.Topk, not_keys=nk, filters=filters)
            _, cnt_c = ix.search_lexical_batch(qk, qt, 0, ResultType.Count, not_keys=nk, filters=filters)
            for i, k in enumerate(qk):
                rej, tup, sv = args[i]
                orc.set_deleted(sorted(set(deleted) | rej))
                kw = dict(filters=tup, set_values=sv) if tup else {}
                want, tot = orc.search(k, oqt, 10, O.RESULT_TOPKCOUNT, not_keys=nk[i], **kw)
                passed += tot > 0
                if got[i] != want or got_t[i] != want or int(cnt[i]) != tot or int(cnt_c[i]) != tot:
                    errs.append((bool(deleted), int(qt), i, filters[i], got[i][:3], want[:3], int(cnt[i]), int(cnt_c[i]), tot))
    ix.set_deleted([])
    orc.set_deleted([])
    assert not errs, (len(errs), errs[:4])
    assert passed > len(qk)


def _matches(w, k, qt, fl):
    rej, tup, sv = _rejected(w, fl)
    w["orc"].set_deleted(sorted(rej))
    hits, tot = all_matches(w["orc"], N, k, qt, filters=tup, set_values=sv)
    w["orc"].set_deleted([])
    return hits, tot


@pytest.mark.parametrize("field, prefix, length", [("tags", "", 10), ("tags", "t000", 7), ("tags", "", 1024), ("tags32", "", 10),
                                                   ("tags32", "t0001", 1024), ("tags", "é", 3)])
def test_member_counts(world, field, prefix, length):
    from seekstorm_b200 import QueryFacet, QueryType
    from seekstorm_b200.index import prefix_rank_interval
    w = world
    qk = w["qk"][:24]
    filters = _filters(w, 79, len(qk))
    s = w["ss"][field]
    raw = w["ix"].search_lexical_facets(qk, QueryType.Union, [QueryFacet(field, prefix=prefix, length=length)], filters=filters)
    lo, hi = prefix_rank_interval(s.members, prefix.encode("utf-8")) if prefix else (0, len(s.members))
    for i, k in enumerate(qk):
        hits, _ = _matches(w, k, O.QUERY_UNION, filters[i])
        docs = np.asarray(hits["doc_id"], dtype=np.int64)
        cnt = S.numpy_member_counts(s.offsets, s.member_ids, len(s.members), s.ids.astype(np.int64), docs)
        assert raw[i].get(field, []) == S.numpy_top(cnt, lo, hi, length), (i, field)


def _first_rank(s):
    pos = {m: i for i, m in enumerate(s.members)}
    first = np.array([pos[c[0].encode("utf-8")] if c else -1 for c in s.combos])
    u = np.unique(first[first >= 0])
    return np.where(first >= 0, np.searchsorted(u, first) + 1, 0)


@pytest.mark.parametrize("desc, tail, filtered", [(True, None, True), (False, None, True), (True, "_id", True), (False, "_score", True),
                                                   (True, None, False), (False, "_id", False)])
def test_sort_by_first_member(world, desc, tail, filtered):
    """filtered: the batch carries member filters (the GEO instantiations); else no filter at all (the common lex_generic rank path)"""
    from seekstorm_b200 import QueryType, ResultSort, ResultType, SortOrder
    w = world
    qk = w["qk"][:16]
    filters = _filters(w, 80, len(qk)) if filtered else None
    s = w["ss"]["tags"]
    rank = _first_rank(s)
    sort = [ResultSort("tags", SortOrder.Descending if desc else SortOrder.Ascending)]
    if tail:
        sort.append(ResultSort(tail, SortOrder.Ascending))
    got, cnt = w["ix"].search_lexical_batch(qk, QueryType.Union, 20, ResultType.TopkCount, filters=filters, sort=sort)
    for i, k in enumerate(qk):
        hits, tot = _matches(w, k, O.QUERY_UNION, filters[i] if filtered else [])
        d = np.asarray(hits["doc_id"], dtype=np.int64)
        sc = np.asarray(hits["score"], dtype=np.float32)
        r = rank[s.ids[d].astype(np.int64)]
        if tail == "_id":
            order = np.lexsort((d, -r if desc else r))
        elif tail == "_score":                                   # ascending score, then doc id ascending
            order = np.lexsort((d, sc, -r if desc else r))
        else:                                                    # ties: score descending, then doc id ascending
            order = np.lexsort((d, -sc, -r if desc else r))
        assert [x for x, _ in got[i]] == d[order][:20].tolist() and int(cnt[i]) == tot, i


def test_empty_query(world):
    from seekstorm_b200 import FacetFilter, QueryFacet, ResultSort, ResultType, SortOrder
    w = world
    ix, s = w["ix"], w["ss"]["tags"]
    deleted = sorted(set(int(x) for x in np.random.default_rng(81).integers(0, N, 2000)))
    ix.set_deleted(deleted)
    live = np.ones(N, dtype=bool)
    live[deleted] = False
    rank = _first_rank(s)
    fls = [[FacetFilter("tags", values=["t00003", "t00010"])], [FacetFilter("tags", values=["t00000_t00001"]), FacetFilter("price", 0, 500)],
           [FacetFilter("tags", values=["nope"])]]
    for sort in ([ResultSort("tags", SortOrder.Ascending)], [ResultSort("tags", SortOrder.Descending), ResultSort("_id", SortOrder.Ascending)], None):
        got, counts = ix.search_empty_batch(len(fls), 25, ResultType.TopkCount, filters=fls, sort=sort)
        for i, fl in enumerate(fls):
            ok = live.copy()
            ok &= S.combination_mask(s.offsets, s.member_ids, s.filter_values(fl[0].values))[s.ids]
            if len(fl) > 1:
                ok &= ix._facet_rows[0][:N, 0:4].copy().view(np.uint32).reshape(-1) < 500
            d = np.nonzero(ok)[0]
            r = rank[s.ids[d].astype(np.int64)]
            if sort is None:
                order = np.argsort(-d)
            elif len(sort) == 1:
                order = np.lexsort((-d, r))                             # ties: doc id descending
            else:
                order = np.lexsort((d, -r))
            assert [x for x, _ in got[i]] == d[order][:25].tolist() and int(counts[i]) == len(d), (i, sort)
    # no filter: the common empty_scan instantiation sorts by the first member too
    got, counts = ix.search_empty_batch(1, 25, ResultType.TopkCount, sort=[ResultSort("tags", SortOrder.Descending)])
    d = np.nonzero(live)[0]
    assert [x for x, _ in got[0]] == d[np.lexsort((-d, -rank[s.ids[d].astype(np.int64)]))][:25].tolist() and int(counts[0]) == len(d)
    ix.set_deleted([])
    for field, length, prefix in (("tags", 10, ""), ("tags32", 1024, ""), ("tags32", 5, "t0002")):
        t = w["ss"][field]
        res = ix.search_empty_facets([QueryFacet(field, prefix=prefix, length=length)])
        from seekstorm_b200.index import prefix_rank_interval
        lo, hi = prefix_rank_interval(t.members, prefix.encode()) if prefix else (0, len(t.members))
        cnt = S.numpy_member_counts(t.offsets, t.member_ids, len(t.members), t.ids.astype(np.int64), np.arange(N))
        assert res[field] == S.numpy_top(cnt, lo, hi, length), field


def test_index_search_end_to_end(world):
    from seekstorm_b200 import FacetFilter, QueryFacet, ResultSort, ResultType, SortOrder
    w = world
    ix, s = w["ix"], w["ss"]["tags"]
    ix.term_key_fn = lambda t: query_keys([[int(t[1:])]])[0][0]
    ro = ix.search("w3 w7", facet_filter=[FacetFilter("tags", values=["t00002"])], query_facets=[QueryFacet("tags", length=5)],
                   result_sort=[ResultSort("tags", SortOrder.Ascending)], length=10, result_type=ResultType.TopkCount)
    k = ix.term_key_fn("w3"), ix.term_key_fn("w7")
    hits, tot = _matches(w, list(k), O.QUERY_UNION, [FacetFilter("tags", values=["t00002"])])
    d = np.asarray(hits["doc_id"], dtype=np.int64)
    cnt = S.numpy_member_counts(s.offsets, s.member_ids, len(s.members), s.ids.astype(np.int64), d)
    assert ro.result_count_total == tot
    assert ro.facets.get("tags", []) == [(s.members[m].decode("utf-8"), c) for m, c in S.numpy_top(cnt, 0, None, 5)]
    rank = _first_rank(s)
    assert [r.doc_id for r in ro.results] == d[np.lexsort((d, -np.asarray(hits["score"]), rank[s.ids[d].astype(np.int64)]))][:10].tolist()
    e = ix.search("", enable_empty_query=True, facet_filter=[FacetFilter("tags", values=["t00002"])], query_facets=[QueryFacet("tags", length=3)])
    ok = S.combination_mask(s.offsets, s.member_ids, s.filter_values(["t00002"]))[s.ids]
    assert e.result_count_total == int(ok.sum()) and [r.doc_id for r in e.results] == np.nonzero(ok)[0][::-1][:10].tolist()
    allc = S.numpy_member_counts(s.offsets, s.member_ids, len(s.members), s.ids.astype(np.int64), np.arange(N))
    assert e.facets["tags"] == [(s.members[m].decode("utf-8"), c) for m, c in S.numpy_top(allc, 0, None, 3)]


def test_refusals(world):
    import ctypes as C
    from seekstorm_b200 import FacetFilter, QueryType, ResultType, _lib
    from seekstorm_b200._lib import SsbError, SsbFacetRequest, lib
    w = world
    ix, s = w["ix"], w["ss"]["tags"]
    idx = ix._facet_schema["tags"][0]
    with pytest.raises(SsbError, match="a String facet takes SSB_FILTER_SET"):
        ix.search_lexical_batch(w["qk"][:1], QueryType.Union, 10, ResultType.TopkCount, filters=[[FacetFilter(idx, 0, 5)]])
    with pytest.raises(SsbError, match="member id"):
        ix.search_lexical_batch(w["qk"][:1], QueryType.Union, 10, ResultType.TopkCount, filters=[[FacetFilter(idx, values=[len(s.members)])]])
    with pytest.raises(SsbError, match="combination id"):
        ix.search_lexical_batch(w["qk"][:1], QueryType.Union, 10, ResultType.TopkCount,
                                filters=[[FacetFilter(idx, values=[_lib.SET_COMBINATION | len(s.combos)])]])
    starts = np.zeros(1, dtype=np.uint64)
    req = (SsbFacetRequest * 1)(SsbFacetRequest(idx, _lib.FACET_COUNT_RANGES, 0, 0, 0, 0, 1, 0, starts.ctypes.data))
    out = np.zeros(4, dtype=np.uint64)
    n_out = np.zeros(2, dtype=np.uint32)
    assert lib().ssb_search_empty_facets(ix._h, C.addressof(req), 1, out.ctypes.data, n_out.ctypes.data) == -1
    bad = np.array([0, 1], dtype=np.uint64)
    mem = np.array([len(s.members)], dtype=np.uint32)
    assert lib().ssb_set_facet_string_sets(ix._h, idx, bad.ctypes.data, mem.ctypes.data, 1, len(s.members)) == -1   # SSB_E_INVALID: the column holds ids >= n_sets
    assert lib().ssb_set_facet_string_sets(ix._h, ix._facet_schema["price"][0], bad.ctypes.data, mem.ctypes.data, 1, 5) == -1
    # the refusals left the facet as it was
    got, cnt = ix.search_lexical_batch(w["qk"][:1], QueryType.Union, 10, ResultType.TopkCount, filters=[[FacetFilter("tags", values=["t00001"])]])
    hits, tot = _matches(w, w["qk"][0], O.QUERY_UNION, [FacetFilter("tags", values=["t00001"])])
    assert int(cnt[0]) == tot


def test_phrase_batches_multifield():
    """member filters on phrase batches over two indexed fields with per-field position runs (lex_generic<true, *, true> and
    lex_facets<true, *, true>), against the phrase oracle with the rejected docs deleted; member counts of the same batches"""
    from seekstorm_b200 import FacetFilter, QueryFacet, QueryType, ResultType
    from seekstorm_b200 import Index
    n = 72000
    docs, levels, ls = multifield_sequence_corpus(n, 200, 2, seed=85)
    boosts = (2.0, 1.0)
    ix = Index(0)
    ix.set_field_boosts(boosts)
    for lv in levels:
        ix.add_lexical_level(lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"], lv["doc_len_bytes"],
                             lv["positions"])
    ix.commit(n, ls)
    orc = PhraseFieldsOracle(levels, n, ls, boosts)
    ix.set_facets({"tags": _tag_lists(n, 30, 86, hi=3)}, string_set_facets=("tags",))
    s = ix._string_sets["tags"]
    qk = query_keys(phrase_queries_mf(docs, 87, 40, 200))
    r = np.random.default_rng(88)
    filters = [[FacetFilter("tags", values=[f"t{int(x):05d}" for x in r.integers(0, 12, 2)])] for _ in qk]
    masks = [S.combination_mask(s.offsets, s.member_ids, s.filter_values(fl[0].values))[s.ids] for fl in filters]
    got, cnt = ix.search_lexical_batch(qk, QueryType.Phrase, 10, ResultType.TopkCount, filters=filters)
    got_t, _ = ix.search_lexical_batch(qk, QueryType.Phrase, 10, ResultType.Topk, filters=filters)
    _, cnt_c = ix.search_lexical_batch(qk, QueryType.Phrase, 0, ResultType.Count, filters=filters)
    raw = ix.search_lexical_facets(qk, QueryType.Phrase, [QueryFacet("tags", length=20)], filters=filters)
    errs, n_hit = [], 0
    for i, k in enumerate(qk):
        orc.set_deleted(np.nonzero(~masks[i])[0].tolist())
        want, tot = orc.search_phrase(k, 10, O.RESULT_TOPKCOUNT)
        every, _ = orc.search_phrase(k, n, O.RESULT_TOPKCOUNT)
        n_hit += tot > 0
        cnt_m = S.numpy_member_counts(s.offsets, s.member_ids, len(s.members), s.ids.astype(np.int64), np.asarray([d for d, _ in every], dtype=np.int64))
        if got[i] != want or got_t[i] != want or int(cnt[i]) != tot or int(cnt_c[i]) != tot or raw[i].get("tags", []) != S.numpy_top(cnt_m, 0, None, 20):
            errs.append((i, got[i][:3], want[:3], int(cnt[i]), int(cnt_c[i]), tot))
    ix.close()
    assert not errs and n_hit > 5, (len(errs), errs[:4], n_hit)
