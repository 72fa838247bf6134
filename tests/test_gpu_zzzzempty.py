"""GPU: the empty query (ssb_search_empty / ssb_search_empty_facets, Index.search("", enable_empty_query=True)).  Expectations come from
helpers_empty: the doc universe of the levels outside the delete set, the typed numpy columns' filter test, and the typed sort order (ranks
of helpers_sort.FacetRows, Point distances restated with math.cos) with ties to the larger doc id — never from the library's keys."""
import ctypes as C

import numpy as np
import pytest

from helpers_empty import live_docs, numpy_route, shard_route, top_values, value_fn
from helpers_facets import facet_columns, random_filters
from helpers_geo import DEG2RAD, decode_np, morton_range, simplified_distance
from helpers_sort import FacetRows
from seekstorm_b200 import DistanceUnit, FacetFilter, Index, QueryFacet, ResultSort, ResultType, SortOrder, _lib

pytestmark = pytest.mark.gpu

E_INVALID, E_UNSUPPORTED = -1, -5                                      # SSB_E_INVALID, SSB_E_UNSUPPORTED

# non-contiguous level ids, two short levels, the last one not a multiple of the tile
LEVELS = [(0, 65536), (1, 65536), (3, 40000), (4, 4097), (7, 1000)]
N_ROWS = (7 << 16) + 1000
BASE = (50.0, 10.0)


def _index(cols, first_doc=0, deleted=(), levels=LEVELS, **kw):
    ix = Index(0)
    for lv, n in levels:
        ix.add_lexical_level(lv, n, np.array([8], dtype=np.uint64), np.array([0, 1], dtype=np.uint32), np.array([0], dtype=np.uint16),
                             np.array([1], dtype=np.uint16), np.ones(n, dtype=np.uint8))
    ix.commit(sum(n for _, n in levels), sum(n for _, n in levels))
    ix.set_facets(cols, first_doc, **kw)
    if deleted:
        ix.set_deleted(deleted)
    return ix


def _point_pass(codes, f):
    """FacetFilter::Point (add_result.rs:462-478) vectorised: inside the Morton interval and start <= euclidian distance < end; no distance
    may lie within a relative 1e-12 of a bound (the precision contract's condition)"""
    lo, hi = morton_range(f.base, f.end, f.unit)
    inside = (codes >= np.uint64(lo)) & (codes < np.uint64(hi)) if lo < hi else np.zeros(len(codes), dtype=bool)
    lat, lon = decode_np(codes)
    x = DEG2RAD * (lon - f.base[1]) * np.cos(DEG2RAD * (f.base[0] + lat) / 2.0)
    y = DEG2RAD * (lat - f.base[0])
    d = (6371.0087714 if f.unit == DistanceUnit.Kilometers else 3958.761315801475) * np.sqrt(x * x + y * y)
    for b in (f.start, f.end):
        assert not np.any(inside & (np.abs(d - b) <= 1e-12 * abs(b))), "a doc lies at a bound"
    return inside & (f.start <= d) & (d < f.end)


def _mask(cols, fl, docs, first_doc=0, pts=None):
    """is_facet_filter on the typed numpy columns, vectorised: True = passes; a doc without a facet row fails every filter"""
    docs = np.asarray(docs, dtype=np.int64)
    n = len(next(iter(cols.values())))
    row = docs - first_doc
    has = (row >= 0) & (row < n)
    rr = np.clip(row, 0, n - 1)
    m = np.ones(len(docs), dtype=bool)
    for f in fl:
        if f.base is not None:
            m &= _point_pass(pts[rr], f)
            continue
        c = cols[f.field][rr]
        if f.values is not None:
            m &= np.isin(c.astype(np.int64), np.asarray(f.values, dtype=np.int64))
        elif c.dtype.kind == "f":
            x = c.astype(np.float64)
            m &= (float(f.start) <= x) & (x < float(f.end))
        else:
            m &= (f.start <= c) & (c < f.end)
    return m & has if fl else m


@pytest.fixture(scope="module")
def world():
    cols, kw = facet_columns(N_ROWS, 41)
    r = np.random.default_rng(5)
    pts = np.stack([r.uniform(45, 55, N_ROWS), r.uniform(5, 15, N_ROWS)], axis=1)
    cols = dict(cols, loc=pts)
    strings = {"s16": [f"v{i:02d}" for i in range(12)][::-1], "s32": [f"w{(i * 7) % 300:03d}" for i in range(300)]}
    deleted = sorted(set(int(x) for x in r.choice(live_docs(LEVELS), 3000, replace=False)))
    ix = _index(cols, 0, deleted, point_facets=("loc",), string_values=strings, **kw)
    facets = FacetRows.of_index(ix, strings)
    from seekstorm_b200.index import point_column
    pcodes = point_column(pts)
    universe = np.asarray(live_docs(LEVELS, deleted), dtype=np.int64)
    yield dict(ix=ix, cols=cols, pcodes=pcodes, facets=facets, universe=universe, deleted=deleted)
    ix.close()


def _filter_batch(w, nq, seed):
    base = {k: v for k, v in w["cols"].items() if k != "loc"}
    fls = random_filters(base, seed, nq)
    for i in range(0, nq, 7):                                            # POINT filters
        fls[i] = fls[i] + [FacetFilter("loc", 0.0, float(50 + 40 * (i % 5)), base=BASE, unit=DistanceUnit.Kilometers)]
    return fls


@pytest.mark.parametrize("rt", [ResultType.TopkCount, ResultType.Count, ResultType.Topk])
def test_filters_every_type(world, rt):
    w = world
    fls = _filter_batch(w, 96, 7)
    got, counts = w["ix"].search_empty_batch(len(fls), 10, rt, filters=fls)
    for i, fl in enumerate(fls):
        m = _mask(w["cols"], fl, w["universe"], 0, w["pcodes"])
        want = [int(d) for d in w["universe"][m][::-1][:10]]
        if rt != ResultType.Count:
            assert [d for d, _ in got[i]] == want, (i, fl)
            assert all(s == 0.0 for _, s in got[i])
        else:
            assert got[i] == []
        if rt != ResultType.Topk:
            assert int(counts[i]) == int(m.sum()), (i, fl)


@pytest.mark.parametrize("k", [1, 10, 32, 100, 1024])
def test_k_paging(world, k):
    w = world
    fls = _filter_batch(w, 12, 11)
    for sort in (None, [ResultSort("u16", SortOrder.Ascending)]):
        got, counts = w["ix"].search_empty_batch(len(fls), k, ResultType.TopkCount, filters=fls, sort=sort)
        for i, fl in enumerate(fls):
            m = _mask(w["cols"], fl, w["universe"], 0, w["pcodes"])
            crit = [("u16", False)] if sort else []
            want = numpy_route(w["universe"], m, k, crit, lambda n, d: w["facets"].rank(n)[d])
            assert [d for d, _ in got[i]] == want, (k, i)
            assert int(counts[i]) == int(m.sum())


SORTS = [[(n, d)] for n in ("u8", "u16", "u32", "u64", "i8", "i16", "i32", "i64", "ts", "f32", "f64", "s16", "s32") for d in (False, True)] + [
    [("_id", True)], [("_id", False)], [("_score", True)], [("_score", False)], [("s16", True), ("u8", False)],
    [("u8", True), ("_id", False)], [("i16", False), ("_score", False)]]


@pytest.mark.parametrize("crit", SORTS, ids=lambda c: "+".join(f"{n}{'D' if d else 'A'}" for n, d in c))
def test_sorted(world, crit):
    w = world
    fls = _filter_batch(w, 8, 13)[:8]
    fls[0] = []
    sort = [ResultSort(n, SortOrder.Descending if d else SortOrder.Ascending) for n, d in crit]
    got, _ = w["ix"].search_empty_batch(len(fls), 40, ResultType.Topk, filters=fls, sort=sort)
    for i, fl in enumerate(fls):
        m = _mask(w["cols"], fl, w["universe"], 0, w["pcodes"])
        want = numpy_route(w["universe"], m, 40, crit, lambda n, d: w["facets"].rank(n)[d])
        assert [d for d, _ in got[i]] == want, (crit, i)


def test_point_sort_with_bases(world):
    w = world
    bases = [(50.0 + 0.5 * i, 10.0 - 0.3 * i) for i in range(6)]
    fls = [[FacetFilter("u8", 0, 12)]] * 6
    for desc in (False, True):
        got, _ = w["ix"].search_empty_batch(6, 20, ResultType.TopkCount, filters=fls,
                                            sort=[ResultSort("loc", SortOrder.Descending if desc else SortOrder.Ascending, base=bases[0])],
                                            sort_bases=bases)
        for i in range(6):
            m = _mask(w["cols"], fls[i], w["universe"])
            docs = w["universe"][m]
            lat, lon = decode_np(w["pcodes"][docs])
            dist = np.array([simplified_distance((a, o), bases[i]) for a, o in zip(lat, lon)])
            rank = np.unique(dist, return_inverse=True)[1]
            lut = dict(zip(docs.tolist(), rank.tolist()))
            want = numpy_route(docs, np.ones(len(docs), bool), 20, [("loc", desc)], lambda n, d: np.array([lut[int(x)] for x in d]))
            assert [d for d, _ in got[i]] == want, (desc, i)


def test_literal_shard_route(world):
    """a few queries against the literal restatement (heap, typed comparator) on the full universe"""
    w = world
    v = value_fn(w["facets"])
    for crit, fl in (([("s32", False), ("u8", True)], [FacetFilter("u16", 0, 3000)]), ([], [FacetFilter("s16", values=[3])]),
                     ([("f32", True)], [FacetFilter("i8", -3, 2)])):
        sort = [ResultSort(n, SortOrder.Descending if d else SortOrder.Ascending) for n, d in crit]
        got, counts = w["ix"].search_empty_batch(1, 25, ResultType.TopkCount, filters=[fl], sort=sort or None)
        m = _mask(w["cols"], fl, w["universe"])
        ok = set(w["universe"][m].tolist())
        want, cnt = shard_route(w["universe"].tolist(), ok.__contains__, 25, _lib.RESULT_TOPKCOUNT, crit, v)
        assert [d for d, _ in got[0]] == want and int(counts[0]) == cnt


def test_zone_skipping_time_ordered():
    n_rows = (7 << 16) + 1000
    ts = (1_600_000_000 + np.arange(n_rows, dtype=np.int64) * 3)
    price = np.random.default_rng(2).integers(0, 1000, n_rows).astype(np.uint32)
    ix = _index({"ts": ts, "price": price}, timestamp_facets=("ts",))
    try:
        universe = np.asarray(live_docs(LEVELS), dtype=np.int64)
        lo, hi = int(ts[100_000]), int(ts[100_000] + 3 * 20_000)
        fls = [[FacetFilter("ts", lo, hi)], [FacetFilter("ts", lo, hi), FacetFilter("price", 100, 300)]]
        got, counts = ix.search_empty_batch(2, 10, ResultType.TopkCount, filters=fls)
        st = ix.last_stats()
        for i, fl in enumerate(fls):
            m = _mask({"ts": ts, "price": price}, fl, universe)
            assert [d for d, _ in got[i]] == [int(d) for d in universe[m][::-1][:10]]
            assert int(counts[i]) == int(m.sum())
        assert st["items_skipped"] > 0 and st["items_processed"] > 0, st
        _, c = ix.search_empty_batch(1, 0, ResultType.Count, filters=[fls[0]])
        assert int(c[0]) == int(_mask({"ts": ts}, fls[0], universe).sum())
    finally:
        ix.close()


def test_docs_without_rows():
    """facet rows start inside level 1: the docs before have none and fail every filter; unfiltered queries still see them"""
    first = (1 << 16) + 5000
    n = N_ROWS - first
    col = (np.arange(n) % 50).astype(np.uint8)
    ix = _index({"c": col}, first_doc=first)
    try:
        universe = np.asarray(live_docs(LEVELS), dtype=np.int64)
        fls = [[], [FacetFilter("c", 0, 10)], [FacetFilter("c", 0, 255)]]
        got, counts = ix.search_empty_batch(3, 5, ResultType.TopkCount, filters=fls, sort=[ResultSort("_id", SortOrder.Ascending)])
        for i, fl in enumerate(fls):
            m = _mask({"c": col}, fl, universe, first)
            assert [d for d, _ in got[i]] == [int(d) for d in universe[m][:5]], i
            assert int(counts[i]) == int(m.sum())
    finally:
        ix.close()


def test_batch_invariance(world):
    w = world
    fls = _filter_batch(w, 1000, 17)
    sort = [ResultSort("u32", SortOrder.Descending)]
    got, counts = w["ix"].search_empty_batch(1000, 10, ResultType.TopkCount, filters=fls, sort=sort)
    for i in range(0, 1000, 97):
        one, c1 = w["ix"].search_empty_batch(1, 10, ResultType.TopkCount, filters=[fls[i]], sort=sort)
        assert one[0] == got[i] and int(c1[0]) == int(counts[i]), i


def test_unfiltered_count_and_stats(world):
    w = world
    _, c = w["ix"].search_empty_batch(3, 0, ResultType.Count)
    assert c.tolist() == [len(w["universe"])] * 3
    assert w["ix"].last_stats()["kernel_launches"] == 0
    got, c = w["ix"].search_empty_batch(2, 10, ResultType.TopkCount)
    assert [d for d, _ in got[0]] == w["universe"][::-1][:10].tolist() and c.tolist() == [len(w["universe"])] * 2
    st = w["ix"].last_stats()
    assert st["kernel_launches"] == 1 and st["dominant_kernel_ns"] > 0


def test_refusals(world):
    w = world
    ix = w["ix"]
    with pytest.raises(_lib.SsbError):
        ix.search_empty_batch(1, 1025, ResultType.Topk)                  # above SSB_K_LIMIT
    b, keep = ix._lex_batch([[8]], 0)
    hits = np.zeros(16, dtype=np.uint8)
    nh, ct = np.zeros(1, np.uint32), np.zeros(1, np.uint64)
    rc = _lib.lib().ssb_search_empty(ix._h, C.byref(b), None, 0, None, 1, 1, hits.ctypes.data, nh.ctypes.data, ct.ctypes.data)
    assert rc == E_INVALID
    ix2 = _index({"c": np.zeros(N_ROWS, np.uint8)})
    try:
        assert _lib.lib().ssb_comm_attach(ix2._h, C.c_void_p(1), 0, 2) == 0
        b, keep = ix2._lex_batch([[]], 0)
        b.term_offsets = None
        rc = _lib.lib().ssb_search_empty(ix2._h, C.byref(b), None, 0, None, 1, 1, hits.ctypes.data, nh.ctypes.data, ct.ctypes.data)
        assert rc == E_UNSUPPORTED
        out = np.zeros(4, dtype=np.uint8)
        assert _lib.lib().ssb_search_empty_facets(ix2._h, None, 0, out.ctypes.data, out.ctypes.data) == E_UNSUPPORTED
        assert _lib.lib().ssb_comm_destroy(ix2._h) == 0
    finally:
        ix2.close()


def test_empty_facets(world):
    w = world
    cols, facets = w["cols"], w["facets"]
    order = w["ix"]._string_order["s32"]
    got = w["ix"].search_empty_facets([QueryFacet("s16", length=5), QueryFacet("s32", length=7, prefix="w1"),
                                       QueryFacet("u8", ranges=[("a", 0), ("b", 100)])])
    rank = {i: order.index(s.encode()) for i, s in enumerate(facets.strings["s32"])}
    lo, hi = [j for j, s in enumerate(order) if s.startswith(b"w1")][0], [j for j, s in enumerate(order) if s.startswith(b"w1")][-1] + 1
    assert got["s16"] == top_values(cols["s16"], 5)                  # every row: deleted docs included
    assert got["s32"] == top_values(cols["s32"], 7, lambda i: lo <= rank[i] < hi)
    assert "u8" not in got


def test_python_mirror_routes(world):
    w = world
    ix, U = w["ix"], w["universe"]
    ro = ix.search("", enable_empty_query=True, offset=3, length=5)
    assert [r.doc_id for r in ro.results] == U[::-1][3:8].tolist() and ro.result_count_total == len(U) and ro.result_count == 5
    ro = ix.search("", enable_empty_query=True, result_sort=[ResultSort("_score", SortOrder.Ascending)])
    assert [r.doc_id for r in ro.results] == U[:10].tolist()
    ro = ix.search("", enable_empty_query=True, result_type=ResultType.Topk, facet_filter=[FacetFilter("u8", 10, 20)])
    m = _mask(w["cols"], [FacetFilter("u8", 10, 20)], U)
    assert [r.doc_id for r in ro.results] == U[m][::-1][:10].tolist() and ro.result_count_total == 0
    ro = ix.search("", enable_empty_query=True, result_type=ResultType.Count, facet_filter=[FacetFilter("u8", 10, 20)],
                   query_facets=[QueryFacet("s16", length=3)])
    assert ro.results == [] and ro.result_count_total == int(m.sum())
    assert ro.facets == {"s16": [(w["facets"].strings["s16"][i], c) for i, c in top_values(w["cols"]["s16"], 3)]}


def test_reference_fixture_test_05(golden):
    """test_05_empty_query (tests/test.rs:215-335) on the reference's 4-doc fixture: default and _id descending start at doc 3, _id
    ascending at doc 0; 4 results, result_count 4 and result_count_total 4"""
    from helpers import gpu_index, level_from_postings
    fx = golden["ref_fixture_lexical"]
    ix = gpu_index([level_from_postings(0, fx["n_docs"], fx["postings"], fx["len_bytes"])], fx["n_docs"], fx["len_sum"])
    try:
        for sort, first in (((), 3), ([ResultSort("_id", SortOrder.Descending)], 3), ([ResultSort("_id", SortOrder.Ascending)], 0)):
            ro = ix.search("", enable_empty_query=True, result_sort=sort)
            assert ro.results[0].doc_id == first and len(ro.results) == 4, sort
            assert ro.result_count == 4 and ro.result_count_total == 4
    finally:
        ix.close()
