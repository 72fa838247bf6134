"""CPU: the sorted-search reference of the GPU tests (helpers_sort: the oracle's exhaustive matches ordered by a restatement of
result_ordering_shard, min_heap.rs:574-1051, and by the lexsort the GPU tests use) pinned against Python's stable sorted() applied
criterion by criterion on the typed numpy columns — every FieldType both ways with NaN / +-inf / +-0.0 and integer extremes, String16 / String32 by their strings, two criteria,
_id, _score ascending, criteria after _id, ties, Count."""
import numpy as np
import pytest

from oracle import oracle as O
from helpers import oracle_index, query_keys, synth_levels
from helpers_facets import facet_columns
from helpers_sort import FacetRows, search_sorted, sort_hits, sort_hits_cmp
from seekstorm_b200 import synth

N = 6000


def _strings(n_ids, seed):
    r = np.random.default_rng(seed)
    alphabet = ["a", "b", "B", "é", "z", "0", " ", "ab"]
    vals = ["".join(r.choice(alphabet, int(r.integers(0, 5)))) for _ in range(n_ids)]
    vals[1] = vals[0] + "a"                                   # a prefix orders first
    return vals


@pytest.fixture(scope="module")
def corpus():
    lvs, ls = synth_levels(N, 400, 501)
    orc = oracle_index([l.to_numpy() for l in lvs], N, ls)
    cols, _ = facet_columns(N, 502)
    cols["few"] = np.random.default_rng(503).integers(0, 3, N, dtype=np.uint8)      # many ties
    strings = {"s16": _strings(12, 504), "s32": _strings(300, 505)}
    qk = query_keys(synth.gen_queries(24, 506, 2, 300, (1, 2, 3), (0.3, 0.4, 0.3)))
    fr = FacetRows.pack(cols, string_facets=("s16", "s32"), timestamp_facets=("ts",), strings=strings)   # the bytes the library gets
    return orc, cols, strings, qk, fr


def _typed_key(cols, strings, name):
    c = cols[name]
    if name in strings:
        return lambda h: strings[name][int(c[h[0]])].encode("utf-8")
    if c.dtype.kind == "f":
        return lambda h: (1, 0.0) if np.isnan(c[h[0]]) else (0, float(c[h[0]]))
    return lambda h: int(c[h[0]])


def _stable_sorted(hits, criteria, cols, strings):
    """least significant first: doc id asc, score desc (or the final _score criterion), then each criterion from last to first"""
    crit = []
    for name, desc in criteria:
        crit.append((name, desc))
        if name in ("_id", "_score"):
            break
    out = sorted(hits, key=lambda h: h[0])
    if crit and crit[-1][0] == "_score":
        out = sorted(out, key=lambda h: np.float32(h[1]), reverse=crit[-1][1])
        crit = crit[:-1]
    else:
        out = sorted(out, key=lambda h: np.float32(h[1]), reverse=True)
    for name, desc in reversed(crit):
        key = (lambda h: h[0]) if name == "_id" else _typed_key(cols, strings, name)
        out = sorted(out, key=key, reverse=desc)
    return out


def _check(corpus, criteria, k=25):
    orc, cols, strings, qk, fr = corpus
    for q in qk:
        for qt in (O.QUERY_UNION, O.QUERY_INTERSECTION):
            all_hits, tot = orc.search(q, qt, N, O.RESULT_TOPKCOUNT)
            got, cnt = search_sorted(orc, N, q, qt, k, O.RESULT_TOPKCOUNT, criteria, fr)
            assert cnt == tot and len(all_hits) == tot
            want = _stable_sorted(all_hits, criteria, cols, strings)
            assert got == want[:k], (criteria, q)
            assert sort_hits_cmp(all_hits, criteria, fr) == want, (criteria, q)


TYPES = ["u8", "u16", "u32", "u64", "i8", "i16", "i32", "i64", "ts", "f32", "f64", "s16", "s32"]


@pytest.mark.parametrize("name", TYPES)
@pytest.mark.parametrize("desc", [True, False])
def test_every_type_both_orders(corpus, name, desc):
    _check(corpus, [(name, desc)], k=40)


def test_float_specials_order(corpus):
    orc, cols, strings, _, fr = corpus
    hits = [(d, 1.0) for d in range(N)]
    for name in ("f32", "f64"):
        desc = [cols[name][d] for d, _ in sort_hits(hits, [(name, True)], fr)]
        asc = [cols[name][d] for d, _ in sort_hits(hits, [(name, False)], fr)]
        n_nan = int(np.isnan(cols[name]).sum())
        assert n_nan > 0 and np.isnan(desc[:n_nan]).all() and np.isnan(asc[-n_nan:]).all()    # NaN above +inf
        assert desc[n_nan] == np.inf and asc[0] == -np.inf
        zeros = [d for d, _ in sort_hits(hits, [(name, True)], fr) if cols[name][d] == 0]
        assert zeros == sorted(zeros) and any(np.signbit(cols[name][d]) for d in zeros)   # -0.0 == +0.0: ties go by doc id


def test_two_criteria_and_ties(corpus):
    _check(corpus, [("few", True), ("f32", False)])
    _check(corpus, [("s16", False), ("u16", True)])
    orc, cols, strings, qk, fr = corpus
    got, _ = search_sorted(orc, N, qk[0], O.QUERY_UNION, 200, O.RESULT_TOPK, [("few", True)], fr)
    for (a, sa), (b, sb) in zip(got, got[1:]):                # inside one value: score desc, then doc id asc
        if cols["few"][a] == cols["few"][b]:
            assert np.float32(sa) > np.float32(sb) or (np.float32(sa) == np.float32(sb) and a < b)


def test_id_score_and_unreachable_criteria(corpus):
    _check(corpus, [("_id", True)])
    _check(corpus, [("_id", False)])
    _check(corpus, [("_score", False)])
    _check(corpus, [("few", False), ("_score", False)])
    orc, cols, strings, qk, fr = corpus
    for q in qk[:6]:
        a = search_sorted(orc, N, q, O.QUERY_UNION, 30, O.RESULT_TOPK, [("_id", False), ("u32", True)], fr)
        b = search_sorted(orc, N, q, O.QUERY_UNION, 30, O.RESULT_TOPK, [("_id", False)], fr)
        assert a == b and [d for d, _ in a[0]] == sorted(d for d, _ in a[0])
    # "_score desc" is the unsorted order
    for q in qk[:6]:
        assert search_sorted(orc, N, q, O.QUERY_UNION, 30, O.RESULT_TOPKCOUNT, [("_score", True)], fr) == \
            orc.search(q, O.QUERY_UNION, 30, O.RESULT_TOPKCOUNT)


def test_count_ignores_sort(corpus):
    orc, cols, strings, qk, fr = corpus
    for q in qk[:6]:
        hits, tot = search_sorted(orc, N, q, O.QUERY_UNION, 10, O.RESULT_COUNT, [("u8", True)], fr)
        assert hits == [] and tot == orc.search(q, O.QUERY_UNION, 10, O.RESULT_TOPKCOUNT)[1]


def test_all_matches_is_the_oracle_search(corpus):
    """all_matches reads the same C entry points as OracleIndex.search / search_phrase, without a Python tuple per hit"""
    from helpers_facets import abi_filters  # noqa: F401  (the filter tuples below are in the same C-ABI encoding)
    from helpers_sort import all_matches
    orc, cols, strings, qk, fr = corpus
    rows = fr.rows
    fields = [fr.fields[name] for name in cols]
    orc.set_facets(rows, fields, 0, N, rows.shape[1])
    u8 = list(cols).index("u8")
    flt = [(u8, 0, 40, 200, 0, 0)]
    for q in qk[:8]:
        for qt in (O.QUERY_UNION, O.QUERY_INTERSECTION):
            for kw in ({}, {"not_keys": qk[-1][:1]}, {"filters": flt}, {"filters": flt, "not_keys": qk[-1][:1]}):
                h, tot = all_matches(orc, N, q, qt, **kw)
                want, wtot = orc.search(q, qt, N, O.RESULT_TOPKCOUNT, **kw)
                assert tot == wtot and [(int(d), float(np.float32(s))) for d, s in zip(h["doc_id"], h["score"])] == want
