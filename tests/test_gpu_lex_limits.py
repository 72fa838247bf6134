"""GPU: the BM25 engine at its structural limits against the exhaustive C oracle — list lengths on both sides of DENSE_MIN (128) and
UNION_WORDS (2048), AND count ratios at 8·cnt_a / 8·cnt_a + 1, plans of 3 to 4096 levels (padded bitonic sort, > 48 KB of plan shared
memory, GMAX / ITEM_W item cuts), level id 65535 with doc 0xFFFFFFFF, exact ties and 1-ulp near-ties across levels, full batches, and
the query-shape / k limits.  Ids, ranks, f32 scores and counts are compared with ==.

The branch-evidence tests pin which count branch a one-query, one-level Count batch takes through `last_stats()`: with one record,
lex_count is the only kernel that counts (lex_plan keeps no stats, lex_generic returns at once for <= 4 terms), so
postings_visited, probes and algorithmic_bytes = 4·postings + 16·probes + 128·records + 8·1024·(word-wise lists) are exact."""
import numpy as np
import pytest

from oracle import oracle as O
import helpers_lexlimits as H
from helpers import gpu_index, key_of, oracle_index

pytestmark = pytest.mark.gpu


def _uniq(keys):
    return list(dict.fromkeys(keys))


def _compare(ix, orc, qkeys, is_and, k, mode, not_keys=None):
    from seekstorm_b200 import QueryType, ResultType
    qt, oqt = (QueryType.Intersection, O.QUERY_INTERSECTION) if is_and else (QueryType.Union, O.QUERY_UNION)
    rt, ort = {"topk": (ResultType.Topk, O.RESULT_TOPK), "topkcount": (ResultType.TopkCount, O.RESULT_TOPKCOUNT),
               "count": (ResultType.Count, O.RESULT_COUNT)}[mode]
    kk = 0 if mode == "count" else k
    got, counts = ix.search_lexical_batch(qkeys, qt, kk, rt, not_keys=not_keys)
    for i, kq in enumerate(qkeys):
        want, tot = orc.search(_uniq(kq), oqt, kk, ort, not_keys=not_keys[i] if not_keys else None)
        if mode != "count":
            assert got[i] == want, (i, is_and, k, mode, got[i][:4], want[:4])
        else:
            assert got[i] == []
        if mode != "topk":
            assert int(counts[i]) == tot, (i, is_and, mode, int(counts[i]), tot)
    return got, counts


def _all_modes(ix, orc, qkeys, ks=(10,), not_keys=None):
    for is_and in (False, True):
        for k in ks:
            _compare(ix, orc, qkeys, is_and, k, "topk", not_keys)
        _compare(ix, orc, qkeys, is_and, ks[-1], "topkcount", not_keys)
        _compare(ix, orc, qkeys, is_and, 0, "count", not_keys)


class Corpus:
    def __init__(self, levels, n_docs, len_sum, **kw):
        self.levels, self.n_docs, self.len_sum = levels, n_docs, len_sum
        self.orc = oracle_index(levels, n_docs, len_sum)
        self.ix = gpu_index(levels, n_docs, len_sum, **kw)


@pytest.fixture(scope="module")
def cutover():
    levels, n_docs, len_sum, lists = H.cutover_corpus()
    c = Corpus(levels, n_docs, len_sum)
    c.lists = lists
    yield c
    c.ix.close()


@pytest.fixture(scope="module")
def mixed40():
    c = Corpus(*H.mixed_levels(40, 11))
    yield c
    c.ix.close()


# ---------------------------------------------------------------- 1. list-length cut-overs in one level
def test_cutover_parity(cutover):
    qk = [H.keys(q) for q in H.cutover_queries()]
    _all_modes(cutover.ix, cutover.orc, qk, ks=(1, 10, 32))


def test_cutover_not_terms_and_delete_set(cutover):
    qs = H.cutover_queries()
    nots_cycle = [["n50"], ["n300"], ["n3000"], ["n50", "n300", "n3000", "c129"], ["c2048"], []]      # 4 NOT terms are accepted
    qk = [H.keys(q) for q in qs]
    nk = [H.keys(nots_cycle[i % len(nots_cycle)]) for i in range(len(qs))]
    _all_modes(cutover.ix, cutover.orc, qk, ks=(10,), not_keys=nk)
    # a delete set on the edge ids and on docs of every list: lex_del_count corrects the word-wise counts
    rng = np.random.default_rng(3)
    dele = {0, 64, 65535} | {int(d) for t in ("c128", "c2048", "c2049", "r1025") for d in rng.choice(cutover.lists[t], 40, replace=False)}
    levels = cutover.levels
    ix = gpu_index(levels, cutover.n_docs, cutover.len_sum)
    orc = oracle_index(levels, cutover.n_docs, cutover.len_sum)
    ix.set_deleted(sorted(dele))
    orc.set_deleted(sorted(dele))
    _all_modes(ix, orc, qk, ks=(10, 32))
    _all_modes(ix, orc, qk, ks=(10,), not_keys=nk)
    ix.close()


# ---------------------------------------------------------------- 2. branch evidence: which count branch ran
def _and_branch(a, b):
    if a >= H.UNION_WORDS:
        return "words"
    return "stream" if b <= H.AND_RATIO * a else "probe"


BRANCH_CASES = [
    # (is_and, terms, expected branch)
    (True, ["c2048", "c2049"], "words"),
    (True, ["c2048", "c16384"], "words"),
    (True, ["c2047", "c2048"], "stream"),
    (True, ["c2047", "c4000"], "stream"),
    (True, ["c2047", "c16384"], "probe"),                      # 16384 > 8 * 2047
    (True, ["r128", "r1024"], "stream"),
    (True, ["r128", "r1025"], "probe"),
    (True, ["r200", "r1600"], "stream"),
    (True, ["r200", "r1601"], "probe"),
    (True, ["c127", "c2049"], "probe"),
    (False, ["c2047", "c2048"], None),
    (False, ["c2048", "c2049"], None),
    (False, ["c127", "c128", "c129"], None),
    (False, ["c127", "c2047", "c2048", "c16384"], None),
]


@pytest.mark.parametrize("is_and,terms,branch", BRANCH_CASES)
def test_count_branch_evidence(cutover, is_and, terms, branch):
    from seekstorm_b200 import QueryType, ResultType
    n = [H.CUTOVER_LISTS[t] for t in terms]
    if is_and:
        a, b = sorted(n)[:2]
        assert _and_branch(a, b) == branch
        visited = {"words": 0, "stream": a + b, "probe": a}[branch]
        probes = a if branch == "probe" else 0                   # two lists: every posting of A probes B once
        words = len(n) if branch == "words" else 0
    else:
        visited = sum(c for c in n if c < H.UNION_WORDS)
        probes = 0
        words = sum(1 for c in n if c >= H.UNION_WORDS)
    qt = QueryType.Intersection if is_and else QueryType.Union
    _, counts = cutover.ix.search_lexical_batch([H.keys(terms)], qt, 0, ResultType.Count)
    st = cutover.ix.last_stats()
    _, tot = cutover.orc.search(H.keys(terms), O.QUERY_INTERSECTION if is_and else O.QUERY_UNION, 0, O.RESULT_COUNT)
    assert int(counts[0]) == tot
    assert (st["postings_visited"], st["probes"]) == (visited, probes), (terms, st)
    assert st["algorithmic_bytes"] == 4 * visited + 16 * probes + 128 * 1 + 8 * 1024 * words, (terms, st)


FACET_CASES = [
    # (is_and, terms, not terms)
    (False, ["c127", "c128", "c2048"], []),
    (False, ["c127", "c129"], ["n300"]),
    (False, ["c2047", "c127"], ["n50", "n3000"]),
    (True, ["c128", "c2048"], []),
    (True, ["c127", "c2048"], ["n300"]),
    (True, ["c129", "c4000", "c16384"], ["n50"]),
]


@pytest.fixture(scope="module")
def facet_ix(cutover):
    ix = gpu_index(cutover.levels, cutover.n_docs, cutover.len_sum)
    ix.set_facets({"v": (np.arange(65536) % 5).astype(np.uint16)})
    yield ix
    ix.close()


@pytest.mark.parametrize("is_and,terms,nots", FACET_CASES)
def test_facet_pass_bytes(cutover, facet_ix, is_and, terms, nots):
    """lex_facets reads a list with a bitmap (>= DENSE_MIN postings) as its 1024 words, a shorter one as postings; AND is driven by the
    shortest list (all bitmaps: word AND of every list).  algorithmic_bytes = 4·postings + 8·words + 8·(counted docs)·(requests)."""
    from seekstorm_b200 import QueryFacet, QueryType
    n = [H.CUTOVER_LISTS[t] for t in terms]
    post = words = 0
    if is_and:
        a = min(n)
        if a >= H.DENSE_MIN:
            words += 1024 * len(n)
        else:
            post += a
    else:
        for c in n:
            if c >= H.DENSE_MIN:
                words += 1024
            else:
                post += c
    for t in nots:
        c = H.CUTOVER_LISTS[t]
        if c >= H.DENSE_MIN:
            words += 1024
        else:
            post += c
    _, tot = cutover.orc.search(H.keys(terms), O.QUERY_INTERSECTION if is_and else O.QUERY_UNION, 0, O.RESULT_COUNT,
                                not_keys=H.keys(nots) or None)
    raw = facet_ix.search_lexical_facets([H.keys(terms)], QueryType.Intersection if is_and else QueryType.Union,
                                         [QueryFacet("v", ranges=[("all", 0)])], not_keys=[H.keys(nots)])
    assert raw[0]["v"] == [tot]
    st = facet_ix.last_stats()
    assert st["algorithmic_bytes"] == 4 * post + 8 * words + 8 * tot, (terms, nots, st)


# ---------------------------------------------------------------- 3. many-level plans
def test_many_levels_mixed_sizes(mixed40):
    qk = [H.keys(q) for q in H.random_queries(120, 10, 12)]
    qk[0] = H.keys(["t0", "t7"])                  # the 1-doc level's only doc, and lists of every size
    _all_modes(mixed40.ix, mixed40.orc, qk, ks=(1, 10, 32))


def test_doc_0xffffffff(mixed40):
    """level 65535, local doc 65535: the packed key's low word is 0 for this doc"""
    from seekstorm_b200 import QueryType, ResultType
    last = mixed40.levels[-1]
    offs = last["posting_offsets"]
    found = 0
    for i, kk in enumerate(last["term_keys"]):
        ids = last["doc_ids"][offs[i]:offs[i + 1]]
        if 65535 not in set(int(d) for d in ids):
            continue
        qk = [[int(kk)]]
        df = mixed40.orc.df(int(kk))
        got, counts = mixed40.ix.search_lexical_batch(qk, QueryType.Union, 1024, ResultType.TopkCount)
        want, tot = mixed40.orc.search(qk[0], O.QUERY_UNION, 1024, O.RESULT_TOPKCOUNT)
        assert got[0] == want and int(counts[0]) == tot == df
        found += 1
    assert found >= 2
    # a query whose only match is doc 0xFFFFFFFF: AND of two lists that share just that doc
    lists = {int(kk): set(int(d) for d in last["doc_ids"][offs[i]:offs[i + 1]]) for i, kk in enumerate(last["term_keys"])}
    pairs = [(a, b) for a in lists for b in lists if a < b and 65535 in lists[a] & lists[b]]
    assert pairs
    for a, b in pairs[:4]:
        for k in (1, 32):
            got, counts = mixed40.ix.search_lexical_batch([[a, b]], QueryType.Intersection, k, ResultType.TopkCount)
            want, tot = mixed40.orc.search([a, b], O.QUERY_INTERSECTION, k, O.RESULT_TOPKCOUNT)
            assert got[0] == want and int(counts[0]) == tot
            if tot <= k:
                assert 0xFFFFFFFF in [d for d, _ in got[0]]


@pytest.mark.parametrize("n_levels", [3, 129, 2049, 4096])
def test_many_small_levels(n_levels):
    from seekstorm_b200 import SsbError
    levels, n_docs, len_sum = H.small_levels(n_levels, 1000 + n_levels)
    c = Corpus(levels, n_docs, len_sum)
    qk = [H.keys(q) for q in H.random_queries(100, 6, 7 + n_levels, prefix="s")]
    _all_modes(c.ix, c.orc, qk, ks=(1, 10, 32))
    c.ix.close()
    if n_levels == H.MAX_LEVELS:
        from seekstorm_b200 import Index
        ix = Index(0)
        for lv in levels:
            ix.add_lexical_level(lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"],
                                 lv["doc_len_bytes"])
        extra = H.build_level(65535, 10, {"s0": np.arange(10)}, np.zeros(10, np.uint8))
        with pytest.raises(SsbError, match="error -5"):          # SSB_E_UNSUPPORTED
            ix.add_lexical_level(extra["level_id"], extra["n_docs"], extra["term_keys"], extra["posting_offsets"], extra["doc_ids"],
                                 extra["tfs"], extra["doc_len_bytes"])
        ix.close()


# ---------------------------------------------------------------- 4. ties across levels
def test_exact_ties_across_levels():
    levels, n_docs, len_sum = H.tie_levels()
    c = Corpus(levels, n_docs, len_sum)
    for k in (1, 10, 32, 33, 100):
        got, _ = _compare(c.ix, c.orc, [H.keys(["all"])], False, k, "topkcount")
        assert [d for d, _ in got[0]] == list(range(k))              # the k smallest doc ids, whatever order the levels are visited in
        _compare(c.ix, c.orc, [H.keys(["all"])], True, k, "topk")
    # "lift" raises a few docs of the last two levels: θ is first set there (high doc ids, equal scores of "all" behind them);
    # equal-score docs of the earlier levels must still enter — only strictly smaller bounds prune
    for k in (1, 6, 7, 10, 32):
        for is_and in (False, True):
            _compare(c.ix, c.orc, [H.keys(["all", "lift"]), H.keys(["lift", "all"])], is_and, k, "topkcount")
    got, _ = _compare(c.ix, c.orc, [H.keys(["all", "lift"])], False, 10, "topk")
    assert [d for d, _ in got[0][6:]] == [0, 1, 2, 3]
    c.ix.close()


def test_near_ties_across_levels():
    levels, n_docs, len_sum, near = H.near_tie_levels()
    c = Corpus(levels, n_docs, len_sum)
    qs = [H.keys(["a", "b", "c"]), H.keys(["c", "b", "a"]), H.keys(["a", "b", "c", "missing-term"])]
    for k in range(1, len(near) + 2):                                 # the k-th place at every position of the near-tie group
        for is_and in (False, True):
            _compare(c.ix, c.orc, qs, is_and, k, "topk")
    _compare(c.ix, c.orc, qs, False, 32, "topkcount")
    c.ix.close()


# ---------------------------------------------------------------- 5. batches
def test_full_batch_4096(mixed40):
    qk = [H.keys(q) for q in H.random_queries(4096, 10, 99)]
    from seekstorm_b200 import QueryType, ResultType
    for is_and in (False, True):
        got, counts = _compare(mixed40.ix, mixed40.orc, qk, is_and, 10, "topkcount")
        qt = QueryType.Intersection if is_and else QueryType.Union
        for s in (0, 2040, 4080):                                     # a 16-query slice gives the full batch's results
            part, pc = mixed40.ix.search_lexical_batch(qk[s:s + 16], qt, 10, ResultType.TopkCount)
            assert part == got[s:s + 16] and list(pc) == list(counts[s:s + 16])


def test_batch_above_max_batch(mixed40):
    """1000 queries on an index built for 256: the workspace grows to the batch"""
    from seekstorm_b200 import QueryType, ResultType
    c = gpu_index(mixed40.levels, mixed40.n_docs, mixed40.len_sum, max_batch=256)
    qk = [H.keys(q) for q in H.random_queries(1000, 10, 98)]
    for is_and in (False, True):
        qt = QueryType.Intersection if is_and else QueryType.Union
        got, counts = _compare(c, mixed40.orc, qk, is_and, 32, "topkcount")
        full, fc = mixed40.ix.search_lexical_batch(qk, qt, 32, ResultType.TopkCount)
        assert full == got and list(fc) == list(counts)
        part, pc = c.search_lexical_batch(qk[500:516], qt, 32, ResultType.TopkCount)
        assert part == got[500:516] and list(pc) == list(counts[500:516])
    c.close()


# ---------------------------------------------------------------- 6. query shape and k
def test_duplicate_keys(cutover):
    from seekstorm_b200 import QueryType, ResultType
    a, b, cc = key_of("c2048"), key_of("c129"), key_of("r1025")
    dup = [[a, a, b], [a, a], [b, a, b, a], [cc, a, cc, b, cc]]
    for qt in (QueryType.Union, QueryType.Intersection):
        got, counts = cutover.ix.search_lexical_batch(dup, qt, 32, ResultType.TopkCount)
        want, wc = cutover.ix.search_lexical_batch([_uniq(q) for q in dup], qt, 32, ResultType.TopkCount)
        assert got == want and list(counts) == list(wc)
    _all_modes(cutover.ix, cutover.orc, dup, ks=(10,))


def test_term_and_not_limits(cutover):
    from seekstorm_b200 import QueryType, ResultType, SsbError
    real = [key_of(t) for t in sorted(H.CUTOVER_LISTS)]                               # 17 lists
    q32 = real + [key_of(f"missing-{i}") for i in range(32 - len(real))]
    assert len(set(q32)) == 32
    _compare(cutover.ix, cutover.orc, [q32, q32[::-1]], False, 10, "topkcount")       # OR drops unknown terms
    _compare(cutover.ix, cutover.orc, [real[:12] + real[:12]], True, 10, "topkcount")  # 24 keys, 12 unique: AND
    with pytest.raises(SsbError):
        cutover.ix.search_lexical_batch([q32 + [key_of("missing-x")]], QueryType.Union, 10, ResultType.TopkCount)
    nots = H.keys(["n50", "n300", "n3000", "c129"])
    _compare(cutover.ix, cutover.orc, [H.keys(["c2048", "c16384"])], False, 10, "topkcount", not_keys=[nots])
    with pytest.raises(SsbError, match="error -5"):
        cutover.ix.search_lexical_batch([H.keys(["c2048"])], QueryType.Union, 10, ResultType.TopkCount, not_keys=[nots + [key_of("c127")]])


def test_k_limits(cutover):
    from seekstorm_b200 import QueryType, ResultType, SsbError
    qk = [H.keys(["c16384"]), H.keys(["c4000", "c2049", "c127"]), H.keys(["c127", "c128"]), H.keys(["r128", "r1025"])]
    for k in (32, 33, 1024):
        for is_and in (False, True):
            got, _ = _compare(cutover.ix, cutover.orc, qk, is_and, k, "topkcount")
            if k == 1024:
                assert len(got[0]) == 1024                                   # a full page ...
                assert not is_and or len(got[2]) < 1024                     # ... and a query with fewer matches than k
    with pytest.raises(SsbError):
        cutover.ix.search_lexical_batch(qk, QueryType.Union, 1025, ResultType.Topk)
