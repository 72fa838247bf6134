"""GPU, BASELINE.json full sizes: C2 (1M x 768 cosine top-10) checked against the oracle on a few queries and by
size-independent properties (planted neighbours, batch-composition invariance, self-match)."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from seekstorm_b200 import synth

pytestmark = pytest.mark.gpu


def test_c2_full_size_vector():
    from seekstorm_b200 import Index, VectorSimilarity
    n, d = 1_000_000, 768
    rows = synth.gen_vectors(n, d, 1002, "cuda")
    ix = Index(0, vector_dims=d, vector_similarity=VectorSimilarity.Cosine)
    ix.add_vectors(rows)
    assert ix.vector_count == n
    q = synth.gen_vectors(48, d, 2002, "cuda")
    planted = torch.arange(0, 48, 3, device="cuda") * 20011 % n
    q[::3] = rows[planted] + 0.05 * q[::3]
    got = ix.search_vector_batch(q.cpu().numpy(), 10)
    # property: planted neighbour is rank 1
    for j, p in enumerate(planted.tolist()):
        assert got[3 * j][0][0] == p
    # property: results do not depend on batch composition / padding.  AUTO switches kernel with the batch size
    # (48 queries -> tensor-core scan, 7 -> FP32 scan): same ids, scores within the 1e-4 tolerance; with the kernel pinned the
    # scores are bit-identical.
    again = ix.search_vector_batch(q[5:12].cpu().numpy(), 10)
    for a_, g_ in zip(again, got[5:12]):
        assert [d for d, _ in a_] == [d for d, _ in g_]
        assert np.allclose([s for _, s in a_], [s for _, s in g_], rtol=1e-4)
    for kern in (1, 2):
        ix.set_vector_kernel(kern)
        full = ix.search_vector_batch(q.cpu().numpy(), 10)
        assert ix.search_vector_batch(q[5:12].cpu().numpy(), 10) == full[5:12]
    # the filter scan (AUTO's choice above 16 queries) against the exact 3-product tensor-core scan: same ids
    ix.set_vector_kernel(4)
    exact = ix.search_vector_batch(q.cpu().numpy(), 10)
    for kern in (7, 8, 9):
        ix.set_vector_kernel(kern)
        filt = ix.search_vector_batch(q.cpu().numpy(), 10)
        st = ix.last_stats()
        assert st["scan_bytes_read"] == n * d * 2 + 48 * 32 * d * 4 and st["filter_fallbacks"] == 0
        for a_, g_ in zip(filt, exact):
            assert [x for x, _ in a_] == [x for x, _ in g_]
            assert np.allclose([s for _, s in a_], [s for _, s in g_], rtol=1e-4)
    ix.set_vector_kernel(0)
    # oracle on 4 queries (multi-threaded exhaustive scan of the normalised corpus)
    nrows = (rows / rows.norm(dim=1, keepdim=True)).cpu().numpy()
    for i in (0, 1, 2, 7):
        want = O.search_vector(nrows, O.normalize(q[i].cpu().numpy()), 10, O.SIM_COSINE, n_threads=16)
        gs = np.array([s for _, s in got[i]]); ws = np.array([s for _, s in want])
        assert np.allclose(gs, ws, rtol=1e-4, atol=1e-6)
        for (gd, gsc), (wd, wsc) in zip(got[i], want):
            assert gd == wd or abs(gsc - wsc) <= 1e-4 * abs(wsc)
    ix.close()


def test_c2_full_size_vector_int8():
    """C2 corpus with Cosine + ScalarQuantizationI8: bit-exact ids and integer scores against the oracle's quantiser +
    an exact CPU scoring (f32 BLAS over int8 values: every partial sum is an integer below 2^24)."""
    from seekstorm_b200 import Index, VectorSimilarity
    n, d = 1_000_000, 768
    rows = synth.gen_vectors(n, d, 1002, "cuda")
    ix = Index(0, vector_dims=d, vector_similarity=VectorSimilarity.Cosine, vector_quantization=1)
    ix.add_vectors(rows)
    assert ix.vector_count == n
    q = synth.gen_vectors(200, d, 2002, "cuda")
    planted = torch.arange(0, 200, 3, device="cuda") * 20011 % n
    q[::3] = rows[planted] + 0.05 * q[::3]
    qh = q.cpu().numpy()
    got = ix.search_vector_batch(qh, 10)
    for j, p in enumerate(planted.tolist()):
        assert got[3 * j][0][0] == p
    assert ix.search_vector_batch(qh[5:12], 10) == got[5:12]        # batch-composition invariance, bit-exact
    rows_h = rows.cpu().numpy()
    r8 = O.quantize_rows_i8(rows_h)
    q8 = O.quantize_rows_i8(qh)
    sel = [0, 1, 2, 7, 100, 199]
    qf = q8[sel].astype(np.float32)
    best = [[] for _ in sel]
    for s in range(0, n, 100_000):
        sc = r8[s:s + 100_000].astype(np.float32) @ qf.T
        for j in range(len(sel)):
            idx = np.argpartition(-sc[:, j], 64)[:64]
            best[j] += [(-float(sc[i, j]), s + int(i)) for i in idx]
    for j, qi in enumerate(sel):
        want = [(doc, -negs) for negs, doc in sorted(best[j])[:10]]
        assert got[qi] == want, (qi, got[qi][:3], want[:3])
    ix.close()


# ---------------------------------------------------------------------------------------------------------------------
# C3 (BM25, 10 M docs) and C4 (hybrid, 5 M docs) at BASELINE.json's full sizes: top-k identity against the exhaustive
# oracle (ids, ranks, scores `==`; counts `==`).  The corpus is generated on the GPU (same seeded law as bench.py),
# handed to the library as device pointers and copied to the host once for the oracle.
def _build_full_lexical(n_docs, seed, want_oracle=True, **index_kw):
    from seekstorm_b200 import Index
    ix = Index(0, max_batch=256, **index_kw)
    orc = O.OracleIndex() if want_oracle else None
    ls = 0
    for lv in synth.gen_lexical_corpus(n_docs, 1_000_000, seed, "cuda"):
        ix.add_synth_level(lv)
        if orc is not None:
            orc.add_level(lv.to_numpy())
        ls += lv.len_sum_normalized
    ix.commit(n_docs, ls)
    if orc is not None:
        orc.commit(n_docs, ls)
    return ix, orc


_c3_open = []   # the module's 10 M-doc index while it is alive


@pytest.fixture(scope="module")
def c3_index():
    ix, orc = _build_full_lexical(10_000_000, 1003)
    _c3_open.append(ix)
    yield ix, orc
    ix.close()


def _c3_queries(n, seed):
    from helpers import query_keys
    return query_keys(synth.gen_queries(n, seed, 20, 100000, (2, 3, 4), (0.4, 0.4, 0.2)))


def test_c3_full_size_or_top10_identity(c3_index):
    """C3: 10 M docs, 64 OR queries of the bench's own law — ids / ranks / scores == exhaustive oracle; TopkCount counts ==."""
    from seekstorm_b200 import QueryType, ResultType
    ix, orc = c3_index
    qk = _c3_queries(64, 2003)                       # the first 64 of the queries bench.py times
    got, _ = ix.search_lexical_batch(qk, QueryType.Union, 10, ResultType.Topk)
    got_c, counts = ix.search_lexical_batch(qk, QueryType.Union, 10, ResultType.TopkCount)
    for i, kq in enumerate(qk):
        want, tot = orc.search(kq, O.QUERY_UNION, 10, O.RESULT_TOPKCOUNT)
        assert len(want) == 10
        assert got[i] == want, (i, kq, got[i], want)          # bit-exact ids, ranks, scores (pruned Topk path)
        assert got_c[i] == want, (i, kq, got_c[i], want)      # and with exact counting switched on
        assert int(counts[i]) == tot, (i, counts[i], tot)


def test_c3_full_size_and_top10_identity(c3_index):
    """C3 corpus, 64 AND queries: ids / ranks / scores / match counts == exhaustive oracle."""
    from seekstorm_b200 import QueryType, ResultType
    ix, orc = c3_index
    qk = _c3_queries(64, 2013)
    got, counts = ix.search_lexical_batch(qk, QueryType.Intersection, 10, ResultType.TopkCount)
    got_t, _ = ix.search_lexical_batch(qk, QueryType.Intersection, 10, ResultType.Topk)
    n_nonempty = 0
    for i, kq in enumerate(qk):
        want, tot = orc.search(kq, O.QUERY_INTERSECTION, 10, O.RESULT_TOPKCOUNT)
        assert got[i] == want, (i, kq, got[i], want)
        assert got_t[i] == want, (i, kq, got_t[i], want)
        assert int(counts[i]) == tot, (i, counts[i], tot)
        n_nonempty += 1 if want else 0
    assert n_nonempty >= 32                                  # the query law produces real intersections at 10 M docs


def test_c3_full_size_batch_invariance_and_paging(c3_index):
    """Size-independent properties at 10 M docs: results do not depend on batch composition; k=100 (paged) extends k=10."""
    from seekstorm_b200 import QueryType, ResultType
    ix, orc = c3_index
    qk = _c3_queries(200, 2023)
    full, _ = ix.search_lexical_batch(qk, QueryType.Union, 10, ResultType.Topk)
    part, _ = ix.search_lexical_batch(qk[37:53], QueryType.Union, 10, ResultType.Topk)
    assert part == full[37:53]
    deep, _ = ix.search_lexical_batch(qk[:8], QueryType.Union, 100, ResultType.Topk)
    for i in range(8):
        assert deep[i][:10] == full[i]
        sc = [s for _, s in deep[i]]
        assert sc == sorted(sc, reverse=True) and len({d for d, _ in deep[i]}) == len(deep[i])
        want, _ = orc.search(qk[i], O.QUERY_UNION, 100, O.RESULT_TOPK)
        assert deep[i] == want


def test_c3_full_size_facet_filter_identity(c3_index):
    """C3 corpus (10 M docs) behind facet filters (a u32 range half of the docs pass + a String16 value set): 32 OR + 32 AND queries, ids / ranks /
    scores / counts == the exhaustive oracle with the same filters (the per-candidate predicate path at BASELINE.json's size)."""
    from seekstorm_b200 import FacetFilter, QueryType, ResultType
    ix, orc = c3_index
    n = 10_000_000
    rng = np.random.default_rng(77)
    cols = {"price": rng.integers(0, 1000, n, dtype=np.uint32), "cat": rng.integers(0, 16, n, dtype=np.uint16)}
    ix.set_facets(cols, string_facets=("cat",))
    rows, fields, first, nd, rb = ix._facet_rows
    orc.set_facets(rows, [(fields[i].type, fields[i].offset) for i in range(2)], first, nd, rb)
    fl = [FacetFilter("price", 250, 750), FacetFilter("cat", values=[1, 3, 5, 7, 9, 11])]
    offs, arr, sv = ix._encode_filters([fl])
    tup = [(arr[i].facet, arr[i].kind, arr[i].start, arr[i].end, arr[i].set_first, arr[i].set_count) for i in range(2)]
    qk = _c3_queries(32, 2033)
    try:
        for qt, oqt in ((QueryType.Union, O.QUERY_UNION), (QueryType.Intersection, O.QUERY_INTERSECTION)):
            got, counts = ix.search_lexical_batch(qk, qt, 10, ResultType.TopkCount, filters=[fl] * len(qk))
            for i, kq in enumerate(qk):
                want, tot = orc.search(kq, oqt, 10, O.RESULT_TOPKCOUNT, filters=tup, set_values=[int(x) for x in sv])
                assert got[i] == want, (qt, i, kq, got[i][:3], want[:3])
                assert int(counts[i]) == tot, (qt, i, counts[i], tot)
                assert all(250 <= cols["price"][(d >> 16) * 65536 + (d & 0xFFFF)] < 750 for d, _ in got[i])
    finally:
        ix.set_facets({})


def test_c4_full_size_hybrid_identity():
    """C4: 5 M docs + 5 M x 768 f32 vectors, 16 hybrid queries: fused ids / RRF scores == O.rrf of the two oracle lists
    (lexical list bit-exact; the vector list is checked to 1e-4 and must agree on ids for the RRF ranks to agree)."""
    from seekstorm_b200 import QueryType, VectorSimilarity
    n, d = 5_000_000, 768
    # an 80 GB GPU holds this index (5 M docs + 5 M x 768 vectors as f32, two bf16 planes and an fp16 plane: 38 GB of vectors) but not
    # next to the C3 index of the tests above, which have run by now: it is released first (its fixture's own close() is then a no-op)
    while _c3_open:
        _c3_open.pop().close()
    ix, orc = _build_full_lexical(n, 1004, vector_dims=d, vector_similarity=VectorSimilarity.Cosine)
    host_rows = np.empty((n, d), dtype=np.float32)
    ix.reserve_vectors(n)
    for lv in range((n + 65535) // 65536):
        r = synth.gen_vectors(min(65536, n - lv * 65536), d, 1005 * 1000 + lv, "cuda")
        ix.add_vector_level(lv, r)
        host_rows[lv * 65536: lv * 65536 + r.shape[0]] = (r / r.norm(dim=1, keepdim=True)).cpu().numpy()
        del r
    qk = _c3_queries(16, 2004)
    qv = synth.gen_vectors(16, d, 2005, "cpu").numpy()
    got = ix.search_hybrid_batch(qk, QueryType.Union, qv, 10)
    lex_got, _ = ix.search_lexical_batch(qk, QueryType.Union, 10)
    vec_got = ix.search_vector_batch(qv, 10)
    for i in range(16):
        lex, _ = orc.search(qk[i], O.QUERY_UNION, 10, O.RESULT_TOPK)
        vec = O.search_vector(host_rows, O.normalize(qv[i]), 10, O.SIM_COSINE, n_threads=32)
        assert lex_got[i] == lex, (i, lex_got[i], lex)
        assert [x for x, _ in vec_got[i]] == [x for x, _ in vec], (i, vec_got[i], vec)
        assert np.allclose([s for _, s in vec_got[i]], [s for _, s in vec], rtol=1e-4, atol=1e-6)
        want = O.rrf(lex, vec)[:10]
        assert [x for x, _ in got[i]] == [x for x, _ in want], (i, got[i], want)
        assert [np.float32(s) for _, s in got[i]] == [np.float32(s) for _, s in want]
    ix.close()
