"""GPU: the C-ABI surface beyond plain search — stats, caller-owned streams, device pointers, raw buffers,
kernel selection, the mirrored Search::search in Vector / Hybrid mode, re-commit after adding levels."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from seekstorm_b200 import synth
from helpers import gpu_index, oracle_index, query_keys, synth_levels

pytestmark = pytest.mark.gpu


def test_stats_and_kernel_selection():
    from seekstorm_b200 import Index, VectorSimilarity
    rows = synth.gen_vectors(70000, 64, 1, "cpu").numpy()
    q = synth.gen_vectors(50, 64, 2, "cpu").numpy()
    ix = Index(0, vector_dims=64, vector_similarity=VectorSimilarity.Dot)
    ix.add_vectors(rows)
    outs = {}
    for kern in (1, 2, 3, 4, 5, 0):
        ix.set_vector_kernel(kern)
        outs[kern] = ix.search_vector_batch(q, 10)
        st = ix.last_stats()
        assert st["kernel_launches"] == {1: 5, 2: 6, 3: 6, 4: 5, 5: 5, 0: 8}[kern]   # FP32: prep + sample(scan, kth) + scan + merge; tf32: prep + split + sample(scan, kth) + scan + merge; bf16: fused prep/split + sample(scan, kth) + scan + merge; AUTO (50 queries) -> filter scan: + refine + fallback scan / merge (both exit at once)
        assert st["dominant_kernel_ns"] > 0
        assert st["h2d_bytes"] == 50 * 64 * 4 and st["d2h_bytes"] == 50 * 32 * 8
        passes = {1: 4, 2: 1, 3: 1, 4: 1, 5: 1, 0: 1}[kern]   # 50 queries: 4 x 16, 1 x 128, 1 x 64, AUTO -> tensor-core scan
        assert st["algorithmic_bytes"] == passes * 70000 * 64 * 4
    for kern in (2, 3, 4, 5, 0):                            # all kernels agree on the ids (scores within tolerance)
        for a, b in zip(outs[1], outs[kern]):
            assert [d for d, _ in a] == [d for d, _ in b]
            assert np.allclose([s for _, s in a], [s for _, s in b], rtol=1e-4, atol=1e-6)
    with pytest.raises(Exception):
        ix.set_vector_kernel(11)
    ix.close()


def test_caller_stream_and_device_queries():
    """ssb_set_stream: library work ordered on a torch stream; queries and key outputs as device pointers."""
    from seekstorm_b200 import Index, VectorSimilarity
    rows = synth.gen_vectors(20000, 96, 3, "cuda")
    q = synth.gen_vectors(24, 96, 4, "cuda")
    ix = Index(0, vector_dims=96, vector_similarity=VectorSimilarity.Cosine)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        ix.set_stream(st.cuda_stream)
        ix.add_vectors(rows)
        keys = torch.zeros((24, 32), dtype=torch.int64, device="cuda")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ix.search_vector_keys(q, 10, keys)
        e1.record()
        st.synchronize()
        assert e0.elapsed_time(e1) > 0
        got = ix.merge_keys(keys.unsqueeze(0).contiguous(), 1, 24, 10)
    ix.set_stream(None)
    want = ix.search_vector_batch(q.cpu().numpy(), 10)
    assert got == want
    hits, nh = ix.hits_buffer(24 * 10), np.zeros(24, dtype=np.uint32)
    ix.search_vector_raw(q, 10, hits, nh)                                   # device queries, host outputs
    assert (nh == 10).all() and [int(d) for d in hits["doc_id"][:10]] == [d for d, _ in want[0]]
    ix.close()


def test_search_mirror_vector_hybrid_and_paging():
    """Index.search (Search::search signature): Vector and Hybrid modes, offset/length, unsupported args raise."""
    from seekstorm_b200 import Index, QueryType, ResultType, SearchMode, VectorSimilarity
    n = 66000
    lvs, ls = synth_levels(n, 3000, 21)
    orc = oracle_index([l.to_numpy() for l in lvs], n, ls)
    rows = synth.gen_vectors(n, 48, 22, "cpu").numpy()
    ix = Index(0, vector_dims=48, vector_similarity=VectorSimilarity.Cosine)
    for l in lvs:
        ix.add_synth_level(l)
    ix.commit(n, ls)
    ix.add_vectors(rows)
    qv = synth.gen_vectors(1, 48, 23, "cpu").numpy()[0]
    terms = [30, 700]
    qk = query_keys([terms])[0]
    qs = " ".join(f"t{t}" for t in terms)
    nrows = np.stack([O.normalize(r) for r in rows])
    vec = O.search_vector(nrows, O.normalize(qv), 12, O.SIM_COSINE)
    lex, tot = orc.search(qk, O.QUERY_UNION, 12, O.RESULT_TOPKCOUNT)
    ro = ix.search(qs, list(qv), QueryType.Union, SearchMode.Vector(), False, 2, 10, ResultType.TopkCount)
    assert [r.doc_id for r in ro.results] == [d for d, _ in vec[2:12]] and ro.result_count == 10
    assert ro.observed_vector_count == n
    ro = ix.search(qs, None, QueryType.Union, SearchMode.Lexical(), False, 2, 10, ResultType.TopkCount)
    assert [(r.doc_id, np.float32(r.score)) for r in ro.results] == [(d, np.float32(s)) for d, s in lex[2:12]]
    assert ro.result_count_total == tot
    ro = ix.search(qs, list(qv), QueryType.Union, SearchMode.Hybrid(), False, 0, 10, ResultType.Topk)
    lex10, _ = orc.search(qk, O.QUERY_UNION, 10, O.RESULT_TOPK)
    want = O.rrf(lex10, vec[:10])[:10]
    assert [r.doc_id for r in ro.results] == [d for d, _ in want]
    ro = ix.search("+t30 +t700", None, QueryType.Union, SearchMode.Lexical(), False, 0, 10, ResultType.TopkCount)
    a, ta = orc.search(qk, O.QUERY_INTERSECTION, 10, O.RESULT_TOPKCOUNT)           # '+' on every term -> Intersection
    assert [r.doc_id for r in ro.results] == [d for d, _ in a] and ro.result_count_total == ta
    ro = ix.search("t30", None, QueryType.Union, SearchMode.Lexical(), False, 0, 0, ResultType.TopkCount)
    assert ro.results == [] and ro.result_count_total == orc.search(qk[:1], O.QUERY_UNION, 0, O.RESULT_COUNT)[1]   # length 0 -> Count
    ro = ix.search("unknownterm", None, QueryType.Union, SearchMode.Lexical(), False, 0, 10, ResultType.TopkCount)
    assert ro.results == [] and ro.result_count_total == 0                          # infallible: empty ResultObject
    with pytest.raises(ValueError):                       # field_filter names a field the (single-field) index does not have
        ix.search(qs, None, QueryType.Union, SearchMode.Lexical(), False, 0, 10, ResultType.Topk, field_filter=["body"])
    with pytest.raises(NotImplementedError):              # facet COUNTING stays outside the GPU hot path
        ix.search(qs, None, QueryType.Union, SearchMode.Lexical(), False, 0, 10, ResultType.Topk, query_facets=["price"])
    from seekstorm_b200 import SsbError
    with pytest.raises(SsbError):                         # a phrase query needs levels loaded with positions
        ix.search('"t30 t700"', None, QueryType.Union, SearchMode.Lexical(), False, 0, 10, ResultType.Topk)
    ix.close()


def test_incremental_levels_recommit():
    """Levels are immutable; adding one and committing again (new N / avgdl) must equal a fresh build."""
    from seekstorm_b200 import QueryType, ResultType
    lvs, ls = synth_levels(140000, 4000, 31)          # 3 levels
    part = lvs[:2]
    n_part = sum(l.n_docs for l in part)
    ls_part = sum(l.len_sum_normalized for l in part)
    ix = gpu_index([l.to_numpy() for l in part], n_part, ls_part)
    qk = query_keys(synth.gen_queries(40, 32, 3, 3000, (2, 3), (0.5, 0.5)))
    o1 = oracle_index([l.to_numpy() for l in part], n_part, ls_part)
    got, cnt = ix.search_lexical_batch(qk, QueryType.Union, 10, ResultType.TopkCount)
    for i, k in enumerate(qk):
        assert (got[i], int(cnt[i])) == o1.search(k, O.QUERY_UNION, 10, O.RESULT_TOPKCOUNT)
    ix.add_synth_level(lvs[2])
    ix.commit(140000, ls)
    o2 = oracle_index([l.to_numpy() for l in lvs], 140000, ls)
    got, cnt = ix.search_lexical_batch(qk, QueryType.Union, 10, ResultType.TopkCount)
    for i, k in enumerate(qk):
        assert (got[i], int(cnt[i])) == o2.search(k, O.QUERY_UNION, 10, O.RESULT_TOPKCOUNT)
    ix.close()


def test_many_term_queries_generic_path():
    """> 4 live terms take the shuffle-broadcast generic path (up to SSB_MAX_QUERY_TERMS = 32, one term per lane)."""
    from seekstorm_b200 import QueryType, ResultType, SsbError
    lvs, ls = synth_levels(80000, 2000, 41)
    orc = oracle_index([l.to_numpy() for l in lvs], 80000, ls)
    ix = gpu_index([l.to_numpy() for l in lvs], 80000, ls)
    qs = synth.gen_queries(30, 42, 2, 1800, (5, 8, 12, 24, 32), (0.3, 0.3, 0.2, 0.1, 0.1))
    qk = query_keys(qs)
    got, cnt = ix.search_lexical_batch(qk, QueryType.Union, 10, ResultType.TopkCount)
    for i, k in enumerate(qk):
        want, tot = orc.search(k, O.QUERY_UNION, 10, O.RESULT_TOPKCOUNT)
        assert [d for d, _ in got[i]] == [d for d, _ in want] and int(cnt[i]) == tot
        assert np.allclose([s for _, s in got[i]], [s for _, s in want], rtol=1e-6)     # same query-order sums
    got, cnt = ix.search_lexical_batch(qk[:10], QueryType.Intersection, 10, ResultType.TopkCount)
    for i, k in enumerate(qk[:10]):
        want, tot = orc.search(k, O.QUERY_INTERSECTION, 10, O.RESULT_TOPKCOUNT)
        assert got[i] == want and int(cnt[i]) == tot
    with pytest.raises(SsbError):
        ix.search_lexical_batch([list(range(33))], QueryType.Union, 10, ResultType.Topk)
    ix.close()


def test_add_level_rejects_malformed_postings():
    """Input contract of ssb_lexical_add_level is validated on the device (status code, not UB)."""
    from seekstorm_b200 import Index, SsbError
    from helpers import level_from_postings
    ix = Index(0)
    good = level_from_postings(0, 50, {"a": [(1, 1), (5, 2), (9, 1)], "b": [(5, 3)]}, [10] * 50)
    for bad_post in ({"a": [(5, 1), (1, 2)]},            # ids not ascending
                     {"a": [(3, 1), (3, 1)]},            # duplicate id
                     {"a": [(60, 1)]},                   # id >= n_docs
                     {"a": [(2, 0)]}):                   # tf = 0
        lv = level_from_postings(0, 50, bad_post, [10] * 50)
        with pytest.raises(SsbError, match="malformed"):
            ix.add_lexical_level(lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"], lv["doc_len_bytes"])
    ix.add_lexical_level(good["level_id"], good["n_docs"], good["term_keys"], good["posting_offsets"], good["doc_ids"], good["tfs"], good["doc_len_bytes"])
    ix.commit(50, 500)
    ix.close()


@pytest.mark.parametrize("kern", [1, 2, 4])
def test_vector_paging_beyond_32(kern):
    """offset+length > 32 (the reference's heap is min(offset+length, N), search.rs:2527-2531): the host-facing call pages
    internally with an exclusive key ceiling; results must equal the oracle's top-k for k = 100 and k = N."""
    from seekstorm_b200 import Index, VectorSimilarity
    rows = synth.gen_vectors(70000, 64, 51, "cpu").numpy()
    q = synth.gen_vectors(20, 64, 52, "cpu").numpy()
    rows[7] = rows[3]                                       # exact duplicate rows: tie broken by doc id across pages
    ix = Index(0, vector_dims=64, vector_similarity=VectorSimilarity.Dot, vector_kernel=kern)
    ix.add_vectors(rows)
    got = ix.search_vector_batch(q, 100)
    for i in (0, 7, 19):
        want = O.search_vector(rows, q[i], 100, O.SIM_DOT)
        assert len(got[i]) == 100
        assert [d for d, _ in got[i]] == [d for d, _ in want]
        assert np.allclose([s for _, s in got[i]], [s for _, s in want], rtol=1e-4, atol=1e-5)
    small = Index(0, vector_dims=64, vector_similarity=VectorSimilarity.Dot, vector_kernel=kern)
    small.add_vectors(rows[:50])
    got = small.search_vector_batch(q[:3], 80)              # fewer rows than k: every row, best first, then stop
    for i in range(3):
        want = O.search_vector(rows[:50], q[i], 80, O.SIM_DOT)
        assert [d for d, _ in got[i]] == [d for d, _ in want] and len(got[i]) == 50
    ix.close(); small.close()


def test_lexical_paging_beyond_32():
    from seekstorm_b200 import QueryType, ResultType, SearchMode
    lvs, ls = synth_levels(90000, 1500, 61)
    orc = oracle_index([l.to_numpy() for l in lvs], 90000, ls)
    ix = gpu_index([l.to_numpy() for l in lvs], 90000, ls)
    qs = synth.gen_queries(25, 62, 2, 1400, (1, 2, 3), (0.2, 0.5, 0.3))
    qk = query_keys(qs)
    for qt, oqt in ((QueryType.Union, O.QUERY_UNION), (QueryType.Intersection, O.QUERY_INTERSECTION)):
        got, cnt = ix.search_lexical_batch(qk, qt, 77, ResultType.TopkCount)
        for i, k in enumerate(qk):
            want, tot = orc.search(k, oqt, 77, O.RESULT_TOPKCOUNT)
            assert got[i] == want, (qt, i)                 # bit-exact across page boundaries (ties by doc id)
            assert int(cnt[i]) == tot
    # the mirrored Search::search with offset paging past 32
    terms = qs[0]
    ro = ix.search(" ".join(f"t{t}" for t in terms), None, QueryType.Union, SearchMode.Lexical(), False, 40, 10, ResultType.TopkCount)
    want, tot = orc.search(qk[0], O.QUERY_UNION, 50, O.RESULT_TOPKCOUNT)
    assert [(r.doc_id, np.float32(r.score)) for r in ro.results] == [(d, np.float32(s)) for d, s in want[40:50]]
    assert ro.result_count_total == tot
    ix.close()


def test_search_vector_ex_threshold_int8_and_ext():
    """ssb_search_vector_ex: similarity_threshold pre-map (vector.rs:388-399), vb fields / post-map (vector.rs:1485-1503),
    observed_vector_count, int8 query codes for a ScalarQuantizationI8 index."""
    from seekstorm_b200 import Index, VectorSimilarity
    n, dims = 30000, 64
    rows = synth.gen_vectors(n, dims, 91, "cpu").numpy()
    qs = synth.gen_vectors(6, dims, 92, "cpu").numpy()
    qs[1] = rows[777] + 0.01 * qs[1]
    ix = Index(0, vector_dims=dims, vector_similarity=VectorSimilarity.Cosine)
    ix.add_vectors(rows)
    nrows = np.stack([O.normalize(r) for r in rows])
    t = 0.50002                                            # cut = (2t-1)*16129 ~ 0.645: only the planted neighbour passes
    cut = np.float32((np.float32(t) * np.float32(2.0) - np.float32(1.0)) / np.float32(1.0 / 16129.0))
    got, ext, observed = ix.search_vector_ex(qs, 10, similarity_threshold=t)
    for i in range(len(qs)):
        want = [(d, s) for d, s in O.search_vector(nrows, O.normalize(qs[i]), 10, O.SIM_COSINE) if not (np.float32(s) < cut)]
        assert [d for d, _ in got[i]] == [d for d, _ in want]
        assert int(observed[i]) == n
        for j, (d, s) in enumerate(got[i]):
            e = ext[i * 10 + j]
            assert e.level_id == d >> 16 and e.source == 1
            assert abs(e.vector_score - O.lib().orc_vector_score_postmap(np.float32(s), O.SIM_COSINE)) < 1e-6
    assert [d for d, _ in got[1]] == [777]
    no_thr, _, _ = ix.search_vector_ex(qs, 10)
    assert no_thr == ix.search_vector_batch(qs, 10)
    ix.close()
    # int8 query codes == f32 queries quantised by the library
    ix8 = Index(0, vector_dims=dims, vector_similarity=VectorSimilarity.Cosine, vector_quantization=1)
    ix8.add_vectors(rows)
    q8 = O.quantize_rows_i8(qs)
    a, _, _ = ix8.search_vector_ex(q8, 10, int8_queries=True)
    assert a == ix8.search_vector_batch(qs, 10)
    ix8.close()


def test_vector_multi_chunk_documents_are_deduplicated():
    """Several rows with one doc id (one vector per chunk): the best chunk per doc is returned once (TopK::push, vector.rs:436-470),
    through paging, hybrid and the k <= 32 path."""
    from seekstorm_b200 import Index, VectorSimilarity
    dims, n_docs, chunks = 32, 500, 6
    rng = np.random.default_rng(5)
    rows = rng.normal(size=(n_docs * chunks, dims)).astype(np.float32)
    ids = np.repeat(np.arange(n_docs, dtype=np.uint16), chunks)
    ix = Index(0, vector_dims=dims, vector_similarity=VectorSimilarity.Dot)
    ix.add_vector_level(3, rows, ids)
    qs = rng.normal(size=(5, dims)).astype(np.float32)
    for k in (10, 32, 100):
        got = ix.search_vector_batch(qs, k)
        sc = rows @ qs.T                                                          # [rows, nq] (score tolerance 1e-4 below)
        for i in range(len(qs)):
            best = sc[:, i].reshape(n_docs, chunks).max(axis=1)
            order = np.lexsort((np.arange(n_docs), -best))[:k]
            assert [d for d, _ in got[i]] == [(3 << 16) | int(d) for d in order]
            assert np.allclose([s for _, s in got[i]], best[order], rtol=1e-4, atol=1e-5)
    ix.close()


def test_delete_set_lexical_vector_hybrid():
    """ssb_set_deleted (shard.delete_hashset): deleted docs are neither scored nor counted — lexical OR / AND incl. exact counts,
    >4-term queries, vector scan (both kernels), hybrid; clearing the set restores the results."""
    from seekstorm_b200 import Index, QueryType, ResultType, VectorSimilarity
    n, dims = 140000, 48
    lvs, ls = synth_levels(n, 3000, 51)
    levels = [l.to_numpy() for l in lvs]
    orc = oracle_index(levels, n, ls)
    rows = synth.gen_vectors(n, dims, 52, "cpu").numpy()
    ix = gpu_index(levels, n, ls, vector_dims=dims, vector_similarity=VectorSimilarity.Cosine)
    ix.add_vectors(rows)
    qk = query_keys(synth.gen_queries(60, 53, 2, 2500, (1, 2, 3, 4, 6), (0.1, 0.3, 0.3, 0.2, 0.1)))
    qv = synth.gen_vectors(40, dims, 54, "cpu").numpy()
    base_lex, _ = ix.search_lexical_batch(qk, QueryType.Union, 10, ResultType.TopkCount)
    base_vec = ix.search_vector_batch(qv, 10)
    # delete the current top hits of every query (forces new results) plus a random spread over all levels
    rng = np.random.default_rng(55)
    deleted = {d for r in base_lex for d, _ in r[:3]} | {d for r in base_vec for d, _ in r[:2]} | {int(x) for x in rng.integers(0, n, 3000)}
    deleted = {((d >> 16) << 16) | (d & 0xFFFF) for d in deleted}
    ix.set_deleted(sorted(deleted)); orc.set_deleted(sorted(deleted))
    for qt, oqt in ((QueryType.Union, O.QUERY_UNION), (QueryType.Intersection, O.QUERY_INTERSECTION)):
        got, cnt = ix.search_lexical_batch(qk, qt, 10, ResultType.TopkCount)
        got_t, _ = ix.search_lexical_batch(qk, qt, 10, ResultType.Topk)
        for i, k in enumerate(qk):
            want, tot = orc.search(k, oqt, 10, O.RESULT_TOPKCOUNT)
            if len(k) <= 4:
                assert got[i] == want and got_t[i] == want, (i, k)
            else:
                assert [d for d, _ in got[i]] == [d for d, _ in want]
            assert int(cnt[i]) == tot, (i, k, int(cnt[i]), tot)
            assert not any(d in deleted for d, _ in got[i])
    nrows = np.stack([O.normalize(r) for r in rows])
    for kern in (1, 4, 7):
        ix.set_vector_kernel(kern)
        got = ix.search_vector_batch(qv, 10)
        for i in range(len(qv)):
            want = [(d, s) for d, s in O.search_vector(nrows, O.normalize(qv[i]), 10 + len(deleted), O.SIM_COSINE) if d not in deleted][:10]
            assert [d for d, _ in got[i]] == [d for d, _ in want]
    ix.set_vector_kernel(0)
    hyb = ix.search_hybrid_batch(qk[:20], QueryType.Union, qv[:20], 10)
    for i in range(20):
        lex, _ = orc.search(qk[i], O.QUERY_UNION, 10, O.RESULT_TOPK)
        vec = [(d, s) for d, s in O.search_vector(nrows, O.normalize(qv[i]), 10 + len(deleted), O.SIM_COSINE) if d not in deleted][:10]
        assert [d for d, _ in hyb[i]] == [d for d, _ in O.rrf(lex, vec)[:10]]
    ix.set_deleted([])
    again, _ = ix.search_lexical_batch(qk, QueryType.Union, 10, ResultType.TopkCount)
    assert again == base_lex and ix.search_vector_batch(qv, 10) == base_vec
    ix.close()


def test_not_lists_lexical():
    """'-' terms (not_query_list, add_result.rs:3440-3496): docs containing a NOT term are neither scored nor counted — OR / AND,
    exact counts, > 4 positive terms, combined with a delete set, and through the mirrored Search::search ('-t7')."""
    from seekstorm_b200 import QueryType, ResultType, SearchMode
    n = 140000
    lvs, ls = synth_levels(n, 1500, 61)
    levels = [l.to_numpy() for l in lvs]
    orc = oracle_index(levels, n, ls)
    ix = gpu_index(levels, n, ls)
    rng = np.random.default_rng(62)
    qs = synth.gen_queries(50, 63, 2, 1200, (1, 2, 3, 4, 6), (0.1, 0.3, 0.3, 0.2, 0.1))
    qk = query_keys(qs)
    nots_ids = [[int(x) for x in rng.integers(0, 60, int(rng.integers(0, 3)))] for _ in qs]       # frequent terms: real exclusions
    nots_ids = [[t for t in ns if t not in q] for ns, q in zip(nots_ids, qs)]
    nk = query_keys([ns if ns else [0] for ns in nots_ids])
    nk = [k if ns else [] for k, ns in zip(nk, nots_ids)]
    nk[3] = nk[3] + [0xDEAD0008]                                          # unknown NOT term: excludes nothing
    for deleted in ([], [int(x) for x in rng.integers(0, n, 2000)]):
        ix.set_deleted(deleted); orc.set_deleted(deleted)
        for qt, oqt in ((QueryType.Union, O.QUERY_UNION), (QueryType.Intersection, O.QUERY_INTERSECTION)):
            got, cnt = ix.search_lexical_batch(qk, qt, 10, ResultType.TopkCount, not_keys=nk)
            for i, k in enumerate(qk):
                want, tot = orc.search(k, oqt, 10, O.RESULT_TOPKCOUNT, not_keys=nk[i])
                if len(k) <= 4:
                    assert got[i] == want, (i, k, nk[i])
                else:
                    assert [d for d, _ in got[i]] == [d for d, _ in want]
                assert int(cnt[i]) == tot, (i, k, nk[i], int(cnt[i]), tot)
    ix.set_deleted([]); orc.set_deleted([])
    ro = ix.search("t30 t700 -t5", None, QueryType.Union, SearchMode.Lexical(), False, 0, 10, ResultType.TopkCount)
    k3 = query_keys([[30, 700], [5]])
    want, tot = orc.search(k3[0], O.QUERY_UNION, 10, O.RESULT_TOPKCOUNT, not_keys=k3[1])
    assert [(r.doc_id, np.float32(r.score)) for r in ro.results] == [(d, np.float32(s)) for d, s in want] and ro.result_count_total == tot
    ix.close()
