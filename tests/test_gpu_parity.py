"""GPU parity tests (-m gpu): the CUDA path through the C-ABI vs the CPU oracle on the same seeded inputs.

Bars: bit-exact doc ids / ranks / counts and bit-exact BM25 scores (every f32 op individually rounded on both
sides); cosine / dot / Euclidean scores within 1e-4 relative (different reduction tree)."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from seekstorm_b200 import synth
from helpers import gpu_index, key_of, level_from_postings, oracle_index, query_keys, synth_levels

pytestmark = pytest.mark.gpu

RTOL = 1e-4   # north_star tolerance for floating-point scores


def _check_vec(got, want, strict_ids=True):
    assert len(got) == len(want)
    gs = np.array([s for _, s in got], dtype=np.float64)
    ws = np.array([s for _, s in want], dtype=np.float64)
    assert np.allclose(gs, ws, rtol=RTOL, atol=1e-6), (got, want)
    if [d for d, _ in got] != [d for d, _ in want]:
        # ids may only differ inside a near-tie group (scores closer than the tolerance)
        for (gd, gsc), (wd, wsc) in zip(got, want):
            if gd != wd:
                assert abs(gsc - wsc) <= RTOL * max(abs(wsc), 1e-6), (got, want)


@pytest.mark.parametrize("n,dims,sim", [
    (1, 32, "cos"), (255, 128, "cos"), (257, 128, "dot"), (5000, 100, "cos"), (5000, 768, "cos"),
    (70000, 64, "euc"), (3000, 960, "dot"), (1000, 33, "euc")])
def test_vector_parity_small(n, dims, sim):
    from seekstorm_b200 import Index, VectorSimilarity
    simv = {"cos": VectorSimilarity.Cosine, "dot": VectorSimilarity.Dot, "euc": VectorSimilarity.Euclidean}[sim]
    osim = {"cos": O.SIM_COSINE, "dot": O.SIM_DOT, "euc": O.SIM_EUCLIDEAN}[sim]
    rows = synth.gen_vectors(n, dims, 1000 + n, "cpu").numpy()
    qs = synth.gen_vectors(19, dims, 2000 + n, "cpu").numpy()      # 19: exercises query padding to 16
    qs[3] = rows[n // 2] + 0.05 * qs[3]                            # planted neighbour
    ix = Index(0, vector_dims=dims, vector_similarity=simv)
    ix.add_vectors(rows)
    assert ix.vector_count == n
    for k in (1, 10, 32):
        got = ix.search_vector_batch(qs, k)
        ref_rows = np.stack([O.normalize(r) for r in rows]) if sim == "cos" else rows
        for i in range(len(qs)):
            q = O.normalize(qs[i]) if sim == "cos" else qs[i]
            want = O.search_vector(ref_rows, q, k, osim)
            _check_vec(got[i], want)
    if sim == "cos":
        assert got[3][0][0] == n // 2
    ix.close()


def test_vector_reference_fixture(golden):
    """tests/test.rs:693-745 through the mirrored Search::search: 3 results / count 3 / total 3."""
    from seekstorm_b200 import Index, QueryType, ResultType, SearchMode, VectorSimilarity
    rows = np.array([[(128 * j + i + 1) / 1000.0 for i in range(128)] for j in range(3)], dtype=np.float32)
    ix = Index(0, vector_dims=128, vector_similarity=VectorSimilarity.Euclidean)
    ix.add_vectors(rows)
    ro = ix.search("", list(rows[0]), QueryType.Union, SearchMode.Vector(None), False, 0, 10, ResultType.TopkCount)
    assert len(ro.results) == 3 and ro.result_count == 3 and ro.result_count_total == 3
    want = golden["ref_fixture_vector"]["results"]
    assert [r.doc_id for r in ro.results] == [d for d, _ in want]
    for r, (_, s) in zip(ro.results, want):
        assert abs(r.score - s) <= 1e-5 * max(1.0, abs(s))
    ix.close()


def test_vector_doc_ids_and_levels():
    """doc_id = level<<16 | local (vector.rs:1448) with explicit local ids and non-contiguous levels."""
    from seekstorm_b200 import Index, VectorSimilarity
    rows = synth.gen_vectors(300, 64, 5, "cpu").numpy()
    ix = Index(0, vector_dims=64, vector_similarity=VectorSimilarity.Dot)
    ix.add_vector_level(2, rows[:100], np.arange(100, 200, dtype=np.uint16))
    ix.add_vector_level(7, rows[100:], None)
    ids = np.concatenate([(2 << 16) | np.arange(100, 200), (7 << 16) | np.arange(200)]).astype(np.uint32)
    q = rows[150:151]
    got = ix.search_vector_batch(q, 5)[0]
    want = O.search_vector(rows, q[0], 5, O.SIM_DOT, doc_ids=ids)
    _check_vec(got, want)
    assert got[0][0] == (7 << 16) | 50
    ix.close()


def test_lexical_reference_fixture(golden):
    """tests/test.rs:150-208 through the mirrored Search::search."""
    from seekstorm_b200 import QueryType, ResultType, SearchMode
    fx = golden["ref_fixture_lexical"]
    post = {t: [(d, tf) for d, tf in p] for t, p in fx["postings"].items()}
    ix = gpu_index([level_from_postings(0, fx["n_docs"], post, fx["len_bytes"])], fx["n_docs"], fx["len_sum"])
    ro = ix.search("+body2 +test", None, QueryType.Intersection, SearchMode.Lexical(), False, 0, 10, ResultType.TopkCount)
    assert len(ro.results) == 1 and ro.result_count == 1 and ro.result_count_total == 1
    assert ro.results[0].doc_id == 2 and np.float32(ro.results[0].score) == np.float32(fx["and_body2_test"]["results"][0][1])
    ro = ix.search("test", None, QueryType.Union, SearchMode.Lexical(), False, 0, 10, ResultType.Count)
    assert len(ro.results) == 0 and ro.result_count == 0 and ro.result_count_total == 2
    ro = ix.search("body2 test", None, QueryType.Union, SearchMode.Lexical(), False, 0, 10, ResultType.TopkCount)
    assert [(r.doc_id, np.float32(r.score)) for r in ro.results] == [(d, np.float32(s)) for d, s in fx["or_body2_test"]["results"]]
    assert ro.result_count_total == 2
    # offset / length paging (search.rs:2108-2121)
    ro = ix.search("body2 test", None, QueryType.Union, SearchMode.Lexical(), False, 1, 10, ResultType.TopkCount)
    assert [r.doc_id for r in ro.results] == [3]
    ix.close()


def test_lexical_hand_corpus(golden):
    from seekstorm_b200 import QueryType, ResultType
    h = golden["hand_corpus"]
    post = {t: [(d, tf) for d, tf in p] for t, p in h["postings"].items()}
    ix = gpu_index([level_from_postings(0, h["n_docs"], post, h["len_bytes"])], h["n_docs"], h["len_sum"])
    for q in h["queries"]:
        qt = QueryType.Intersection if q["type"] == "and" else QueryType.Union
        res, counts = ix.search_lexical_batch([[key_of(t) for t in q["terms"]]], qt, 3, ResultType.TopkCount)
        assert int(counts[0]) == q["count_total"], q
        assert [d for d, _ in res[0]] == [d for d, _ in q["top3"]], q
        for (_, s), (_, w) in zip(res[0], q["top3"]):
            assert abs(s - w) <= 2e-7 * abs(w), q
    ix.close()


def _compare_lexical(ix, orc, qkeys, qt, oqt, k, rt, ort):
    got, counts = ix.search_lexical_batch(qkeys, qt, k, rt)
    for i, kq in enumerate(qkeys):
        want, tot = orc.search(kq, oqt, k, ort)
        if ort != O.RESULT_COUNT:
            assert got[i] == want, (i, kq, got[i], want)        # bit-exact ids, ranks, scores
        else:
            assert got[i] == []
        if ort != O.RESULT_TOPK:
            assert int(counts[i]) == tot, (i, counts[i], tot)


def test_lexical_c1_and_parity():
    """C1: 100k docs, 1000 2-term AND queries, TopkCount (SURVEY.md §8d) vs the exhaustive oracle."""
    from seekstorm_b200 import QueryType, ResultType
    lvs, ls = synth_levels(100000, 100000, 1001)
    orc = oracle_index([l.to_numpy() for l in lvs], 100000, ls)
    ix = gpu_index([l.to_numpy() for l in lvs], 100000, ls)
    qk = query_keys(synth.gen_queries(1000, 2001, 20, 20000))
    _compare_lexical(ix, orc, qk, QueryType.Intersection, O.QUERY_INTERSECTION, 10, ResultType.TopkCount, O.RESULT_TOPKCOUNT)
    _compare_lexical(ix, orc, qk[:200], QueryType.Intersection, O.QUERY_INTERSECTION, 10, ResultType.Topk, O.RESULT_TOPK)
    _compare_lexical(ix, orc, qk[:200], QueryType.Intersection, O.QUERY_INTERSECTION, 0, ResultType.Count, O.RESULT_COUNT)
    ix.close()


@pytest.mark.parametrize("seed,n_docs,vocab", [(3, 150000, 20000), (4, 66000, 500)])
def test_lexical_or_parity(seed, n_docs, vocab):
    """OR with block-max / MAXSCORE pruning == exhaustive oracle, 1-4 terms, dense and sparse lists, k in {1,10,32}."""
    from seekstorm_b200 import QueryType, ResultType
    lvs, ls = synth_levels(n_docs, vocab, seed)
    orc = oracle_index([l.to_numpy() for l in lvs], n_docs, ls)
    ix = gpu_index([l.to_numpy() for l in lvs], n_docs, ls)
    qs = synth.gen_queries(300, 50 + seed, 1, min(vocab, 20000), (1, 2, 3, 4), (0.1, 0.4, 0.3, 0.2))
    qk = query_keys(qs)
    qk[5] = qk[5] + [key_of("missing-term")]          # OR drops unknown terms (search.rs:3295-3296)
    for k in (1, 10, 32):
        _compare_lexical(ix, orc, qk, QueryType.Union, O.QUERY_UNION, k, ResultType.Topk, O.RESULT_TOPK)
    _compare_lexical(ix, orc, qk, QueryType.Union, O.QUERY_UNION, 10, ResultType.TopkCount, O.RESULT_TOPKCOUNT)
    _compare_lexical(ix, orc, qk[:50], QueryType.Union, O.QUERY_UNION, 0, ResultType.Count, O.RESULT_COUNT)
    qa = [q for q in qk if len(q) >= 2]
    qa[3] = qa[3] + [key_of("missing-term")]          # AND with an unknown term -> empty (search.rs:3290-3294)
    _compare_lexical(ix, orc, qa, QueryType.Intersection, O.QUERY_INTERSECTION, 10, ResultType.TopkCount, O.RESULT_TOPKCOUNT)
    ix.close()


def test_lexical_device_pointers_and_tf_overflow():
    """Levels handed over as DEVICE pointers (torch tensors) + tf >= 255 exception path."""
    from seekstorm_b200 import Index, QueryType, ResultType
    post = {"big": [(0, 300), (5, 255), (9, 254), (70, 1000)], "x": [(5, 2), (9, 1), (11, 7)]}
    lens = [synth.int_to_byte4(l) for l in ([400] * 100)]
    lv = level_from_postings(0, 100, post, lens)
    len_sum = sum(synth.byte4_to_int(b) for b in lens)
    orc = oracle_index([lv], 100, len_sum)
    ix = Index(0)
    dev = {k: (torch.from_numpy(v.view(np.int64) if v.dtype == np.uint64 else v.view(np.int32) if v.dtype == np.uint32
                                else v.view(np.int16) if v.dtype == np.uint16 else v).cuda())
           for k, v in lv.items() if isinstance(v, np.ndarray)}
    ix.add_lexical_level(0, 100, dev["term_keys"], dev["posting_offsets"], dev["doc_ids"], dev["tfs"], dev["doc_len_bytes"])
    ix.commit(100, len_sum)
    qk = [[key_of("big")], [key_of("big"), key_of("x")], [key_of("x"), key_of("big")]]
    for qt, oqt in ((QueryType.Union, O.QUERY_UNION), (QueryType.Intersection, O.QUERY_INTERSECTION)):
        _compare_lexical(ix, orc, qk, qt, oqt, 10, ResultType.TopkCount, O.RESULT_TOPKCOUNT)
    ix.close()


def test_hybrid_parity():
    """SearchMode::Hybrid: RRF (search.rs:1962-2035) of the two top-k lists vs the oracle's rrf on oracle lists."""
    from seekstorm_b200 import Index, QueryType, VectorSimilarity
    n = 70000
    lvs, ls = synth_levels(n, 5000, 9)
    orc = oracle_index([l.to_numpy() for l in lvs], n, ls)
    rows = synth.gen_vectors(n, 96, 10, "cpu").numpy()
    ix = Index(0, vector_dims=96, vector_similarity=VectorSimilarity.Cosine)
    for l in lvs:
        ix.add_synth_level(l)
    ix.commit(n, ls)
    ix.add_vectors(rows)
    qs = synth.gen_queries(40, 77, 5, 4000, (2, 3), (0.5, 0.5))
    qk = query_keys(qs)
    qv = synth.gen_vectors(40, 96, 78, "cpu").numpy()
    got = ix.search_hybrid_batch(qk, QueryType.Union, qv, 10)
    nrows = np.stack([O.normalize(r) for r in rows])
    for i in range(40):
        lex, _ = orc.search(qk[i], O.QUERY_UNION, 10, O.RESULT_TOPK)
        vec = O.search_vector(nrows, O.normalize(qv[i]), 10, O.SIM_COSINE)
        want = O.rrf(lex, vec)[:10]
        assert [d for d, _ in got[i]] == [d for d, _ in want], (i, got[i], want)
        assert [np.float32(s) for _, s in got[i]] == [np.float32(s) for _, s in want]
    ix.close()


def test_errors_are_status_codes():
    from seekstorm_b200 import Index, QueryType, ResultType, SsbError
    ix = Index(0, vector_dims=32)
    with pytest.raises(SsbError, match="commit"):
        ix.search_lexical_batch([[1]], QueryType.Union, 10, ResultType.Topk)
    with pytest.raises(SsbError, match="k"):
        ix.search_vector_batch(np.zeros((1, 32), dtype=np.float32), 1025)      # SSB_K_LIMIT = 1024 (paged beyond 32)
    with pytest.raises(SsbError, match="dims"):
        ix.add_vector_level(0, np.zeros((4, 16), dtype=np.float32))
    assert ix.search_vector_batch(np.ones((2, 32), dtype=np.float32), 5) == [[], []]   # empty index -> empty results
    ix.close()


@pytest.mark.parametrize("kernel", [2, 3, 4, 5, 6, 7, 8, 9])
@pytest.mark.parametrize("n,dims,sim", [(300, 32, "dot"), (5000, 128, "cos"), (40000, 768, "cos"), (1000, 100, "dot")])
def test_vector_tcgen05_parity(n, dims, sim, kernel):
    """Tensor-core (wgmma, 3xTF32 / 3xBF16 split) scan vs the oracle: same ids, scores within 1e-4 relative."""
    from seekstorm_b200 import Index, VectorSimilarity
    simv = {"cos": VectorSimilarity.Cosine, "dot": VectorSimilarity.Dot}[sim]
    osim = {"cos": O.SIM_COSINE, "dot": O.SIM_DOT}[sim]
    rows = synth.gen_vectors(n, dims, 3000 + n, "cpu").numpy()
    qs = synth.gen_vectors(150, dims, 4000 + n, "cpu").numpy()      # 150 -> padded to 256 = two query groups
    qs[3] = rows[n // 2] + 0.05 * qs[3]
    ix = Index(0, vector_dims=dims, vector_similarity=simv, vector_kernel=kernel)   # 2/3: 3xTF32 (128/64 queries per pass), 4/5/6: 3xBF16 (128/64/256), 7/8/9: fp16 filter + f32 refine (128 / 256 / 256 on CTA pairs)
    ix.add_vectors(rows)
    ref_rows = np.stack([O.normalize(r) for r in rows]) if sim == "cos" else rows
    for k in (10, 32) if kernel < 7 else (1, 10, 16, 32):
        got = ix.search_vector_batch(qs, k)
        if kernel >= 7:
            # the filter scan really ran for k <= 16 (it streams 2 bytes per element + the candidate rows); k = 32 takes the exact scan
            qt = 128 if kernel == 7 else 256
            passes = (len(qs) + qt - 1) // qt
            p128, p256 = (len(qs) + 127) // 128, (len(qs) + 255) // 256
            exact_passes = p256 if (kernel in (8, 9) and p256 * 237 < p128 * 108) else p128      # k > 16: the exact 3-product scan AUTO would pick
            want_bytes = passes * n * dims * 2 + len(qs) * 32 * dims * 4 if k <= 16 else exact_passes * n * dims * 4
            assert ix.last_stats()["scan_bytes_read"] == want_bytes
        for i in range(0, len(qs), 7):
            q = O.normalize(qs[i]) if sim == "cos" else qs[i]
            _check_vec(got[i], O.search_vector(ref_rows, q, k, osim))
    ix.close()


def _i8_want(r8, q8, k):
    """exact int32 scores via f32 BLAS (every partial sum is an integer < 2^24), canonical tie rule"""
    sc = r8.astype(np.float32) @ q8.astype(np.float32).T            # [n, nq]
    out = []
    for j in range(sc.shape[1]):
        order = np.lexsort((np.arange(sc.shape[0]), -sc[:, j]))[:k]
        out.append([(int(i), float(sc[i, j])) for i in order])
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("n,dims", [(1, 32), (300, 100), (5000, 128), (5000, 768), (70000, 200), (140000, 64), (3000, 1100)])
def test_vector_int8_parity(n, dims):
    """Cosine + ScalarQuantizationI8 (SURVEY §8f row 2): s8 wgmma scan, BIT-EXACT ids and scores vs the oracle."""
    from seekstorm_b200 import Index, VectorSimilarity
    rows = synth.gen_vectors(n, dims, 5000 + n, "cpu").numpy()
    qs = synth.gen_vectors(150, dims, 6000 + n, "cpu").numpy()      # 150 -> padded to 256 = two query groups
    qs[3] = rows[n // 2] + 0.05 * qs[3]
    ix = Index(0, vector_dims=dims, vector_similarity=VectorSimilarity.Cosine, vector_quantization=1)
    ix.add_vectors(rows)
    assert ix.vector_count == n
    r8 = O.quantize_rows_i8(rows)
    q8 = O.quantize_rows_i8(qs)
    for k in (1, 10, 32, 100):
        got = ix.search_vector_batch(qs, k)
        want = _i8_want(r8, q8, k)
        for i in range(len(qs)):
            assert got[i] == want[i], (i, k, got[i][:3], want[i][:3])
    # and against the C oracle's own scan for a few queries
    got = ix.search_vector_batch(qs[:5], 10)
    for i in range(5):
        assert got[i] == O.search_vector_i8(r8, q8[i], 10)
    assert got[3][0][0] == n // 2
    # single query (padding slots must stay empty), device-resident queries
    one = ix.search_vector_batch(torch.from_numpy(qs[7:8]).cuda(), 10)
    assert one[0] == _i8_want(r8, q8[7:8], 10)[0]
    ix.close()


@pytest.mark.gpu
def test_vector_int8_config_errors():
    from seekstorm_b200 import Index, VectorSimilarity
    from seekstorm_b200._lib import SsbError
    with pytest.raises(SsbError):
        Index(0, vector_dims=64, vector_quantization=7)
    # Euclidean + SQ: the FIRST vector decides the quantiser for the life of the index (vector.rs:657-664) — integer-valued 0..255 data takes the
    # affine one (scores = exact negated squared distances here), anything else the non-affine one
    ix = Index(0, vector_dims=8, vector_similarity=VectorSimilarity.Euclidean, vector_quantization=1)
    rows = np.arange(24, dtype=np.float32).reshape(3, 8)
    ix.add_vectors(rows)
    got = ix.search_vector_batch(rows[1:2] + 1, 3)[0]
    c, s, nrm, zp, sq, st = O.quantize_affine_rows_i8(rows)
    qc, qsc, qn, qz, qsum, _ = O.quantize_affine_rows_i8(rows[1:2] + 1, st, False)
    assert st == (0.0, 31.0) and got == O.search_vector_i8_affine(c, s, nrm, zp, sq, qc[0], qsc[0], qn[0], qz[0], qsum[0], 3)
    assert [d for d, _ in got] == [1, 2, 0]
    ix.close()
    with pytest.raises(SsbError):                       # TurboQuantI8 needs its sign mask before the first vector
        ix = Index(0, vector_dims=8, vector_similarity=VectorSimilarity.Dot, vector_quantization=2)
        ix.add_vectors(rows)


@pytest.mark.gpu
@pytest.mark.parametrize("sim", ["dot", "euc"])
@pytest.mark.parametrize("n,dims", [(300, 100), (5000, 128), (70000, 200), (3000, 1100)])
def test_vector_int8_scaled_parity(n, dims, sim):
    """Dot / Euclidean + ScalarQuantizationI8 (per-vector scale [+ norm], vector.rs:597-660): s8 wgmma scan with the scaled
    epilogue, BIT-EXACT ids and scores vs the oracle (QuantizedVector::new_scale[_norm], dot_i8_quantized / euclidean_i8_quantized)."""
    from seekstorm_b200 import Index, VectorSimilarity
    simv, osim = (VectorSimilarity.Dot, O.SIM_DOT) if sim == "dot" else (VectorSimilarity.Euclidean, O.SIM_EUCLIDEAN)
    rows = synth.gen_vectors(n, dims, 7000 + n, "cpu").numpy() * np.float32(0.37)
    qs = synth.gen_vectors(40, dims, 8000 + n, "cpu").numpy()
    qs[3] = rows[n // 2] + 0.01 * qs[3]
    ix = Index(0, vector_dims=dims, vector_similarity=simv, vector_quantization=1)
    ix.add_vectors(rows)
    rc, rs, rn = O.quantize_scale_rows_i8(rows, sim == "euc")
    qc, qsc, qn = O.quantize_scale_rows_i8(qs, sim == "euc")
    for k in (1, 10, 32, 50):
        got = ix.search_vector_batch(qs, k)
        for i in range(0, len(qs), 3):
            want = O.search_vector_i8_scaled(rc, rs, rn, qc[i], float(qsc[i]), float(qn[i]), osim, k)
            assert [d for d, _ in got[i]] == [d for d, _ in want], (i, k, got[i][:3], want[:3])
            assert [np.float32(s) for _, s in got[i]] == [np.float32(s) for _, s in want]
    assert ix.search_vector_batch(qs[3:4], 1)[0][0][0] == n // 2
    ix.close()


@pytest.mark.gpu
def test_hybrid_with_int8_vectors():
    """Hybrid RRF over BM25 + the int8 vector path: fused list equals RRF of the two oracle lists."""
    from seekstorm_b200 import Index, QueryType, VectorSimilarity
    n, dims = 30000, 96
    levels, ls = synth_levels(n, 3000, 21)
    ix = gpu_index([lv.to_numpy() for lv in levels], n, ls, vector_dims=dims, vector_similarity=VectorSimilarity.Cosine,
                   vector_quantization=1)
    orc = oracle_index([lv.to_numpy() for lv in levels], n, ls)
    rows = synth.gen_vectors(n, dims, 22, "cpu").numpy()
    ix.add_vectors(rows)
    r8 = O.quantize_rows_i8(rows)
    queries = synth.gen_queries(6, 23, 5, 1500, (2, 3), (0.5, 0.5))
    qkeys = query_keys(queries)
    qv = synth.gen_vectors(6, dims, 24, "cpu").numpy()
    q8 = O.quantize_rows_i8(qv)
    got = ix.search_hybrid_batch(qkeys, QueryType.Union, qv, 10)
    for i in range(6):
        lex, _ = orc.search(qkeys[i], O.QUERY_UNION, 10, O.RESULT_TOPK)
        vec = O.search_vector_i8(r8, q8[i], 10)
        want = O.rrf(lex, vec)[:10]
        assert [d for d, _ in got[i]] == [d for d, _ in want], (i, got[i], want)
        assert np.allclose([s for _, s in got[i]], [s for _, s in want], rtol=1e-6)
    ix.close()


@pytest.mark.parametrize("kernel", [7, 8, 9])
def test_vector_filter_scan_fallback_on_dense_ties(kernel):
    """Filter scan: when more than 32 rows sit within the error margin of the k-th best approximate score the candidate set does not
    fit the list; those queries must be re-run by the exact fallback scan on the device (vec_refine.cu) and still return the exact top-k
    under the canonical tie rule.  Corpus: 60 identical copies and 60 near-copies (1e-4 noise) of two base vectors among 30k others."""
    from seekstorm_b200 import Index, VectorSimilarity
    n, dims = 30000, 96
    rng = np.random.default_rng(77)
    rows = synth.gen_vectors(n, dims, 5001, "cpu").numpy()
    v1, v2 = rows[11].copy(), rows[12].copy()
    dup = rng.choice(np.arange(100, n), size=120, replace=False)
    rows[dup[:60]] = v1
    rows[dup[60:]] = v2 + 1e-4 * rng.normal(size=(60, dims)).astype(np.float32)
    qs = synth.gen_vectors(140, dims, 5002, "cpu").numpy()
    qs[0] = v1 + 0.01 * qs[0]          # top = the 61 identical rows: ties broken by doc id
    qs[1] = v2 + 0.01 * qs[1]          # top = 61 near-identical rows: exact f32 order decides
    ix = Index(0, vector_dims=dims, vector_similarity=VectorSimilarity.Cosine, vector_kernel=kernel)
    ix.add_vectors(rows)
    nrows = np.stack([O.normalize(r) for r in rows])
    for k in (10, 16):
        got = ix.search_vector_batch(qs, k)
        st = ix.last_stats()
        assert st["filter_fallbacks"] >= 2, st
        for i in (0, 1, 2, 70, 139):
            _check_vec(got[i], O.search_vector(nrows, O.normalize(qs[i]), k, O.SIM_COSINE))
        ident = sorted([11] + dup[:60].tolist())[:k]
        assert [d for d, _ in got[0]] == ident
    # a deleted duplicate never comes back through the fallback either
    ix.set_deleted([ident[0], ident[3]])
    got = ix.search_vector_batch(qs[:2], 10)
    want = [d for d in sorted([11] + dup[:60].tolist()) if d not in (ident[0], ident[3])][:10]
    assert [d for d, _ in got[0]] == want
    ix.close()


def _turbo_mask(dims, seed):
    dim = 1
    while dim < dims:
        dim *= 2
    return np.where(np.random.default_rng(seed).random(dim) < 0.5, 1.0, -1.0).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("sim", ["dot", "cos", "euc"])
@pytest.mark.parametrize("n,dims", [(300, 100), (5000, 128), (70000, 200), (20000, 768), (2000, 1100)])
def test_vector_turboquant_parity(n, dims, sim):
    """TurboQuantI8 (vector_similarity.rs:1825-2093): sign mask + FWHT + sigma/32 quantiser on the device, s8 wgmma scan over the
    next_power_of_two(dims)-byte codes, scores rebuilt in the reference's order (Dot / Cosine NEGATED like the reference, :161-176) —
    BIT-EXACT codes (implied by the scores), ids and scores vs the oracle."""
    from seekstorm_b200 import Index, VectorSimilarity
    simv, osim = {"dot": (VectorSimilarity.Dot, O.SIM_DOT), "cos": (VectorSimilarity.Cosine, O.SIM_COSINE), "euc": (VectorSimilarity.Euclidean, O.SIM_EUCLIDEAN)}[sim]
    rows = synth.gen_vectors(n, dims, 9000 + n, "cpu").numpy() * np.float32(0.53)
    qs = synth.gen_vectors(24, dims, 9500 + n, "cpu").numpy()
    qs[3] = rows[n // 2] + 0.01 * qs[3]
    mask = _turbo_mask(dims, 17)
    ix = Index(0, vector_dims=dims, vector_similarity=simv, vector_quantization=2)
    with pytest.raises(Exception):
        ix.add_vectors(rows[:10])                      # no mask yet
    ix.set_turboquant_mask(mask)
    ix.add_vectors(rows)
    rc, rs, rn = O.turboquant_rows_i8(rows, mask, sim == "cos")
    qc, qsc, qn = O.turboquant_rows_i8(qs, mask, sim == "cos")
    for k in (1, 10, 40):
        got = ix.search_vector_batch(qs, k)
        for i in range(0, len(qs), 3):
            want = O.search_vector_i8_turbo(rc, rs, rn, qc[i], float(qsc[i]), float(qn[i]), osim, k)
            assert [d for d, _ in got[i]] == [d for d, _ in want], (i, k, got[i][:3], want[:3])
            assert [np.float32(s) for _, s in got[i]] == [np.float32(s) for _, s in want]
    if sim == "euc":                                   # Euclidean keeps its meaning: the planted neighbour is the best hit
        assert ix.search_vector_batch(qs[3:4], 1)[0][0][0] == n // 2
    ix.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n,dims", [(300, 100), (70000, 128), (3000, 1100)])
def test_vector_int8_affine_parity(n, dims):
    """Euclidean + ScalarQuantizationI8 over integer-valued 0..255 data (SIFT-like): the reference's AFFINE quantiser
    (new_scale_norm_affine with its running min / max state, vector_similarity.rs:1414-1463) and euclidean_i8_quantized_affine (:1770-1795):
    BIT-EXACT ids and scores vs the oracle, incl. the rows quantised while the state was still growing and several levels."""
    from seekstorm_b200 import Index, VectorSimilarity
    rng = np.random.default_rng(1000 + n)
    rows = np.clip(np.abs(rng.normal(0, 45, (n, dims))).round(), 0, 255).astype(np.float32)
    rows[0] = np.clip(rows[0], 3, 90)                     # the state starts narrow: (3, raster(87) = 127) ...
    rows[1] = np.clip(rows[1], 1, 120)
    rows[5, 0] = 0; rows[7, 1] = 255                      # ... and reaches (0, 255) a few rows later
    qs = np.clip(np.abs(rng.normal(0, 45, (24, dims))).round(), 0, 255).astype(np.float32)
    qs[3] = np.clip(rows[n // 2] + rng.integers(-2, 3, dims), 0, 255)
    ix = Index(0, vector_dims=dims, vector_similarity=VectorSimilarity.Euclidean, vector_quantization=1)
    ix.add_vectors(rows)
    rc, rs, rn, rz, rsum, st = O.quantize_affine_rows_i8(rows)
    qc, qsc, qn, qz, qsum, _ = O.quantize_affine_rows_i8(qs, st, False)
    for k in (1, 10, 40):
        got = ix.search_vector_batch(qs, k)
        for i in range(0, len(qs), 3):
            want = O.search_vector_i8_affine(rc, rs, rn, rz, rsum, qc[i], float(qsc[i]), float(qn[i]), int(qz[i]), int(qsum[i]), k)
            assert [d for d, _ in got[i]] == [d for d, _ in want], (i, k, got[i][:3], want[:3])
            assert [np.float32(s) for _, s in got[i]] == [np.float32(s) for _, s in want]
    assert ix.search_vector_batch(qs[3:4], 1)[0][0][0] == n // 2
    ix.close()
