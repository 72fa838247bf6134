"""GPU: multi-vector documents — the field filter inside every vector scan, the best row's field / chunk in the vb results, observed
counts under a mask, and the hybrid / loader / mirror plumbing, against the numpy restatement of search_vector_shard + TopK::push
(tests/helpers_vecfields.py)."""
import numpy as np
import pytest

from helpers_vecfields import search_fields_fast, tagged_corpus, threshold_premap, write_vector_bin_fields
from oracle import oracle as O
from seekstorm_b200 import Index, VectorSimilarity
from seekstorm_b200._lib import SsbError

DOCS_PER_LEVEL = 10000
MASKS = [0, 0b001, 0b110, 1 << 9]          # none, one field, two fields, a field no row holds


def _levels(ids):
    """(level id, local ids, row range) per level of DOCS_PER_LEVEL docs; doc id = level << 16 | local"""
    out = []
    for lv in range(int(ids.max()) // DOCS_PER_LEVEL + 1):
        sel = np.nonzero(ids // DOCS_PER_LEVEL == lv)[0]
        out.append((lv, (ids[sel] % DOCS_PER_LEVEL).astype(np.uint16), sel[0], sel[-1] + 1))
    return out


def _doc_ids(ids):
    return ((ids // DOCS_PER_LEVEL) << 16) | (ids % DOCS_PER_LEVEL)


def _index(rows, ids, fields, chunks, sim, tagged=True, quant=0, mask=None):
    ix = Index(0, vector_dims=rows.shape[1], vector_similarity=sim, vector_quantization=quant)
    if mask is not None:
        ix.set_turboquant_mask(mask)
    for lv, loc, a, b in _levels(ids):
        if tagged:
            ix.add_vector_level(lv, rows[a:b], loc, field_ids=fields[a:b], chunk_ids=chunks[a:b])
        else:
            ix.add_vector_level(lv, rows[a:b], loc)
    return ix


def _check(got, ext, k, want, exact=False, rel=1e-4, q=None):
    """ids and scores against the restatement (exact: bit for bit), field / chunk of every hit whose best row is decided"""
    gd, gs = [d for d, _ in got], [s for _, s in got]
    wd, ws = [h[0] for h in want], [h[1] for h in want]
    assert len(gd) == len(wd), (q, got[:3], want[:3])
    for j in range(len(gd)):
        if exact:
            assert np.float32(gs[j]) == np.float32(ws[j]), (q, j, gs[j], ws[j])
        else:
            assert abs(gs[j] - ws[j]) <= rel * max(1.0, abs(ws[j])), (q, j, gs[j], ws[j])
        if gd[j] != wd[j]:    # only a near-tie may swap two docs
            assert exact is False and abs(ws[j] - gs[j]) < 1e-5 * max(1.0, abs(ws[j])), (q, j, gd[j], wd[j], gs[j], ws[j])
            continue
        h = want[j]
        if exact or h[4] > rel * max(1.0, abs(h[1])):
            e = ext[q * k + j]
            assert (e.field_id, e.chunk_id) == (h[2], h[3]), (q, j, (e.field_id, e.chunk_id), h)


@pytest.fixture(scope="module")
def corpus():
    rows, ids, fields, chunks = tagged_corpus(4 * DOCS_PER_LEVEL - 5000, 64, 11)   # ~210 K rows, 3 fields x 1-3 chunks
    assert rows.shape[0] >= 200000
    qs = np.random.default_rng(12).standard_normal((300, 64)).astype(np.float32)
    qs[5] = rows[100] + np.float32(0.01) * qs[5]
    masks = np.array([MASKS[i % 4] for i in range(300)], dtype=np.uint32)
    return rows, ids, fields, chunks, qs, masks


def _scores(rows, qs, sim):
    if sim == VectorSimilarity.Cosine:
        r = rows / np.linalg.norm(rows, axis=1, keepdims=True); q = qs / np.linalg.norm(qs, axis=1, keepdims=True)
        return (q.astype(np.float64) @ r.T.astype(np.float64)).astype(np.float32)
    if sim == VectorSimilarity.Dot:
        return (qs.astype(np.float64) @ rows.T.astype(np.float64)).astype(np.float32)
    d = (qs.astype(np.float64) ** 2).sum(1)[:, None] + (rows.astype(np.float64) ** 2).sum(1)[None, :] - 2 * qs.astype(np.float64) @ rows.T.astype(np.float64)
    return (-d).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("sim,kernels", [(VectorSimilarity.Cosine, range(1, 10)), (VectorSimilarity.Dot, range(1, 10)),
                                         (VectorSimilarity.Euclidean, (1,))])
def test_f32_every_kernel_masked(corpus, sim, kernels):
    rows, ids, fields, chunks, qs, masks = corpus
    S = _scores(rows, qs, sim)
    doc = _doc_ids(ids)
    k = 10
    want = [search_fields_fast(S[q], doc, fields, chunks, k, int(masks[q])) for q in range(len(qs))]
    ix = _index(rows, ids, fields, chunks, sim)
    for kern in kernels:
        ix.set_vector_kernel(kern)
        for b in (1, 8, 64, 200, 256, 300):
            got, ext, obs = ix.search_vector_ex(qs[:b], k, field_masks=masks[:b])
            for q in range(b):
                _check(got[q], ext, k, want[q][0], q=q)
                assert int(obs[q]) == want[q][1], (kern, b, q)
        assert got[3] == [] and int(obs[3]) == 0           # mask of a field no row holds
    ix.close()


@pytest.mark.gpu
def test_tagging_changes_nothing_unmasked(corpus):
    rows, ids, fields, chunks, qs, _ = corpus
    a = _index(rows, ids, fields, chunks, VectorSimilarity.Cosine, tagged=True)
    u = _index(rows, ids, fields, chunks, VectorSimilarity.Cosine, tagged=False)
    for kern in (0, 1, 2, 4, 6, 7, 8, 9):
        a.set_vector_kernel(kern); u.set_vector_kernel(kern)
        for b in (8, 256, 300):
            ga = a.search_vector_batch(qs[:b], 10); la = a.last_stats()["kernel_launches"]
            gu = u.search_vector_batch(qs[:b], 10); lu = u.last_stats()["kernel_launches"]
            assert ga == gu and la == lu, (kern, b)
            gz, _, oz = a.search_vector_ex(qs[:b], 10, field_masks=np.zeros(b, np.uint32))   # all-zero masks: the unmasked path
            assert gz == gu and a.last_stats()["kernel_launches"] >= lu
            assert (oz == rows.shape[0]).all()
    with pytest.raises(SsbError):                           # a mask on an index without field ids
        u.search_vector_ex(qs[:2], 10, field_masks=[1, 0])
    a.close(); u.close()


def _i8_scores(kind, rows, qs, mask=None):
    """per-row scores of the int8 quantisers through the oracle (k = every row, doc id = row): bit-exact references"""
    n = rows.shape[0]
    ids = np.arange(n, dtype=np.uint32)
    S = np.full((len(qs), n), np.nan, dtype=np.float32)
    if kind == "sq_cos":
        r8, q8 = O.quantize_rows_i8(rows), O.quantize_rows_i8(qs)
        res = [O.search_vector_i8(r8, q8[i], n, ids) for i in range(len(qs))]
    elif kind in ("sq_dot", "sq_euc"):
        euc = kind == "sq_euc"
        r8, rs, rn = O.quantize_scale_rows_i8(rows, euc); q8, qsc, qn = O.quantize_scale_rows_i8(qs, euc)
        res = [O.search_vector_i8_scaled(r8, rs, rn, q8[i], float(qsc[i]), float(qn[i]), O.SIM_EUCLIDEAN if euc else O.SIM_DOT, n, ids)
               for i in range(len(qs))]
    elif kind == "affine":
        r8, rs, rn, rz, ru, st = O.quantize_affine_rows_i8(rows)
        q8, qsc, qn, qz, qu, _ = O.quantize_affine_rows_i8(qs, st, update_state=False)
        res = [O.search_vector_i8_affine(r8, rs, rn, rz, ru, q8[i], float(qsc[i]), float(qn[i]), int(qz[i]), int(qu[i]), n, ids)
               for i in range(len(qs))]
    else:
        r8, rs, rn = O.turboquant_rows_i8(rows, mask, True); q8, qsc, qn = O.turboquant_rows_i8(qs, mask, True)
        res = [O.search_vector_i8_turbo(r8, rs, rn, q8[i], float(qsc[i]), float(qn[i]), O.SIM_COSINE, n, ids) for i in range(len(qs))]
    for i, hits in enumerate(res):
        for d, s in hits:
            S[i, d] = s
    return S


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sq_cos", "sq_dot", "sq_euc", "turbo", "affine"])
def test_int8_masked_bit_exact(kind):
    rows, ids, fields, chunks = tagged_corpus(900, 96, 21)
    if kind == "affine":
        rows = np.clip(np.round(rows * 30 + 128), 0, 255).astype(np.float32)
    qs = np.random.default_rng(22).standard_normal((40, 96)).astype(np.float32)
    if kind == "affine":
        qs = np.clip(np.round(qs * 30 + 128), 0, 255).astype(np.float32)
    sim = {"sq_cos": VectorSimilarity.Cosine, "sq_dot": VectorSimilarity.Dot, "sq_euc": VectorSimilarity.Euclidean, "affine": VectorSimilarity.Euclidean,
           "turbo": VectorSimilarity.Cosine}[kind]
    tmask = np.where(np.random.default_rng(23).random(128) < 0.5, 1.0, -1.0).astype(np.float32) if kind == "turbo" else None
    S = _i8_scores(kind, rows, qs, tmask)
    masks = np.array([MASKS[i % 4] for i in range(len(qs))], dtype=np.uint32)
    ix = _index(rows, ids, fields, chunks, sim, quant=2 if kind == "turbo" else 1, mask=tmask)
    doc = _doc_ids(ids)
    for k in (10, 100):
        got, ext, obs = ix.search_vector_ex(qs, k, field_masks=masks)
        for q in range(len(qs)):
            w, o = search_fields_fast(S[q], doc, fields, chunks, k, int(masks[q]))
            _check(got[q], ext, k, w, exact=True, q=q)
            assert int(obs[q]) == o
    ix.close()


@pytest.mark.gpu
def test_paging_threshold_delete(corpus):
    rows, ids, fields, chunks, qs, masks = corpus
    sim = VectorSimilarity.Cosine
    S = _scores(rows, qs, sim)
    doc = _doc_ids(ids)
    ix = _index(rows, ids, fields, chunks, sim)
    rng = np.random.default_rng(31)
    deleted = sorted(set(int(x) for x in doc[rng.integers(0, len(doc), 3000)]) | {int(doc[100])})
    del_rows = np.isin(doc, deleted)
    thr = 0.62
    for kern in (1, 2, 4, 7, 8):
        ix.set_vector_kernel(kern)
        ix.set_deleted([])
        got, ext, _ = ix.search_vector_ex(qs[:64], 100, field_masks=masks[:64])            # paging beyond 32 results
        for q in range(64):
            _check(got[q], ext, 100, search_fields_fast(S[q], doc, fields, chunks, 100, int(masks[q]))[0], q=q)
        got, ext, _ = ix.search_vector_ex(qs[:64], 10, similarity_threshold=thr, field_masks=masks[:64])
        for q in range(64):
            _check(got[q], ext, 10, search_fields_fast(S[q], doc, fields, chunks, 10, int(masks[q]), threshold=threshold_premap(thr, False))[0], q=q)
        ix.set_deleted(deleted)
        got, ext, obs = ix.search_vector_ex(qs, 10, field_masks=masks)
        for q in range(len(qs)):
            w, o = search_fields_fast(S[q], doc, fields, chunks, 10, int(masks[q]), del_rows)
            _check(got[q], ext, 10, w, q=q)
            assert int(obs[q]) == o
    ix.set_deleted([])
    ix.close()


@pytest.mark.gpu
def test_filter_scan_masked_and_fallback(corpus):
    """One row per doc (no multi-chunk de-duplication, so k <= 16 runs the fp16 filter scans 7 / 8 / 9 with their exact refine), then
    near-duplicate rows: the filter scan's candidate set overflows and those queries take the exact fallback scan, still masked."""
    rows, _, _, _, qs, masks = corpus
    sim = VectorSimilarity.Cosine
    n = 60000
    one = rows[:n]
    fld = (np.arange(n) % 3).astype(np.uint8); chk = (np.arange(n) % 5).astype(np.uint32); dids = np.arange(n)
    ix = Index(0, vector_dims=64, vector_similarity=sim)
    ix.add_vector_level(0, one, dids.astype(np.uint16), field_ids=fld, chunk_ids=chk)
    S = _scores(one, qs, sim)
    for kern in (7, 8, 9):
        ix.set_vector_kernel(kern)
        for b in (64, 256, 300):
            got, ext, obs = ix.search_vector_ex(qs[:b], 10, field_masks=masks[:b])
            passes = -(-b // (128 if kern == 7 else 256))
            assert ix.last_stats()["scan_bytes_read"] == passes * n * 64 * 2 + b * 32 * 64 * 4   # the fp16 plane + refine: a filter scan ran
            for q in range(b):
                w, o = search_fields_fast(S[q], dids, fld, chk, 10, int(masks[q]))
                _check(got[q], ext, 10, w, q=q)
                assert int(obs[q]) == o
    ix.close()
    dup = np.repeat(rows[:1], n, axis=0) + np.float32(1e-4) * np.random.default_rng(32).standard_normal((n, 64)).astype(np.float32)
    ix2 = Index(0, vector_dims=64, vector_similarity=sim)
    ix2.add_vector_level(0, dup, dids.astype(np.uint16), field_ids=fld, chunk_ids=chk)
    qd = np.concatenate([dup[:128] + np.float32(0.01) * qs[:128], qs[128:256]])
    md = np.array([MASKS[i % 4] for i in range(256)], dtype=np.uint32)
    Sd = _scores(dup, qd, sim)
    for kern in (8, 9):
        ix2.set_vector_kernel(kern)
        got, ext, _ = ix2.search_vector_ex(qd, 10, field_masks=md)
        assert ix2.last_stats()["filter_fallbacks"] > 0
        for q in range(256):
            w, _ = search_fields_fast(Sd[q], dids, fld, chk, 10, int(md[q]))
            assert len(got[q]) == len(w), q
            assert all(abs(a - b[1]) < 1e-5 for (_, a), b in zip(got[q], w)), q
            assert all(fld[d] in [f for f in range(3) if md[q] == 0 or (md[q] >> f) & 1] for d, _ in got[q]), q
    ix2.close()


def _ivf_scope(levels, qn, ann_mode, n_probe, cthr):
    """rows (global indices) the IVF probe scans for one query: per level the n_probe best medoids (vector.rs:1300-1320)"""
    thr = O.ivf_premap_threshold(cthr, O.SIM_COSINE) if ann_mode in (2, 3) else None
    out = []
    for base, rn, counts in levels:
        starts = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
        scored = []
        for c, st in enumerate(starts):
            m = np.ascontiguousarray(rn[st])
            s = np.float32(O.lib().orc_dot_f32(O._ptr(qn), O._ptr(m), qn.size))
            if thr is not None and s < thr:
                continue
            scored.append((-float(s), c))
        scored.sort()
        np_eff = min(n_probe, len(counts)) if ann_mode in (1, 3) else len(counts)
        for _, c in scored[:np_eff]:
            out.extend(range(base + starts[c], base + starts[c] + counts[c]))
    return np.array(out, dtype=np.int64)


@pytest.mark.gpu
def test_ann_modes_observed():
    rows, ids, fields, chunks = tagged_corpus(6000, 48, 41)
    qs = np.random.default_rng(42).standard_normal((24, 48)).astype(np.float32)
    masks = np.array([MASKS[i % 4] for i in range(24)], dtype=np.uint32)
    ix = Index(0, vector_dims=48, vector_similarity=VectorSimilarity.Cosine)
    rn = rows / np.linalg.norm(rows, axis=1, keepdims=True)
    lv_meta = []
    for lv, loc, a, b in [(0, ids[:17000], 0, 17000), (1, ids[17000:], 17000, len(ids))]:
        n = b - a
        counts = [n // 7] * 6 + [n - 6 * (n // 7)]
        ix.add_vector_level(lv, rows[a:b], (loc % 65536).astype(np.uint16), cluster_counts=counts, field_ids=fields[a:b], chunk_ids=chunks[a:b])
        lv_meta.append((a, rn[a:b].astype(np.float32), counts))
    doc = np.where(np.arange(len(ids)) < 17000, ids, (1 << 16) | ids)
    S = _scores(rows, qs, VectorSimilarity.Cosine)
    for mode, n_probe, cthr in ((0, 0, 0.0), (1, 2, 0.0), (2, 0, 0.52), (3, 3, 0.5)):
        got, ext, obs = ix.search_vector_ex(qs, 10, ann_mode=mode, n_probe=n_probe, cluster_threshold=cthr, field_masks=masks)
        for q in range(len(qs)):
            qn = (qs[q] / np.linalg.norm(qs[q])).astype(np.float32)
            scope = np.zeros(len(ids), dtype=bool)
            scope[_ivf_scope(lv_meta, qn, mode, n_probe, cthr)] = True
            w, o = search_fields_fast(S[q], doc, fields, chunks, 10, int(masks[q]), scope=scope)
            assert int(obs[q]) == o, (mode, q)
            _check(got[q], ext, 10, w, q=q)
    ix.close()


@pytest.mark.gpu
def test_hybrid_loader_mirror_and_errors():
    from helpers import gpu_index, oracle_index, query_keys, synth_levels
    from seekstorm_b200 import QueryType, SearchMode, synth
    n = 3000
    lvs, ls = synth_levels(n, 400, 61)
    levels = [l.to_numpy() for l in lvs]
    orc = oracle_index(levels, n, ls)
    rng = np.random.default_rng(62)
    vrows = rng.standard_normal((2 * n, 32)).astype(np.float32)          # two rows per doc: field 0 and field 1
    vid = np.repeat(np.arange(n), 2); vf = np.tile(np.array([0, 1], np.uint8), n); vc = np.zeros(2 * n, np.uint32)
    qk = query_keys(synth.gen_queries(12, 63, 2, 400, (1, 2), (0.5, 0.5)))
    qv = rng.standard_normal((12, 32)).astype(np.float32)
    S = _scores(vrows, qv, VectorSimilarity.Cosine)
    for tagged in (True, False):
        ix = gpu_index(levels, n, ls, vector_dims=32, vector_similarity=VectorSimilarity.Cosine)
        if tagged:
            ix.add_vector_level(0, vrows, vid.astype(np.uint16), field_ids=vf, chunk_ids=vc)
        else:
            ix.add_vector_level(0, vrows, vid.astype(np.uint16))
        fm = [0b10] * 12
        hyb = ix.search_hybrid_batch(qk, QueryType.Union, qv, 10, field_masks=fm)
        for i in range(12):
            lex, _ = orc.search(qk[i], O.QUERY_UNION, 10, O.RESULT_TOPK)   # single-field lexical index: the mask does not touch it
            w, _ = search_fields_fast(S[i], vid, vf, vc, 10, 0b10 if tagged else 0)
            assert [d for d, _ in hyb[i]] == [d for d, _ in O.rrf(lex, [(h[0], h[1]) for h in w])[:10]], (tagged, i)
        ix.close()
    # Index.search: field_filter reaches the vector rows of a tagged index, the same in Vector and Hybrid mode
    ix = Index(0, vector_dims=32, vector_similarity=VectorSimilarity.Cosine)
    ix.field_names = ["title", "body"]
    ix.add_vector_level(0, vrows, vid.astype(np.uint16), field_ids=vf, chunk_ids=vc)
    rv = ix.search("", qv[0], search_mode=SearchMode.Vector(), field_filter=["body"], length=10)
    rh = ix.search("", qv[0], search_mode=SearchMode.Hybrid(), field_filter=["body"], length=10)
    w, _ = search_fields_fast(S[0], vid, vf, vc, 10, 0b10)
    assert [r.doc_id for r in rv.results] == [h[0] for h in w] == [r.doc_id for r in rh.results]
    assert rv.observed_vector_count == n
    # errors: field id >= 32, mixing tagged and untagged levels, a mask on an untagged index
    with pytest.raises(SsbError):
        ix.add_vector_level(1, vrows[:4], None, field_ids=np.array([0, 1, 32, 0], np.uint8), chunk_ids=np.zeros(4, np.uint32))
    with pytest.raises(SsbError):
        ix.add_vector_level(1, vrows[:4])
    assert ix.vector_count == 2 * n
    ix.close()
    u = Index(0, vector_dims=32, vector_similarity=VectorSimilarity.Cosine)
    u.add_vector_level(0, vrows[:10])
    with pytest.raises(SsbError):
        u.add_vector_level(1, vrows[:4], None, field_ids=np.zeros(4, np.uint8), chunk_ids=np.zeros(4, np.uint32))
    with pytest.raises(SsbError):
        u.search_vector_ex(qv[:1], 5, field_masks=[1])
    u.close()
    # loader: vector.bin with field / chunk ids == the tagged add; the plain loader ignores them
    data = write_vector_bin_fields([(vid.astype(np.uint16), vrows, vf, vc + 3)])
    a = Index(0, vector_dims=32, vector_similarity=VectorSimilarity.Cosine); a.load_vector_bin(data, keep_fields=True)
    b = Index(0, vector_dims=32, vector_similarity=VectorSimilarity.Cosine); b.add_vector_level(0, vrows, vid.astype(np.uint16), field_ids=vf, chunk_ids=vc + 3)
    c = Index(0, vector_dims=32, vector_similarity=VectorSimilarity.Cosine); c.load_vector_bin(data)
    d = Index(0, vector_dims=32, vector_similarity=VectorSimilarity.Cosine); d.add_vector_level(0, vrows, vid.astype(np.uint16))
    fm = [0b01, 0b10, 0] * 4
    ga, ea, oa = a.search_vector_ex(qv, 10, field_masks=fm)
    gb, eb, ob = b.search_vector_ex(qv, 10, field_masks=fm)
    assert ga == gb and (oa == ob).all()
    assert [(e.field_id, e.chunk_id) for e in ea] == [(e.field_id, e.chunk_id) for e in eb]
    assert all(e.chunk_id == 3 for i, e in enumerate(ea) if i % 10 < len(ga[i // 10]))
    assert c.search_vector_batch(qv, 10) == d.search_vector_batch(qv, 10)
    bad = write_vector_bin_fields([(vid[:4].astype(np.uint16), vrows[:4], np.array([0, 40, 0, 0]), vc[:4])])
    e = Index(0, vector_dims=32, vector_similarity=VectorSimilarity.Cosine)
    with pytest.raises(SsbError):
        e.load_vector_bin(bad, keep_fields=True)
    for x in (a, b, c, d, e):
        x.close()
