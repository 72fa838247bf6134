"""GPU: levels of a field-tagged vector index — empty levels (a block whose docs carry no vectors, vector.rs:1056-1073) through the add
call and the vector.bin loader, levels added out of level order, many levels appended in order, masked batches above 4096 queries, and
the Python mirror's field_filter past the lexical fields."""
import numpy as np
import pytest

from helpers_vecfields import search_fields_fast, write_vector_bin_fields
from seekstorm_b200 import Index, SearchMode, VectorSimilarity

MASKS = [0, 0b001, 0b110, 1 << 9]


def _level(seed, n_docs, dims=32):
    """one level: docs with 1-3 rows over fields 0-2, record order doc by doc"""
    rng = np.random.default_rng(seed)
    ids, fld, chk = [], [], []
    for d in range(n_docs):
        for c in range(int(rng.integers(1, 4))):
            ids.append(d); fld.append(int(rng.integers(0, 3))); chk.append(c)
    rows = rng.standard_normal((len(ids), dims)).astype(np.float32)
    return np.array(ids, np.uint16), rows, np.array(fld, np.uint8), np.array(chk, np.uint32)


def _scores(rows, qs):
    r = rows / np.linalg.norm(rows, axis=1, keepdims=True); q = qs / np.linalg.norm(qs, axis=1, keepdims=True)
    return (q.astype(np.float64) @ r.T.astype(np.float64)).astype(np.float32)


def _check(ix, levels, qs, masks, k=10):
    """levels: list of (level id, (ids, rows, fields, chunks)) in any add order; rows are compared in the library's record order"""
    doc = np.concatenate([(lv << 16) | ids.astype(np.int64) for lv, (ids, _, _, _) in levels])
    rows = np.concatenate([r for _, (_, r, _, _) in levels])
    fld = np.concatenate([f for _, (_, _, f, _) in levels]); chk = np.concatenate([c for _, (_, _, _, c) in levels])
    S = _scores(rows, qs)
    got, ext, obs = ix.search_vector_ex(qs, k, field_masks=masks)
    for q in range(len(qs)):
        w, o = search_fields_fast(S[q], doc, fld, chk, k, int(masks[q]))
        assert int(obs[q]) == o, q
        assert len(got[q]) == len(w), q
        for j, h in enumerate(w):
            d, sc = got[q][j]
            assert abs(sc - h[1]) <= 1e-4, (q, j, sc, h)
            if d != h[0]:                                  # only a near-tie may swap two docs
                assert abs(sc - h[1]) < 2e-5, (q, j, d, h)
                continue
            if h[4] > 1e-4:
                assert (ext[q * k + j].field_id, ext[q * k + j].chunk_id) == (h[2], h[3]), (q, j)


@pytest.mark.gpu
def test_empty_levels_are_neutral():
    qs = np.random.default_rng(5).standard_normal((40, 32)).astype(np.float32)
    masks = np.array([MASKS[i % 4] for i in range(40)], np.uint32)
    l0, l2 = _level(1, 500), _level(2, 400)
    ix = Index(0, vector_dims=32, vector_similarity=VectorSimilarity.Cosine)
    ix.add_vector_level(0, l0[1], l0[0], field_ids=l0[2], chunk_ids=l0[3])
    e = np.zeros((0, 32), np.float32)
    ix.add_vector_level(1, e, np.zeros(0, np.uint16), field_ids=np.zeros(0, np.uint8), chunk_ids=np.zeros(0, np.uint32))
    ix.add_vector_level(1, e)                               # an empty untagged add is neutral too
    ix.add_vector_level(2, l2[1], l2[0], field_ids=l2[2], chunk_ids=l2[3])
    _check(ix, [(0, l0), (2, l2)], qs, masks)
    # the same shard as a vector.bin with an empty middle level (one cluster of 0 records, as the reference writes it)
    empty = (np.zeros(0, np.uint16), e, np.zeros(0, np.uint8), np.zeros(0, np.uint32))
    data = write_vector_bin_fields([l0, empty, l2])
    a = Index(0, vector_dims=32, vector_similarity=VectorSimilarity.Cosine)
    assert a.load_vector_bin(data, keep_fields=True) == len(l0[0]) + len(l2[0])
    _check(a, [(0, l0), (2, l2)], qs, masks)
    g1, e1, o1 = a.search_vector_ex(qs, 10, field_masks=masks)
    g2, e2, o2 = ix.search_vector_ex(qs, 10, field_masks=masks)
    assert g1 == g2 and (o1 == o2).all() and [(x.field_id, x.chunk_id) for x in e1] == [(x.field_id, x.chunk_id) for x in e2]
    b = Index(0, vector_dims=32, vector_similarity=VectorSimilarity.Cosine)
    assert b.load_vector_bin(data) == len(l0[0]) + len(l2[0])   # the plain loader reads the same file
    for x in (ix, a, b):
        x.close()


@pytest.mark.gpu
def test_levels_out_of_order_and_many_in_order():
    qs = np.random.default_rng(6).standard_normal((64, 32)).astype(np.float32)
    masks = np.array([MASKS[i % 4] for i in range(64)], np.uint32)
    lv = {i: _level(10 + i, 300 + 50 * i) for i in range(12)}
    ix = Index(0, vector_dims=32, vector_similarity=VectorSimilarity.Cosine)
    order = [3, 0, 7, 1, 2, 11, 4, 5, 6, 8, 10, 9]           # a doc table rebuilt, then appended, then rebuilt again
    for i in order:
        ix.add_vector_level(i, lv[i][1], lv[i][0], field_ids=lv[i][2], chunk_ids=lv[i][3])
        if i in (0, 11):                                   # checked between adds too
            done = order[:order.index(i) + 1]
            _check(ix, [(j, lv[j]) for j in done], qs, masks)
    _check(ix, [(j, lv[j]) for j in order], qs, masks)
    ix.close()
    ix = Index(0, vector_dims=32, vector_similarity=VectorSimilarity.Cosine)
    for i in range(12):
        ix.add_vector_level(i, lv[i][1], lv[i][0], field_ids=lv[i][2], chunk_ids=lv[i][3])
    _check(ix, [(j, lv[j]) for j in range(12)], qs, masks)
    ix.close()


@pytest.mark.gpu
def test_masked_batch_above_4096_queries():
    l0 = _level(20, 1500)
    qs = np.random.default_rng(21).standard_normal((5000, 32)).astype(np.float32)
    masks = np.array([MASKS[i % 4] for i in range(5000)], np.uint32)
    ix = Index(0, vector_dims=32, vector_similarity=VectorSimilarity.Cosine, max_batch=8192)
    ix.add_vector_level(0, l0[1], l0[0], field_ids=l0[2], chunk_ids=l0[3])
    _check(ix, [(0, l0)], qs, masks, k=5)
    ix.close()


@pytest.mark.gpu
def test_search_field_filter_past_the_lexical_fields():
    l0 = _level(30, 800)
    q = np.random.default_rng(31).standard_normal(32).astype(np.float32)
    ix = Index(0, vector_dims=32, vector_similarity=VectorSimilarity.Cosine)
    ix.field_names = ["title", "body"]
    ix.add_vector_level(0, l0[1], l0[0], field_ids=l0[2], chunk_ids=l0[3])
    plain = ix.search("", q, search_mode=SearchMode.Vector(), length=10)
    past = ix.search("", q, search_mode=SearchMode.Vector(), field_filter=[5], length=10)      # names no lexical field: no filter
    assert [r.doc_id for r in past.results] == [r.doc_id for r in plain.results] and len(plain.results) == 10
    body = ix.search("", q, search_mode=SearchMode.Vector(), field_filter=[1, 5], length=10)   # only the lexical bit counts
    S = _scores(l0[1], q[None])[0]
    w, _ = search_fields_fast(S, l0[0].astype(np.int64), l0[2], l0[3], 10, 0b10)
    assert [r.doc_id for r in body.results] == [h[0] for h in w] and len(w) == 10
    ix.close()
