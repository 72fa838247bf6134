"""CPU: the multi-vector restatement (tests/helpers_vecfields.py) on hand cases — the field filter, the best row per doc and its tie
rule, the threshold, the delete set, observed — and the vector.bin writer with field / chunk ids."""
import numpy as np

from helpers_vecfields import (TopK, passes, read_vector_bin_headers, search_fields, search_fields_topk, tagged_corpus,
                               threshold_premap, write_vector_bin_fields)
from refwriter import write_vector_bin


def _case():
    # rows in record order: doc, field, chunk, score
    rows = [(0, 0, 0, 0.90), (0, 1, 0, 0.10), (1, 0, 0, 0.80), (1, 1, 3, 0.85), (2, 1, 0, 0.70), (2, 1, 1, 0.70), (3, 2, 0, 0.60)]
    doc = np.array([r[0] for r in rows]); field = np.array([r[1] for r in rows], dtype=np.uint8)
    chunk = np.array([r[2] for r in rows], dtype=np.uint32); S = np.array([[r[3] for r in rows]], dtype=np.float32)
    return S, doc, field, chunk


def test_mask_bits():
    assert passes(0, 5) and passes(0b10, 1) and not passes(0b10, 0)


def test_chunks_on_both_sides_of_the_list_edge():
    S, doc, field, chunk = _case()
    # k = 2: doc 0's field-0 chunk is first; its field-1 chunk (0.10) is below the edge and must not replace it
    (hits, obs), = search_fields(S, doc, field, chunk, 2, [0])
    assert [(h[0], h[2], h[3]) for h in hits] == [(0, 0, 0), (1, 1, 3)] and obs == 7
    # only field 1: doc 0 survives through its weak chunk, below the others
    (hits, obs), = search_fields(S, doc, field, chunk, 4, [0b10])
    assert [(h[0], h[2], h[3]) for h in hits] == [(1, 1, 3), (2, 1, 0), (0, 1, 0)] and obs == 4
    assert abs(hits[2][1] - 0.10) < 1e-6


def test_equal_scores_inside_a_doc_keep_the_earliest_row():
    S, doc, field, chunk = _case()
    (hits, _), = search_fields(S, doc, field, chunk, 10, [0b10])
    assert (2, 1, 0) in [(h[0], h[2], h[3]) for h in hits]         # rows (2, 1, 0) and (2, 1, 1) tie at 0.70: chunk 0 comes first


def test_mask_selecting_no_row():
    S, doc, field, chunk = _case()
    (hits, obs), = search_fields(S, doc, field, chunk, 10, [1 << 7])
    assert hits == [] and obs == 0


def test_threshold():
    S, doc, field, chunk = _case()
    (hits, _), = search_fields(S, doc, field, chunk, 10, [0b01], threshold=np.float32(0.75))
    assert [(h[0], h[2]) for h in hits] == [(0, 0), (1, 0)]
    assert threshold_premap(0.5, False) == np.float32(0.0) and threshold_premap(0.3, True) == np.float32(-0.3)


def test_deleted_doc_whose_other_chunk_is_best():
    S, doc, field, chunk = _case()
    # doc 1's best row is its field-1 chunk; deleting doc 1 removes both rows (deletion is per doc), observed still counts them
    (hits, obs), = search_fields(S, doc, field, chunk, 10, [0], deleted=[1])
    assert 1 not in [h[0] for h in hits] and obs == 7
    (hits, _), = search_fields(S, doc, field, chunk, 10, [0b01], deleted=[0])
    assert [(h[0], h[2], h[3]) for h in hits] == [(1, 0, 0)]


def test_ivf_scope():
    S, doc, field, chunk = _case()
    scope = np.array([[True, True, True, True, False, False, False]])
    (hits, obs), = search_fields(S, doc, field, chunk, 10, [0b10], in_scope=scope)
    assert [h[0] for h in hits] == [1, 0] and obs == 2


def test_restatement_equals_the_reference_topk_without_ties():
    rng = np.random.default_rng(5)
    n = 400
    doc = rng.integers(0, 90, n); field = rng.integers(0, 3, n).astype(np.uint8); chunk = rng.integers(0, 4, n).astype(np.uint32)
    S = rng.standard_normal((6, n)).astype(np.float32)               # continuous scores: no ties
    masks = [0, 1, 2, 3, 4, 1 << 9]
    thr = np.float32(-0.5)
    for k in (1, 5, 10, 32):
        a = search_fields(S, doc, field, chunk, k, masks, deleted=[3, 17], threshold=thr)
        b = search_fields_topk(S, doc, field, chunk, k, masks, deleted=[3, 17], threshold=thr)
        for (ha, oa), (hb, ob) in zip(a, b):
            assert oa == ob
            assert [(h[0], h[2], h[3]) for h in ha] == [(h[0], h[2], h[3]) for h in hb]


def test_topk_push_replaces_only_on_a_better_score():
    t = TopK(2)
    t.push(7, 0, 0, np.float32(0.5)); t.push(7, 1, 2, np.float32(0.5)); t.push(7, 2, 1, np.float32(0.4))
    assert t.result() == [(7, np.float32(0.5), 0, 0)]


def test_vector_bin_writer_with_fields():
    rng = np.random.default_rng(1)
    rows = rng.standard_normal((5, 8)).astype(np.float32)
    ids = np.array([0, 0, 1, 2, 2], dtype=np.uint16)
    fields = np.array([0, 2, 1, 31, 0], dtype=np.uint8); chunks = np.array([0, 1, 0, 7, 70000], dtype=np.uint32)
    data = write_vector_bin_fields([(ids, rows, fields, chunks, [2, 3])])
    assert read_vector_bin_headers(data, 8) == list(zip(ids.tolist(), fields.tolist(), chunks.tolist()))
    assert len(data) == 4 + 8 + 5 * (24 + 32)
    # zero field / chunk ids are today's bytes
    zeros = np.zeros(5, dtype=np.uint32)
    assert write_vector_bin_fields([(ids, rows, zeros, zeros)]) == write_vector_bin([(ids, rows)])


def test_tagged_corpus_shape():
    rows, ids, fields, chunks = tagged_corpus(20, 16, 3)
    assert rows.shape == (len(ids), 16) and rows.dtype == np.float32
    for d in range(20):
        sel = ids == d
        assert set(fields[sel].tolist()) == {0, 1, 2}
        for f in range(3):
            c = chunks[sel & (fields == f)]
            assert list(c) == list(range(len(c))) and 1 <= len(c) <= 3


def test_vectorised_restatement_equals_the_loop():
    from helpers_vecfields import search_fields_fast
    rng = np.random.default_rng(0)
    n = 500
    doc = rng.integers(0, 60, n); field = rng.integers(0, 3, n).astype(np.uint8); chunk = rng.integers(0, 5, n).astype(np.uint32)
    S = np.round(rng.standard_normal((5, n)), 1).astype(np.float32)     # rounded: many equal scores inside and across docs
    dr = np.isin(doc, [3, 4])
    for m in (0, 1, 6, 1 << 9):
        for q in range(5):
            (a, oa), = search_fields(S[q:q + 1], doc, field, chunk, 10, [m], deleted=[3, 4], threshold=np.float32(-0.5))
            b, ob = search_fields_fast(S[q], doc, field, chunk, 10, m, dr, np.float32(-0.5))
            assert oa == ob and [(h[0], h[2], h[3]) for h in a] == [(h[0], h[2], h[3]) for h in b]
