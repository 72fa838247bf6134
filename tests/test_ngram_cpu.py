"""CPU: the n-gram query rewrite (tokenizer.rs:898-1387), the n-gram key composition (tokenizer.rs:678-685) and known-answer BM25 of
n-gram lists under both similarities (add_result.rs:1448-1478, search.rs:3221-3269), on the restatement in tests/helpers_ngram.py."""
import numpy as np
import pytest

from seekstorm_b200 import NgramSet as S, NgramType as T, ngram_key, ngram_rewrite
from seekstorm_b200.index import fnv1a64
from seekstorm_b200 import synth

import helpers_ngram as H

FREQUENT = {"the", "who", "is", "to", "be", "or", "not", "it", "up"}


def rw(q, ngram_set):
    return [("_".join(w), T(t).name) for w, t in ngram_rewrite(q.split(), FREQUENT, ngram_set)]


@pytest.mark.parametrize("ngram_set, want", [
    (S.SingleTerm, [("to", "SingleTerm"), ("be", "SingleTerm"), ("or", "SingleTerm"), ("not", "SingleTerm"), ("to", "SingleTerm"), ("be", "SingleTerm")]),
    (S.NgramFF, [("to_be", "NgramFF"), ("or_not", "NgramFF"), ("to_be", "NgramFF")]),
    (S.NgramFF | S.NgramFFF, [("to_be_or", "NgramFFF"), ("not_to_be", "NgramFFF")]),
    (S.NgramFFF, [("to_be_or", "NgramFFF"), ("not_to_be", "NgramFFF")]),
    (S.NgramFF | S.NgramFR | S.NgramRF | S.NgramFFF, [("to_be_or", "NgramFFF"), ("not_to_be", "NgramFFF")]),
])
def test_rewrite_to_be_or_not_to_be(ngram_set, want):
    assert rw("to be or not to be", ngram_set) == want


@pytest.mark.parametrize("q, ngram_set, want", [
    ("the who", S.NgramFF, [("the_who", "NgramFF")]),
    ("who is who", S.NgramFF | S.NgramFFF, [("who_is_who", "NgramFFF")]),
    ("who is who", S.NgramFF, [("who_is", "NgramFF"), ("who", "SingleTerm")]),
    ("let it be", S.NgramFF, [("let", "SingleTerm"), ("it_be", "NgramFF")]),
    ("let it be", S.NgramRF | S.NgramFF, [("let_it", "NgramRF"), ("be", "SingleTerm")]),
    ("let it be", S.NgramRFF | S.NgramFF, [("let_it_be", "NgramRFF")]),
    ("tallest trees in the world", S.NgramFF, [("tallest", "SingleTerm"), ("trees", "SingleTerm"), ("in", "SingleTerm"), ("the", "SingleTerm"),
                                               ("world", "SingleTerm")]),
    ("the tallest who", S.NgramFRF, [("the_tallest_who", "NgramFRF")]),
    ("the who tallest", S.NgramFFR, [("the_who_tallest", "NgramFFR")]),
    ("the tallest", S.NgramFR, [("the_tallest", "NgramFR")]),
    ("tallest trees", S.NgramFF | S.NgramFR | S.NgramRF, [("tallest", "SingleTerm"), ("trees", "SingleTerm")]),
    # trigrams before bigrams, left to right: "up" binds into the first trigram, not the later bigram
    ("up to be it", S.NgramFF | S.NgramFFF, [("up_to_be", "NgramFFF"), ("it", "SingleTerm")]),
])
def test_rewrite_greedy(q, ngram_set, want):
    assert rw(q, ngram_set) == want


def test_index_time_quirk_ffr_frf_under_rff_bit():
    """FFR / FRF lists are generated when the RFF bit is set (tokenizer.rs:817, 850), but looked up under their own bits at query time"""
    fr = {1, 2}
    g = H.index_ngrams([1, 2, 9, 1, 9, 2], fr, S.NgramRFF)
    types = sorted({int(t) for (_, t) in g if t})
    assert types == [T.NgramFFR, T.NgramFRF]
    assert H.index_ngrams([1, 2, 9], fr, S.NgramFFR) .keys() == {((H.word(x),), T.SingleTerm) for x in (1, 2, 9)}


def test_ngram_key():
    assert ngram_key(("the", "who"), T.NgramFF, fnv1a64) == fnv1a64("the who") | 1
    k = ngram_key(("t1", "t2", "t3"), T.NgramFRF)
    assert k & 7 == 7 and k >> 3 == fnv1a64("t1 t2 t3") >> 3
    assert ngram_key(("t5",), T.SingleTerm) == synth.term_keys_np(np.array([5]))[0]


def test_bm25_bigram_known_answer():
    """N = 1000 docs, doc length byte 40 under avgdl 50; components 'the' df 900 (byte4 code), 'who' df 7; tfs 3 and 1"""
    n, len_sum = 1000, 50000
    cache = H.bm25_cache(n, len_sum)
    b = 40
    dl = synth.byte4_to_int(b)
    bc64 = 1.2 * (0.25 + 0.75 * dl / 50.0)
    assert abs(float(cache[b]) - bc64) < 1e-6
    df1, df2 = synth.byte4_to_int(synth.int_to_byte4(900)), synth.byte4_to_int(synth.int_to_byte4(7))
    idf64 = [np.log((n - d + 0.5) / (d + 0.5) + 1.0) for d in (df1, df2)]
    want = sum(i * t * 2.2 / (t + bc64) for i, t in zip(idf64, (3, 1)))
    idfs = [H.idf(n, df1), H.idf(n, df2)]
    got = H.ngram_component_sum(idfs, [3, 1], cache[b])
    assert abs(float(got) - want) < 2e-6 * want
    # the f32 restatement: products first, then the sum (no contraction)
    assert got == np.float32(idfs[0] * H.part(3, cache[b])) + np.float32(idfs[1] * H.part(1, cache[b]))


def test_bm25_trigram_known_answer_distinct_components():
    """a trigram with three distinct component tfs (4, 2, 1) and dfs (600, 40, 3): the sum ((c1 + c2) + c3) in word order"""
    n, len_sum = 5000, 5000 * 30
    cache = H.bm25_cache(n, len_sum)
    bc = cache[30]
    dfs = [synth.byte4_to_int(synth.int_to_byte4(d)) for d in (600, 40, 3)]
    idfs = [H.idf(n, d) for d in dfs]
    got = H.ngram_component_sum(idfs, [4, 2, 1], bc)
    parts = [np.float32(i * H.part(t, bc)) for i, t in zip(idfs, (4, 2, 1))]
    assert got == np.float32(np.float32(parts[0] + parts[1]) + parts[2])
    bc64 = float(bc)
    want = sum(np.log((n - d + 0.5) / (d + 0.5) + 1.0) * t * 2.2 / (t + bc64) for d, t in zip(dfs, (4, 2, 1)))
    assert abs(float(got) - want) < 2e-6 * want
    # the components are not interchangeable: word order decides which tf meets which idf
    assert H.ngram_component_sum(idfs, [1, 2, 4], bc) != got


def test_proximity_single_field_adds_zero():
    """Bm25fProximity fills only `idf` of an n-gram list (search.rs:3221-3230); the single-field scorer reads idf_ngram* (0.0) for it:
    a phrase that rewrites to n-grams only scores 0 on every match"""
    fr = {1, 2}
    docs_, levels, len_sum, stats = H.ngram_corpus(40, 6, 3, fr, S.NgramFF, docs_per_level=20)
    key = ngram_key((H.word(1), H.word(2)), T.NgramFF)
    res = H.phrase_oracle(docs_, levels, len_sum, stats, [key], 1, 0)
    assert res and all(s == 0.0 for _, s in res)
    res_f = H.phrase_oracle(docs_, levels, len_sum, stats, [key], 0, 0)
    assert [d for d, _ in res_f] and all(s > 0.0 for _, s in res_f)
    assert sorted(d for d, _ in res) == sorted(d for d, _ in res_f)
