"""GPU: phrase search over n-gram posting lists (ssb_lexical_add_level_ngrams) against the restated reference in tests/helpers_ngram.py:
ids, counts and bit-exact scores for both similarities and both df-level rules, the match sets of the SingleTerm-only index and of a
substring search, the delete set, paging beyond 32, the Index.search rewrite, and the multi-field / sharded refusals."""
import ctypes

import numpy as np
import pytest

from seekstorm_b200 import Index, LexicalSimilarity, NgramSet as S, QueryType, ResultType, SsbError, _lib, ngram_key, ngram_rewrite

import helpers_ngram as H

pytestmark = pytest.mark.gpu

FREQ = set(range(8))                                  # token ids 0..7 are the frequent terms
ALL7 = S.NgramFF | S.NgramFR | S.NgramRF | S.NgramFFF | S.NgramRFF | S.NgramFFR | S.NgramFRF


@pytest.fixture(scope="module")
def corpus():
    return H.ngram_corpus(6000, 60, 11, FREQ, ALL7, docs_per_level=1500)


def build(corpus, sim, rule, ngrams=True):
    docs, levels, len_sum, stats = corpus
    ix = Index(0)
    if ngrams:
        ix.set_ngram_config(frequent_terms={H.word(t) for t in FREQ}, ngram_set=ALL7, similarity=sim, df_rule=rule)
    for lv in (levels if ngrams else H.single_term_levels(levels)):
        ix.add_lexical_level(lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"],
                             lv["doc_len_bytes"], lv["positions"], lv.get("ngram_tfs") if ngrams else None,
                             lv.get("ngram_df_bytes") if ngrams else None)
    ix.commit(sum(lv["n_docs"] for lv in levels), len_sum)
    return ix


def phrases(docs, n, seed):
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        d = docs[int(rng.integers(0, len(docs)))]
        m = int(rng.integers(2, 7))
        if len(d) >= m:
            s = int(rng.integers(0, len(d) - m + 1))
            out.append([int(x) for x in d[s:s + m]])
    out += [[0, 1], [1, 0, 2], [0, 1, 0, 1, 0], [2, 50, 3], [40, 41, 3, 4]]
    return out


def rewrite_keys(ph):
    return [ngram_key(w, t) for w, t in ngram_rewrite([H.word(x) for x in ph], {H.word(t) for t in FREQ}, ALL7)]


@pytest.mark.parametrize("sim", [LexicalSimilarity.Bm25f, LexicalSimilarity.Bm25fProximity])
@pytest.mark.parametrize("rule", [_lib.NGRAM_DF_FIRST_LEVEL, _lib.NGRAM_DF_LAST_LEVEL])
def test_phrase_against_oracle(corpus, sim, rule):
    docs, levels, len_sum, stats = corpus
    ix = build(corpus, sim, rule)
    qs = phrases(docs, 40, 5 + rule)
    keys = [rewrite_keys(q) for q in qs]
    assert any(any(k & 7 for k in ks) for ks in keys) and any(len(ks) >= 2 for ks in keys)
    k = 10
    res_tc, cnt_tc = ix.search_lexical_batch(keys, QueryType.Phrase, k, ResultType.TopkCount)
    res_t, _ = ix.search_lexical_batch(keys, QueryType.Phrase, k, ResultType.Topk)
    _, cnt_c = ix.search_lexical_batch(keys, QueryType.Phrase, 0, ResultType.Count)
    for i, ks in enumerate(keys):
        want = H.phrase_oracle(docs, levels, len_sum, stats, ks, int(sim), rule)
        assert int(cnt_tc[i]) == len(want) and int(cnt_c[i]) == len(want), (qs[i], ks)
        for got in (res_tc[i], res_t[i]):
            assert [d for d, _ in got] == [d for d, _ in want[:k]], qs[i]
            assert [np.float32(s) for _, s in got] == [s for _, s in want[:k]], qs[i]
    ix.close()


def test_match_sets_equal_single_term_index_and_substring(corpus):
    docs, levels, len_sum, stats = corpus
    ixn = build(corpus, LexicalSimilarity.Bm25f, 0)
    ixs = build(corpus, LexicalSimilarity.Bm25f, 0, ngrams=False)
    qs = phrases(docs, 30, 21)
    k = 1024
    rn, cn = ixn.search_lexical_batch([rewrite_keys(q) for q in qs], QueryType.Phrase, k, ResultType.TopkCount)
    rs, cs = ixs.search_lexical_batch([[ngram_key((H.word(x),), 0) for x in q] for q in qs], QueryType.Phrase, k, ResultType.TopkCount)
    for i, q in enumerate(qs):
        want = set()
        for li, lv in enumerate(levels):
            for d in range(lv["n_docs"]):
                doc = docs[li * 1500 + d]
                m = len(q)
                if any(all(doc[s + j] == q[j] for j in range(m)) for s in range(len(doc) - m + 1)):
                    want.add((li << 16) | d)
        assert int(cn[i]) == int(cs[i]) == len(want), q
        if len(want) <= k:
            assert {d for d, _ in rn[i]} == {d for d, _ in rs[i]} == want, q
    ixn.close(); ixs.close()


def test_delete_set_and_paging(corpus):
    docs, levels, len_sum, stats = corpus
    ix = build(corpus, LexicalSimilarity.Bm25f, 1)
    key = rewrite_keys([0, 1])
    assert len(key) == 1 and key[0] & 7 == 1
    q = [rewrite_keys([0, 1, 2, 3]), key, rewrite_keys([1, 0])]
    full = [H.phrase_oracle(docs, levels, len_sum, stats, ks, 0, 1) for ks in q]
    deleted = [d for d, _ in full[1][::3]]
    ix.set_deleted(deleted)
    k = 100
    res, cnt = ix.search_lexical_batch(q, QueryType.Phrase, k, ResultType.TopkCount)
    for i, ks in enumerate(q):
        want = H.phrase_oracle(docs, levels, len_sum, stats, ks, 0, 1, deleted=deleted)
        assert int(cnt[i]) == len(want)
        assert [(d, np.float32(s)) for d, s in res[i]] == want[:k]
    assert len(full[1]) > 64
    ix.close()


def test_index_search_rewrites_phrases(corpus):
    docs, levels, len_sum, stats = corpus
    ix = build(corpus, LexicalSimilarity.Bm25f, 0)
    q = [0, 1, 2, 0, 1, 2]
    ro = ix.search('"' + " ".join(H.word(x) for x in q) + '"', length=50)
    want = H.phrase_oracle(docs, levels, len_sum, stats, rewrite_keys(q), 0, 0)
    assert ro.result_count_total == len(want)
    assert [(r.doc_id, np.float32(r.score)) for r in ro.results] == want[:50]
    assert ro.query_terms == [H.word(0), H.word(1), H.word(2)]
    ix.close()


def test_refusals(corpus):
    docs, levels, len_sum, stats = corpus
    lv = levels[0]
    ix = Index(0)
    ix.set_field_boosts([1.0, 2.0])
    tfs2 = np.stack([lv["tfs"], np.zeros_like(lv["tfs"])], axis=1).copy()
    lb2 = np.concatenate([lv["doc_len_bytes"], lv["doc_len_bytes"]])
    with pytest.raises(SsbError):
        ix.add_lexical_level(0, lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], tfs2, lb2, lv["positions"],
                             lv["ngram_tfs"], lv["ngram_df_bytes"])
    ix.close()
    ix = build(corpus, LexicalSimilarity.Bm25f, 0)
    assert _lib.lib().ssb_comm_attach(ix._h, ctypes.c_void_p(0x1000), 0, 2) == -5        # SSB_E_UNSUPPORTED
    with pytest.raises(SsbError):
        ix.set_ngram_config(similarity=LexicalSimilarity.Bm25f)                          # after the first level: SSB_E_STATE
    ix.close()
