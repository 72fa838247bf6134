"""GPU: n-gram phrases through the facet filter, result_sort and query_facets (the sorted plan, packed sort bounds and lex_facets read the
n-gram components and bounds), an index.bin with n-gram keys loaded against the neutral layout under both df rules, and the sharded / mixing
refusals; against the restated reference in tests/helpers_ngram.py."""
import ctypes

import numpy as np
import pytest

from seekstorm_b200 import Index, LexicalSimilarity, QueryType, ResultType, SsbError, _lib

import helpers_ngram as H
from test_gpu_zzzzzzngram import ALL7, FREQ, build, corpus, phrases, rewrite_keys  # noqa: F401  (corpus: the shared fixture)

pytestmark = pytest.mark.gpu


# ---- facet filter, result_sort and query_facets on n-gram phrases (the sorted plan, packed sort bounds and lex_facets read the n-gram
# components and bounds too)
def _price_column(levels, seed):
    rng = np.random.default_rng(seed)
    rows = ((len(levels) - 1) << 16) + levels[-1]["n_docs"]
    return rng.integers(0, 100, rows).astype(np.uint32)


def _ngram_queries(docs):
    qs = [q for q in phrases(docs, 30, 41)] + [[0, 1], [0, 1, 2], [1, 2, 0, 1]]
    return [rewrite_keys(q) for q in qs]


def test_facet_filter_sort_and_counts(corpus):
    from seekstorm_b200 import FacetFilter, QueryFacet, ResultSort, SortOrder
    docs, levels, len_sum, stats = corpus
    ix = build(corpus, LexicalSimilarity.Bm25f, 0)
    price = _price_column(levels, 5)
    ix.set_facets({"price": price})
    keys = _ngram_queries(docs)
    assert any(any(k & 7 for k in ks) for ks in keys)
    full = [H.phrase_oracle(docs, levels, len_sum, stats, ks, 0, 0) for ks in keys]
    # a range filter
    flt = [[FacetFilter("price", start=20, end=70)] for _ in keys]
    res, cnt = ix.search_lexical_batch(keys, QueryType.Phrase, 40, ResultType.TopkCount, filters=flt)
    for i in range(len(keys)):
        want = [(d, s) for d, s in full[i] if 20 <= price[d] < 70]
        assert int(cnt[i]) == len(want)
        assert [(d, np.float32(s)) for d, s in res[i]] == want[:40]
    # result_sort: price descending, then score descending, then doc id ascending
    for order in (SortOrder.Descending, SortOrder.Ascending):
        res, cnt = ix.search_lexical_batch(keys, QueryType.Phrase, 40, ResultType.TopkCount, sort=[ResultSort("price", order)])
        for i in range(len(keys)):
            sgn = -1 if order == SortOrder.Descending else 1
            want = sorted(full[i], key=lambda x: (sgn * int(price[x[0]]), -float(x[1]), x[0]))
            assert int(cnt[i]) == len(full[i])
            assert [(d, np.float32(s)) for d, s in res[i]] == want[:40], i
    # query_facets: range counts over every match
    edges = [0, 10, 25, 50, 90]
    qf = [QueryFacet("price", ranges=[(f"r{e}", e) for e in edges])]
    raw = ix.search_lexical_facets(keys, QueryType.Phrase, qf)
    for i in range(len(keys)):
        want = [0] * len(edges)
        for d, _ in full[i]:
            want[int(np.searchsorted(edges, price[d], side="right")) - 1] += 1
        got = [c for _, c in raw[i]["price"]] if raw[i]["price"] and isinstance(raw[i]["price"][0], tuple) else list(raw[i]["price"])
        assert got == want, (i, raw[i]["price"], want)
    ix.close()


# ---- index.bin with n-gram keys, loaded against the neutral layout
@pytest.fixture(scope="module")
def two_level_corpus():
    return H.ngram_corpus(65536 + 2500, 30, 13, FREQ, ALL7, docs_per_level=65536, mean_len=6)


@pytest.mark.parametrize("rule", [_lib.NGRAM_DF_FIRST_LEVEL, _lib.NGRAM_DF_LAST_LEVEL])
def test_loaded_index_bin_matches_neutral_layout(two_level_corpus, rule):
    import refwriter_ngram as RN
    docs, levels, len_sum, stats = two_level_corpus
    n = sum(lv["n_docs"] for lv in levels)
    data, cum = RN.write_index_bin_ngrams(levels, n, 23)
    assert cum == len_sum
    ixl = Index(0)
    ixl.set_ngram_config(frequent_terms={H.word(t) for t in FREQ}, ngram_set=ALL7, similarity=LexicalSimilarity.Bm25f, df_rule=rule)
    assert ixl.load_index_bin(data, key_head_size=23, decode_positions=True, ngrams=True) == n
    ixn = build(two_level_corpus, LexicalSimilarity.Bm25f, rule)
    assert ixl.dict_export()[0].tolist() == ixn.dict_export()[0].tolist()
    qs = phrases(docs, 30, 51 + rule)
    keys = [rewrite_keys(q) for q in qs]
    # the two levels give some n-gram keys different df bytes: the rule matters for them
    assert any(len(set(map(tuple, b))) > 1 for b in stats["dfb"].values())
    rl, cl = ixl.search_lexical_batch(keys, QueryType.Phrase, 20, ResultType.TopkCount)
    rn, cn = ixn.search_lexical_batch(keys, QueryType.Phrase, 20, ResultType.TopkCount)
    assert rl == rn and cl.tolist() == cn.tolist()
    for i, ks in enumerate(keys[:12]):
        want = H.phrase_oracle(docs, levels, len_sum, stats, ks, 0, rule)
        assert int(cl[i]) == len(want) and [(d, np.float32(s)) for d, s in rl[i]] == want[:20]
    ixl.close(); ixn.close()


def test_sharded_refusals_and_mixing(corpus):
    docs, levels, len_sum, stats = corpus
    lv = levels[0]
    L = _lib.lib()
    # a handle that already has a (borrowed, never used) communicator of world 2 refuses n-gram levels and n-gram index.bin loads
    ix = Index(0)
    assert L.ssb_comm_attach(ix._h, ctypes.c_void_p(0x1000), 0, 2) == 0
    with pytest.raises(SsbError):
        ix.add_lexical_level(lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"], lv["doc_len_bytes"],
                             lv["positions"], lv["ngram_tfs"], lv["ngram_df_bytes"])
    assert L.ssb_lexical_add_level_ngrams is not None
    assert L.ssb_comm_destroy(ix._h) == 0
    ix.close()
    # an index with n-gram lists refuses a communicator of world > 1 (init checks before it touches NCCL) and plain levels with n-gram keys
    ix = build(corpus, LexicalSimilarity.Bm25f, 0)
    ident = (ctypes.c_uint8 * 128)()
    assert L.ssb_comm_init(ix._h, ident, 0, 2) == -5
    assert L.ssb_comm_attach(ix._h, ctypes.c_void_p(0x1000), 0, 2) == -5
    assert L.ssb_lexical_sync_df(ix._h) == 0                         # no communicator: nothing to synchronise
    lv2 = dict(levels[-1]); lv2["level_id"] = 10
    with pytest.raises(SsbError, match="low bits"):
        ix.add_lexical_level(lv2["level_id"], lv2["n_docs"], lv2["term_keys"], lv2["posting_offsets"], lv2["doc_ids"], lv2["tfs"],
                             lv2["doc_len_bytes"], lv2["positions"])
    ix.close()
    # and the other order: a plain level with n-gram keys first, then an n-gram level
    ix = Index(0)
    ix.add_lexical_level(lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"], lv["doc_len_bytes"],
                         lv["positions"])
    lv3 = levels[1]
    with pytest.raises(SsbError, match="low bits"):
        ix.add_lexical_level(lv3["level_id"], lv3["n_docs"], lv3["term_keys"], lv3["posting_offsets"], lv3["doc_ids"], lv3["tfs"],
                             lv3["doc_len_bytes"], lv3["positions"], lv3["ngram_tfs"], lv3["ngram_df_bytes"])
    ix.close()
