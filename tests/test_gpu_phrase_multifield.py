"""GPU: QueryType::Phrase on an index with several indexed fields (add_result.rs:3247-3389) — per posting one position run per field, the
phrase checked inside each field on its own (never across two fields), a field filter limiting the fields searched.  Ids, scores and counts
== the CPU oracle (whose matches equal a substring search inside one field, tests/test_phrase_multifield_cpu.py) for 2, 3 and 4 fields with
boosts: Topk / TopkCount / Count, field filters, a facet filter, a delete set, paging to k = 100, and the public Index.search call."""
import numpy as np
import pytest

from oracle import oracle as O
from helpers import query_keys
from helpers_phrase_mf import PhraseFieldsOracle, contains_phrase_fields, levels_from_docs, multifield_sequence_corpus, phrase_queries_mf

pytestmark = pytest.mark.gpu

BOOSTS = {2: (2.0, 1.0), 3: (3.0, 1.0, 0.5), 4: (1.0, 1.5, 0.75, 1.0)}


def _indexes(levels, n, ls, boosts):
    from seekstorm_b200 import Index
    ix = Index(0)
    ix.set_field_boosts(boosts)
    for lv in levels:
        ix.add_lexical_level(lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"], lv["doc_len_bytes"],
                             lv["positions"])
    ix.commit(n, ls)
    return ix, PhraseFieldsOracle(levels, n, ls, boosts)


@pytest.mark.parametrize("n_fields", [2, 3, 4])
def test_multifield_phrase_parity(n_fields):
    from seekstorm_b200 import FacetFilter, QueryType, ResultType, SearchMode
    n, vocab = 72000, 200
    docs, levels, ls = multifield_sequence_corpus(n, vocab, n_fields, seed=60 + n_fields)
    assert len(levels) == 2
    ix, orc = _indexes(levels, n, ls, BOOSTS[n_fields])
    phrases = phrase_queries_mf(docs, 70 + n_fields, 120, vocab)
    phrases.append([3, 100000])                                       # a term that is not in the dictionary -> no hit
    phrases.append([7])                                               # one token: a plain term query
    qk = query_keys(phrases)
    qk[-2][1] = 0xDEAD0008
    rng = np.random.default_rng(80 + n_fields)
    masks = [int(rng.integers(1, 1 << n_fields)) if rng.random() < 0.7 else 0 for _ in qk]
    errs, n_hit, n_masked_hit = [], 0, 0
    for deleted in ([], [int(x) for x in rng.integers(0, n, 2500)]):
        ix.set_deleted(deleted); orc.set_deleted(deleted)
        for fm in (None, masks):
            got, cnt = ix.search_lexical_batch(qk, QueryType.Phrase, 10, ResultType.TopkCount, field_masks=fm)
            got_t, _ = ix.search_lexical_batch(qk, QueryType.Phrase, 10, ResultType.Topk, field_masks=fm)
            _, cnt_c = ix.search_lexical_batch(qk, QueryType.Phrase, 0, ResultType.Count, field_masks=fm)
            for i, k in enumerate(qk):
                m = fm[i] if fm else 0
                want, tot = orc.search_phrase(k, 10, O.RESULT_TOPKCOUNT, field_mask=m)
                n_hit += tot > 0
                n_masked_hit += tot > 0 and m != 0
                if got[i] != want or got_t[i] != want or int(cnt[i]) != tot or int(cnt_c[i]) != tot:
                    errs.append((bool(deleted), m, i, phrases[i], got[i][:2], want[:2], int(cnt[i]), int(cnt_c[i]), tot))
    assert not errs, (len(errs), errs[:5])
    assert n_hit > 250 and n_masked_hit > 50
    ix.set_deleted([]); orc.set_deleted([])
    # ground truth straight from the token sequences, for a few phrases
    for i in range(4):
        _, cnt = ix.search_lexical_batch(qk[i:i + 1], QueryType.Phrase, 0, ResultType.Count, field_masks=[masks[i]])
        assert int(cnt[0]) == sum(contains_phrase_fields(d, phrases[i], masks[i]) for d in docs)
    # paging beyond 32 hits: a frequent bigram, without and with a field filter
    big = query_keys([[0, 1]])
    for m in (0, 2):
        got, cnt = ix.search_lexical_batch(big, QueryType.Phrase, 100, ResultType.TopkCount, field_masks=[m])
        want, tot = orc.search_phrase(big[0], 100, O.RESULT_TOPKCOUNT, field_mask=m)
        assert got[0] == want and int(cnt[0]) == tot and tot > 100, (m, tot)
    # a facet filter on the same candidates as the phrase check and the field filter
    price = rng.integers(0, 100, n, dtype=np.uint32)
    ix.set_facets({"price": price})
    for m in (0, 1):
        got, cnt = ix.search_lexical_batch(big, QueryType.Phrase, 20, ResultType.TopkCount, filters=[[FacetFilter("price", 10, 40)]], field_masks=[m])
        allw, _ = orc.search_phrase(big[0], n, O.RESULT_TOPKCOUNT, field_mask=m)
        keep = [(d, s) for d, s in allw if 10 <= price[(d >> 16) * 65536 + (d & 0xFFFF)] < 40]
        assert got[0] == keep[:20] and int(cnt[0]) == len(keep)
    ix.set_facets({})
    # the public call: a quoted query string with a field filter by name and by index
    for ff, m in (((), 0), (("field1",), 2), ((0,), 1)):
        want, tot = orc.search_phrase(big[0], 10, O.RESULT_TOPKCOUNT, field_mask=m)
        ro = ix.search('"t0 t1"', None, QueryType.Union, SearchMode.Lexical(), False, 0, 10, ResultType.TopkCount, field_filter=list(ff))
        assert [(r.doc_id, np.float32(r.score)) for r in ro.results] == [(d, np.float32(s)) for d, s in want] and ro.result_count_total == tot
    with pytest.raises(NotImplementedError):                         # NOT terms next to a phrase
        ix.search("t0 t1 -t2", None, QueryType.Phrase, SearchMode.Lexical(), False, 0, 10, ResultType.TopkCount, field_filter=[0])
    ix.close()


def test_multifield_phrase_traps_on_the_gpu():
    """the hand-made cases of the CPU test through the device check: positions restart per field, no phrase across the field boundary,
    terms spread over fields, repeated tokens, a field filter that excludes / includes the only field holding the phrase"""
    from seekstorm_b200 import QueryType, ResultType
    docs = [
        [[9, 9, 9, 1], [9, 9, 9, 9, 2]],
        [[5, 6, 3], [4, 7]],
        [[10, 12], [11, 12]],
        [[9], [20, 21, 22, 23, 20, 21]],
        [[40, 41], [9, 9]],
        [[9, 9], [40, 9, 41]],
    ] + [[[9, 8, 9], [8, 9, 8, 9]] for _ in range(20)]
    levels, ls = levels_from_docs(docs, 2)
    ix, orc = _indexes(levels, len(docs), ls, (2.0, 1.0))
    cases = [([1, 2], 0, []), ([3, 4], 0, []), ([10, 11], 0, []), ([10, 12], 0, [2]), ([20, 21, 22, 23, 20, 21], 0, [3]),
             ([23, 20, 21], 0, [3]), ([20, 21, 20, 21], 0, []), ([40, 41], 0, [4]), ([40, 41], 2, []), ([40, 41], 1, [4]), ([20, 21], 1, [])]
    got, cnt = ix.search_lexical_batch(query_keys([c[0] for c in cases]), QueryType.Phrase, 10, ResultType.TopkCount, field_masks=[c[1] for c in cases])
    for i, (ph, m, want) in enumerate(cases):
        w, tot = orc.search_phrase(query_keys([ph])[0], 10, O.RESULT_TOPKCOUNT, field_mask=m)
        assert [d for d, _ in got[i]] == want and got[i] == w and int(cnt[i]) == tot == len(want), (ph, m, got[i], want)
    ix.close()


def test_multifield_positions_contract_errors():
    from seekstorm_b200 import Index, SsbError
    docs, levels, ls = multifield_sequence_corpus(3000, 50, 3, seed=90)
    lv = levels[0]
    args = (lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"], lv["doc_len_bytes"])
    ix = Index(0)
    ix.set_field_boosts(BOOSTS[3])
    with pytest.raises(SsbError):                                      # one position short of Σ tfs
        ix.add_lexical_level(*args, lv["positions"][:-1].copy())
    # a run that does not ascend inside one field: swap two positions of the first posting with >= 2 occurrences in one field
    tfs = lv["tfs"].astype(np.int64)
    j, f = map(int, np.argwhere(tfs >= 2)[0])
    start = int(tfs[:j].sum() + tfs[j, :f].sum())
    bad = lv["positions"].copy()
    bad[start], bad[start + 1] = bad[start + 1], bad[start]
    with pytest.raises(SsbError):
        ix.add_lexical_level(*args, bad)
    # runs that ascend per field but not across fields are valid (every field restarts from 0)
    ix.add_lexical_level(*args, lv["positions"])
    ix.commit(lv["n_docs"], ls)
    ix.close()
