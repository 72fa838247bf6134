"""CPU oracle: phrase queries on an index with several indexed fields (add_result.rs:3247-3389).  A posting's positions are one run per field,
each restarting from 0; the phrase must occur inside one field, and with a field filter inside one field of the filter.  The oracle
(helpers_phrase_mf.PhraseFieldsOracle: the C oracle's BM25F intersection + the phrase condition read from the levels' position layout) equals
a substring search over the token sequences, on random corpora with 2, 3 and 4 fields and on hand-made traps; on one field it equals the C
oracle's single-field phrase search."""
import numpy as np
import pytest

from oracle import oracle as O
from helpers import query_keys
from helpers_phrase import sequence_corpus
from helpers_phrase_mf import PhraseFieldsOracle, contains_phrase_fields, levels_from_docs, multifield_sequence_corpus, phrase_queries_mf

BOOSTS = {2: (2.0, 1.0), 3: (3.0, 1.0, 0.5), 4: (1.0, 1.5, 0.75, 1.0)}


def _oracle(levels, n, ls, boosts):
    return PhraseFieldsOracle(levels, n, ls, boosts)


def _doc_id(i, per_level):
    return ((i // per_level) << 16) | (i % per_level)


@pytest.mark.parametrize("n_fields", [2, 3, 4])
def test_oracle_matches_substring_truth(n_fields):
    n, vocab, per_level = 3000, 30, 1700                               # two levels
    docs, levels, ls = multifield_sequence_corpus(n, vocab, n_fields, seed=100 + n_fields, docs_per_level=per_level)
    assert len(levels) == 2
    orc = _oracle(levels, n, ls, BOOSTS[n_fields])
    phrases = phrase_queries_mf(docs, 200 + n_fields, 60, vocab)
    qk = query_keys(phrases)
    rng = np.random.default_rng(300 + n_fields)
    deleted = sorted({_doc_id(int(i), per_level) for i in rng.integers(0, n, 150)})
    n_hit = 0
    for i, ph in enumerate(phrases):
        for mask in (0, int(rng.integers(1, 1 << n_fields))):
            truth = {_doc_id(d, per_level) for d in range(n) if contains_phrase_fields(docs[d], ph, mask)}
            got, tot = orc.search_phrase(qk[i], n, O.RESULT_TOPKCOUNT, field_mask=mask)
            assert {d for d, _ in got} == truth and tot == len(truth), (n_fields, ph, mask)
            assert [s for _, s in got] == sorted((s for _, s in got), reverse=True)
            _, tot_c = orc.search_phrase(qk[i], 0, O.RESULT_COUNT, field_mask=mask)
            assert tot_c == tot
            n_hit += tot > 0
            # the delete set: the same matches minus the deleted docs, scores unchanged
            orc.set_deleted(deleted)
            got_d, tot_d = orc.search_phrase(qk[i], n, O.RESULT_TOPKCOUNT, field_mask=mask)
            orc.set_deleted([])
            assert got_d == [(d, s) for d, s in got if d not in set(deleted)] and tot_d == len(truth - set(deleted))
    assert n_hit > 60


def test_scores_are_the_bm25f_of_the_unique_terms():
    """a matching doc scores what the plain intersection of the phrase's unique terms scores (get_bm25f_multiterm_multifield)"""
    n, vocab = 2500, 25
    docs, levels, ls = multifield_sequence_corpus(n, vocab, 3, seed=7)
    orc = _oracle(levels, n, ls, BOOSTS[3])
    for ph in phrase_queries_mf(docs, 8, 30, vocab):
        k = query_keys([ph])[0]
        got, _ = orc.search_phrase(k, n, O.RESULT_TOPKCOUNT)
        inter, _ = orc.orc.search(list(dict.fromkeys(k)), O.QUERY_INTERSECTION, n, O.RESULT_TOPKCOUNT)
        score = dict(inter)
        assert all(score[d] == s for d, s in got)


def test_single_field_phrase_unchanged():
    """one indexed field: the field-aware oracle returns exactly what the C oracle's single-field phrase search returns"""
    from helpers import oracle_index
    from helpers_phrase import phrase_queries
    n, vocab = 4000, 40
    docs, levels, ls = sequence_corpus(n, vocab, 5, docs_per_level=2500)
    orc = oracle_index(levels, n, ls)
    mf = PhraseFieldsOracle(levels, n, ls)
    n_hit = 0
    for k in query_keys(phrase_queries(docs, 6, 40, vocab)):
        want = orc.search_phrase(k, 50, O.RESULT_TOPKCOUNT)
        assert mf.search_phrase(k, 50, O.RESULT_TOPKCOUNT) == want
        n_hit += want[1] > 0
    assert n_hit > 20


# ---- hand-made traps: token ids; filler docs make every trap term rare but present
A, B, C, D, E, F_, G = 1, 2, 3, 4, 5, 6, 7
TO, BE, OR, NOT = 20, 21, 22, 23
X, Y = 40, 41


def _trap_corpus():
    docs = [
        [[9, 9, 9, A], [9, 9, 9, 9, B]],                          # 0: "a" at position 3 of field 0, "b" at position 4 of field 1
        [[E, F_, C], [D, G]],                                     # 1: C ends field 0, D starts field 1
        [[10, 12], [11, 12]],                                     # 2: 10 and 11 both in the doc, never in one field
        [[9], [TO, BE, OR, NOT, TO, BE]],                         # 3: "to be or not to be" in field 1
        [[X, Y], [9, 9]],                                         # 4: "x y" only in field 0
        [[9, 9], [X, 9, Y]],                                      # 5: x and y in field 1, not adjacent
    ]
    docs += [[[9, 8, 9], [8, 9, 8, 9]] for _ in range(20)]
    levels, ls = levels_from_docs(docs, 2)
    return docs, _oracle(levels, len(docs), ls, (2.0, 1.0))


@pytest.mark.parametrize("phrase,mask,want", [
    ([A, B], 0, []),                     # positions restart per field: 3 (field 0) and 4 (field 1) are not adjacent
    ([C, D], 0, []),                     # the end of field 0 and the start of field 1 do not join
    ([10, 11], 0, []),                   # every term in the doc, never all in one field
    ([10, 12], 0, [2]),
    ([TO, BE, OR, NOT, TO, BE], 0, [3]),  # repeated tokens
    ([NOT, TO, BE], 0, [3]),
    ([TO, BE, TO, BE], 0, []),
    ([BE, OR, BE], 0, []),
    ([X, Y], 0, [4]),
    ([X, Y], 2, []),                     # the filter excludes the only field that holds the phrase
    ([X, Y], 1, [4]),                    # ... and includes it
    ([X, Y], 3, [4]),
    ([TO, BE], 1, []),
    ([TO, BE], 2, [3]),
])
def test_traps(phrase, mask, want):
    docs, orc = _trap_corpus()
    got, tot = orc.search_phrase(query_keys([phrase])[0], 10, O.RESULT_TOPKCOUNT, field_mask=mask)
    assert [d for d, _ in got] == want and tot == len(want)
    assert [d for d in range(len(docs)) if contains_phrase_fields(docs[d], phrase, mask)] == want
