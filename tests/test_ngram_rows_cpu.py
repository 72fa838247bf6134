"""CPU: the n-gram query rewrite (tokenizer.rs:898-1387) for every NgramSet row of NGRAM_SEARCH.md's benchmark tables."""
import pytest

from seekstorm_b200 import NgramSet as S, NgramType as T, ngram_rewrite

FREQUENT = {"the", "who", "is", "to", "be", "or", "not", "it", "up"}


def rw(q, ngram_set):
    return [("_".join(w), T(t).name) for w, t in ngram_rewrite(q.split(), FREQUENT, ngram_set)]


@pytest.mark.parametrize("ngram_set, want", [
    (S.NgramFF | S.NgramFR | S.NgramRF, [("to_be", "NgramFF"), ("or_not", "NgramFF"), ("to_be", "NgramFF")]),
    (S.NgramFF | S.NgramFR | S.NgramRF | S.NgramFFF | S.NgramRFF | S.NgramFFR | S.NgramFRF, [("to_be_or", "NgramFFF"), ("not_to_be", "NgramFFF")]),
])
def test_rewrite_to_be_or_not_to_be_mixed_rows(ngram_set, want):
    assert rw("to be or not to be", ngram_set) == want

ALL_SETS = {
    "SingleTerm": S.SingleTerm,
    "Frequent Bigrams": S.NgramFF,
    "Frequent Bigrams/Frequent Trigrams": S.NgramFF | S.NgramFFF,
    "Frequent Bigrams/Mixed Trigrams": S.NgramFF | S.NgramFFF | S.NgramRFF | S.NgramFFR | S.NgramFRF,
    "Mixed Bigrams": S.NgramFF | S.NgramFR | S.NgramRF,
    "Mixed Bigrams/Frequent Trigrams": S.NgramFF | S.NgramFR | S.NgramRF | S.NgramFFF,
    "Mixed Bigrams/Mixed Trigrams": S(127),
}


@pytest.mark.parametrize("row, pump, doors", [
    ("SingleTerm", ["pump", "it", "up"], ["the", "doors"]),
    ("Frequent Bigrams", ["pump", "it_up"], ["the", "doors"]),
    ("Frequent Bigrams/Frequent Trigrams", ["pump", "it_up"], ["the", "doors"]),
    ("Frequent Bigrams/Mixed Trigrams", ["pump_it_up"], ["the", "doors"]),
    ("Mixed Bigrams", ["pump_it", "up"], ["the_doors"]),
    ("Mixed Bigrams/Frequent Trigrams", ["pump_it", "up"], ["the_doors"]),
    ("Mixed Bigrams/Mixed Trigrams", ["pump_it_up"], ["the_doors"]),
])
def test_rewrite_each_ngram_set_row(row, pump, doors):
    """"pump it up" (pump rare) and "the doors" (doors rare) under every NgramSet row of NGRAM_SEARCH.md's benchmark tables"""
    assert [w for w, _ in rw("pump it up", ALL_SETS[row])] == pump
    assert [w for w, _ in rw("the doors", ALL_SETS[row])] == doors
