"""CPU: the index.bin parser on files with n-gram keys (tests/refwriter_ngram.py, 22- and 23-byte key heads): ssb_index_bin_inspect_ngrams
returns every n-gram key's df bytes and every posting's doc id, tf, component tfs and positions as written; ssb_index_bin_inspect and the
single-term data are exactly what the same shard written without n-gram keys gives."""
import ctypes

import numpy as np
import pytest

from seekstorm_b200 import NgramSet as S, _lib

import helpers_ngram as H
import refwriter as R
import refwriter_ngram as RN

FREQ = set(range(6))


def _inspect(fn, data, khs, pos):
    prm = _lib.SsbIndexBinParams(1, khs, R.SEGMENT_BITS, 1 if pos else 0)
    out = (ctypes.c_uint64 * 8)()
    buf = np.frombuffer(data, dtype=np.uint8)
    rc = getattr(_lib.lib(), fn)(buf.ctypes.data, buf.size, ctypes.byref(prm), out)
    assert rc == 0, _lib.lib().ssb_last_error()
    return list(out)


@pytest.mark.parametrize("khs, ngram_set", [(22, S.NgramFF | S.NgramFR | S.NgramRF),
                                            (23, S.NgramFF | S.NgramFR | S.NgramRF | S.NgramFFF | S.NgramRFF | S.NgramFFR | S.NgramFRF)])
@pytest.mark.parametrize("pos", [False, True])
def test_ngram_round_trip(khs, ngram_set, pos):
    docs, levels, len_sum, stats = H.ngram_corpus(3000, 40, 7, FREQ, ngram_set, docs_per_level=65536, mean_len=12)
    data, cum = RN.write_index_bin_ngrams(levels, 3000, khs)
    assert cum == len_sum
    got = _inspect("ssb_index_bin_inspect_ngrams", data, khs, pos)
    want = RN.ngram_checksum(levels, pos)
    assert got[1] > 100 and got == want


@pytest.mark.parametrize("pos", [False, True])
def test_single_terms_load_as_before(pos):
    """ssb_index_bin_inspect skips the n-gram keys: its output equals that of the same shard written without them (20-byte heads)"""
    docs, levels, len_sum, stats = H.ngram_corpus(3000, 40, 9, FREQ, S.NgramFF | S.NgramFFF, docs_per_level=65536, mean_len=12)
    data, _ = RN.write_index_bin_ngrams(levels, 3000, 23)
    plain, _ = R.write_index_bin(H.single_term_levels(levels), 3000)
    a = _inspect("ssb_index_bin_inspect", data, 23, pos)
    b = _inspect("ssb_index_bin_inspect", plain, 20, pos)
    assert a == b
    assert a[1] == sum(int((lv["term_keys"] & np.uint64(7) == 0).sum()) for lv in levels)


def test_ngram_inspect_needs_df_bytes():
    docs, levels, len_sum, stats = H.ngram_corpus(200, 20, 3, FREQ, S.NgramFF, docs_per_level=65536, mean_len=8)
    plain, _ = R.write_index_bin(H.single_term_levels(levels), 200)
    prm = _lib.SsbIndexBinParams(1, 20, R.SEGMENT_BITS, 0)
    out = (ctypes.c_uint64 * 8)()
    buf = np.frombuffer(plain, dtype=np.uint8)
    assert _lib.lib().ssb_index_bin_inspect_ngrams(buf.ctypes.data, buf.size, ctypes.byref(prm), out) == -1
