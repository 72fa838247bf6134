"""CPU: the corpora of tests/test_gpu_lex_limits.py really sit on the limits they claim — list lengths on both sides of DENSE_MIN and
UNION_WORDS, AND ratios at 8·cnt_a and 8·cnt_a + 1, doc ids on the coarse-byte boundaries, level counts, and the item cuts (first item
of 2, full 8-record items, ITEM_W cuts) of lex_plan's rule run over the bound-sorted records from the oracle's cache."""
import numpy as np
import pytest

from oracle import oracle as O
import helpers_lexlimits as H


def _lists_of(lv):
    offs = lv["posting_offsets"]
    return {int(k): (lv["doc_ids"][offs[i]:offs[i + 1]], lv["tfs"][offs[i]:offs[i + 1]]) for i, k in enumerate(lv["term_keys"])}


@pytest.fixture(scope="module")
def cutover():
    return H.cutover_corpus()


def test_cutover_list_lengths_and_edges(cutover):
    levels, n_docs, len_sum, lists = cutover
    (lv,) = levels
    got = _lists_of(lv)
    for t, n in H.CUTOVER_LISTS.items():
        ids, tfs = got[H.key_of(t)]
        assert len(ids) == n, t
        assert np.all(np.diff(ids.astype(np.int64)) > 0), t
        assert {0, 63, 64, 65535} <= set(int(d) for d in ids), t           # every list holds the edge ids
    for a, b in (("c127", "c128"), ("c128", "c129"), ("c2047", "c2048"), ("c2048", "c2049")):
        assert H.CUTOVER_LISTS[b] == H.CUTOVER_LISTS[a] + 1
    assert H.CUTOVER_LISTS["c127"] < H.DENSE_MIN <= H.CUTOVER_LISTS["c128"]
    assert H.CUTOVER_LISTS["c2047"] < H.UNION_WORDS <= H.CUTOVER_LISTS["c2048"]
    # cnt_b at 8 cnt_a (mark-and-stream) and 8 cnt_a + 1 (probe)
    assert H.CUTOVER_LISTS["r1024"] == H.AND_RATIO * H.CUTOVER_LISTS["r128"]
    assert H.CUTOVER_LISTS["r1025"] == H.AND_RATIO * H.CUTOVER_LISTS["r128"] + 1
    assert H.CUTOVER_LISTS["r1600"] == H.AND_RATIO * H.CUTOVER_LISTS["r200"]
    assert H.CUTOVER_LISTS["r1601"] == H.AND_RATIO * H.CUTOVER_LISTS["r200"] + 1
    # tfs 1, 254, 255, 256, 65535 and length bytes 0 / 255 occur; lists overlap (AND has matches)
    all_tfs = set(int(x) for x in lv["tfs"])
    assert {1, 254, 255, 256, 65535} <= all_tfs
    assert lv["doc_len_bytes"][0] == 0 and lv["doc_len_bytes"][65535] == 255 and lv["n_docs"] == 65536
    for a, b in (("c127", "c128"), ("r128", "r1025"), ("c2047", "c2048")):
        assert len(np.intersect1d(lists[a], lists[b])) >= 8


def test_cutover_queries_cover_every_count_branch(cutover):
    q = H.cutover_queries()
    n = H.CUTOVER_LISTS
    and_branch = set()
    for terms in q:
        if len(terms) > 4:
            continue
        cs = sorted(n[t] for t in terms)
        a, b = cs[0], cs[1]
        and_branch.add("words" if a >= H.UNION_WORDS else "stream" if b <= H.AND_RATIO * a else "probe")
    assert and_branch == {"words", "stream", "probe"}
    assert any(len(t) == 5 for t in q) and any(len(t) == 6 for t in q)                  # lex_generic
    assert any(all(n[t] >= H.UNION_WORDS for t in terms) for terms in q)                # OR: word-wise only
    assert any(all(n[t] < H.UNION_WORDS for t in terms) for terms in q)                 # OR: postings only


def test_cut_items_rule():
    assert H.cut_items([10] * 20) == [2, 8, 8, 2]
    assert H.cut_items([4032 - 64] * 3) == [1, 1, 1]                                    # one record of 4032 + 64 fills an item
    assert H.cut_items([1000] * 6) == [2, 3, 1]                                          # 3 x 1064 = 3192, a 4th would pass 4096
    assert H.cut_items([5000, 10, 10]) == [1, 2]                                         # an oversized record still forms an item
    assert H.cut_items([]) == []
    assert H.cut_items([10] * 10, why=True) == [(2, "lim"), (8, "end")]


def test_many_level_plans_cut_by_gmax_and_item_w():
    levels, n_docs, len_sum = H.mixed_levels(40, 11)
    assert len(levels) == 40
    ids = [lv["level_id"] for lv in levels]
    assert ids == sorted(ids) and ids[-1] == 65535 and ids[0] == 0
    assert levels[1]["n_docs"] == 1 and levels[-1]["n_docs"] == 65536
    last = _lists_of(levels[-1])
    assert any(65535 in set(int(d) for d in v[0]) for v in last.values())             # doc 0xFFFFFFFF exists
    causes, firsts = set(), set()
    for terms in H.random_queries(120, 10, 12):
        for is_and in (False, True):
            recs, items = H.plan_items(levels, n_docs, len_sum, H.keys(terms), is_and)
            if not items:
                continue
            firsts.add(items[0][0])
            assert items[0][0] <= H.FIRST_LIM and all(s <= H.GMAX for s, _ in items)
            assert sum(s for s, _ in items) == len(recs)
            causes |= {(s, c) for s, c in items}
            b = [r[0] for r in recs]
            assert b == sorted(b, reverse=True)
    assert 2 in firsts
    assert (H.GMAX, "lim") in causes                                                   # full 8-record items
    assert any(c == "w" for _, c in causes)                                            # ITEM_W cuts
    assert any(c == "w" and s > 1 for s, c in causes)                                  # ... of items holding several records


@pytest.mark.parametrize("n", [3, 129, 2049, 4096])
def test_small_level_counts(n):
    levels, n_docs, len_sum = H.small_levels(n, 1000 + n)
    assert len(levels) == n
    ids = [lv["level_id"] for lv in levels]
    assert ids == sorted(ids) and len(set(ids)) == n and ids[-1] == (65535 if n < H.MAX_LEVELS else 65520)
    assert (n & (n - 1) == 0) == (n == 4096)                                           # 3, 129, 2049: the bitonic sort pads to a power of 2
    assert n <= H.MAX_LEVELS
    smem = n * (8 + 2 * 4) + 16 + (1 << (n - 1).bit_length()) * 8                     # lex_plan's dynamic shared memory
    assert (smem > 48 * 1024) == (n >= 2049)


def test_tie_levels_every_score_equal():
    levels, n_docs, len_sum = H.tie_levels()
    orc = O.OracleIndex()
    for lv in levels:
        orc.add_level(lv)
    orc.commit(n_docs, len_sum)
    got, tot = orc.search(H.keys(["all"]), O.QUERY_UNION, 32, O.RESULT_TOPKCOUNT)
    assert tot == n_docs and len({s for _, s in got}) == 1
    assert [d for d, _ in got] == list(range(32))
    got, _ = orc.search(H.keys(["all", "lift"]), O.QUERY_UNION, 10, O.RESULT_TOPK)
    lifted = [(li << 16) | d for li in (38, 39) for d in (3, 7, 11)]
    assert sorted(d for d, _ in got[:6]) == lifted and [d for d, _ in got[6:]] == [0, 1, 2, 3]


def test_near_tie_levels_sit_one_ulp_apart():
    levels, n_docs, len_sum, near = H.near_tie_levels()
    orc = O.OracleIndex()
    for lv in levels:
        orc.add_level(lv)
    orc.commit(n_docs, len_sum)
    got, _ = orc.search(H.keys(["a", "b", "c"]), O.QUERY_UNION, len(near), O.RESULT_TOPK)
    assert sorted(d for d, _ in got) == sorted(d for d, _ in near)                    # the planted docs are the top
    bits = sorted({int(np.float32(s).view(np.uint32)) for _, s in got})
    assert len(bits) == 3 and bits[2] - bits[0] == 2                                   # S - 1 ulp, S, S + 1 ulp
    lv_of = {}
    for d, s in got:
        lv_of.setdefault(np.float32(s), set()).add(d >> 16)
    assert all(len(v) >= 2 for v in lv_of.values())                                    # each score occurs in several levels
    assert dict((d, np.float32(s)) for d, s in near) == dict((d, np.float32(s)) for d, s in got)   # the helper's sums are the oracle's
