"""Deterministic lexical corpora that sit on the BM25 engine's structural limits (bm25.cu), and a restatement of how lex_plan cuts a
query's bound-sorted records into work items.

Every list length, doc id, tf and length byte below is chosen, not sampled from a distribution: the tests assert the exact branch each
query takes.  No scoring code lives here — scores come from the C oracle; `comp` / `plan_items` only restate the plan's bound order
and item weights so that the CPU test can show which item cuts a corpus produces.

The limits (bm25.cu):
- DENSE_MIN = 128: a list of at least this many postings gets a bitmap (probes in O(1), word-wise reads in the facet pass);
- UNION_WORDS = 2048: from this many postings the count paths read a list as its 1024 bitmap words;
- cnt_b <= 8 * cnt_a: an AND count marks the shortest list and streams the second shortest, otherwise it probes;
- items: the first holds at most FIRST_LIM records, later ones at most GMAX, or until acc + cnt + 64 > ITEM_W postings;
- MAX_LEVELS = 4096 levels per GPU."""
import itertools

import numpy as np

from oracle import oracle as O
from seekstorm_b200 import synth
from helpers import key_of, level_from_postings

DENSE_MIN, UNION_WORDS, AND_RATIO = 128, 2048, 8
FIRST_LIM, GMAX, ITEM_W = 2, 8, 4096
MAX_LEVELS = 4096
EDGE_IDS = (0, 63, 64, 65535)                # the 64-doc coarse-byte boundaries and the last local id
TF_CYCLE = (1, 254, 255, 256, 65535, 1, 2, 3)  # 255 and up: the tf exception path of the reference's posting encoding
K1P = np.float32(np.float32(1.2) + np.float32(1.0))


def doc_order(seed: int = 7) -> np.ndarray:
    """A fixed permutation of the 65536 local ids that starts with EDGE_IDS: a list of n postings takes n ids out of the first
    max(4n, 1024) entries, so lists of every length share docs (AND has matches) and the edge ids sit in every list."""
    rest = np.setdiff1d(np.arange(65536), np.array(EDGE_IDS))
    return np.concatenate([np.array(EDGE_IDS), np.random.default_rng(seed).permutation(rest)]).astype(np.int64)


def spread_ids(n: int, order: np.ndarray, seed: int, n_docs: int = 65536) -> np.ndarray:
    """n distinct sorted local ids < n_docs: the edge ids below n_docs first, then a seeded pick from the head of `order`"""
    order = order[order < n_docs]
    n = min(n, n_docs)
    head = [int(d) for d in order[:4] if d < n_docs][:n]
    pool = order[len(head):min(len(order), max(4 * n, 1024))]
    pick = np.random.default_rng(seed).choice(pool, size=n - len(head), replace=False) if n > len(head) else np.zeros(0, np.int64)
    return np.sort(np.concatenate([np.array(head, dtype=np.int64), pick])).astype(np.int64)


def tf_of(term_idx: int, d: int) -> int:
    return TF_CYCLE[(d + 3 * term_idx) % len(TF_CYCLE)]


def build_level(level_id: int, n_docs: int, lists: dict, len_bytes, tf_fn=tf_of) -> dict:
    """lists: term -> sorted local ids; tf_fn(term index in sorted term order, doc) -> tf"""
    post = {}
    for ti, t in enumerate(sorted(lists)):
        post[t] = [(int(d), int(tf_fn(ti, int(d)))) for d in lists[t]]
    return level_from_postings(level_id, n_docs, post, np.asarray(len_bytes, dtype=np.uint8))


def len_sum_of(levels) -> int:
    return int(sum(sum(synth.byte4_to_int(int(b)) for b in lv["doc_len_bytes"]) for lv in levels))


# ---------------------------------------------------------------- 1. one level, every list-length cut-over
CUTOVER_LISTS = {
    "c127": 127, "c128": 128, "c129": 129, "c2047": 2047, "c2048": 2048, "c2049": 2049,   # DENSE_MIN and UNION_WORDS, both sides
    "c4000": 4000, "c16384": 16384,                                                          # longer partners of a 2047 / 2048 shortest list
    "r128": 128, "r1024": 1024, "r1025": 1025,                                               # cnt_b = 8 cnt_a and 8 cnt_a + 1
    "r200": 200, "r1600": 1600, "r1601": 1601,
    "n50": 50, "n300": 300, "n3000": 3000,                                                   # NOT lists: sparse, bitmap, word-wise
}


def cutover_corpus():
    """One full level (id 0, 65536 docs).  Length byte = doc id mod 256 (0 at doc 0, 255 at doc 65535); tfs from TF_CYCLE."""
    order = doc_order()
    lists = {t: spread_ids(n, order, 100 + i) for i, (t, n) in enumerate(sorted(CUTOVER_LISTS.items()))}
    lens = (np.arange(65536) % 256).astype(np.uint8)
    lv = build_level(0, 65536, lists, lens)
    return [lv], 65536, len_sum_of([lv]), lists


def cutover_queries():
    """2-4 term mixes of the six cut-over lists, the AND ratio pairs, 5- and 6-term queries (lex_generic)"""
    six = ["c127", "c128", "c129", "c2047", "c2048", "c2049"]
    qs = [list(c) for r in (2, 3, 4) for c in itertools.combinations(six, r)]
    qs += [["c2047", "c4000"], ["c2048", "c4000"], ["c2047", "c16384"], ["c2048", "c4000", "c16384"], ["c2049", "c2048", "c16384"],
           ["r128", "r1024"], ["r128", "r1025"], ["r200", "r1600"], ["r200", "r1601"], ["r128", "r1024", "c4000"],
           ["r200", "r1601", "c16384"], ["c127", "c16384", "c4000", "c2049"]]
    qs += [list(c) for c in itertools.combinations(six, 5)] + [six, six[::-1]]
    return qs


# ---------------------------------------------------------------- 3. many-level plans
def mixed_levels(n_levels: int, seed: int, vocab: int = 10, sizes=None, level_ids=None, density=None):
    """n_levels levels with sparse ascending level ids; mixed level sizes and list densities so that items are cut both by GMAX (short
    lists) and by ITEM_W (long ones).  The last level has id 65535 and 65536 docs, so doc 0xFFFFFFFF exists; level 1 has a single doc."""
    rng = np.random.default_rng(seed)
    order = doc_order(seed)
    if level_ids is None:
        step = max(1, 65535 // n_levels)
        level_ids = [i * step for i in range(n_levels - 1)] + [65535]
    if sizes is None:
        cyc = (65536, 1, 300, 5000, 20000, 700, 65536, 64, 12000, 2500)
        sizes = [cyc[i % len(cyc)] for i in range(n_levels)]
        sizes[-1] = 65536
    dens = density if density is not None else (0.3, 0.1, 0.03, 0.01, 0.2, 0.05, 0.002, 0.5, 0.08, 0.015)
    levels = []
    for li, (lid, nd) in enumerate(zip(level_ids, sizes)):
        f = (0.25, 1.0, 2.5, 0.6)[li % 4]
        lists = {}
        for t in range(vocab):
            n = int(round(nd * min(1.0, dens[t % len(dens)] * f)))
            if nd == 1:
                n = 1 if t in (0, 7) else 0
            if n:
                lists[f"t{t}"] = spread_ids(n, order, seed * 7919 + li * 31 + t, nd)
        lens = rng.integers(0, 256, nd).astype(np.uint8)
        lens[0] = 0
        lens[-1] = 255
        levels.append(build_level(int(lid), int(nd), lists, lens))
    return levels, int(sum(sizes)), len_sum_of(levels)


def small_levels(n_levels: int, seed: int, vocab: int = 6):
    """n_levels small levels (48..200 docs, lists of 0..60 postings): the plan's level count without the memory of big levels.
    Level ids i * (65536 // n_levels), the last one 65535 below MAX_LEVELS levels (at MAX_LEVELS, 65535 stays free for a 4097th level
    that is valid in every respect but the count)."""
    rng = np.random.default_rng(seed)
    step = max(1, 65536 // n_levels)
    ids = [i * step for i in range(n_levels)]
    if n_levels < MAX_LEVELS:
        ids[-1] = 65535
    levels = []
    for li, lid in enumerate(ids):
        nd = int(rng.integers(48, 201))
        lists = {}
        for t in range(vocab):
            n = int(rng.integers(0, 61)) if (li + t) % 3 else int(rng.integers(0, 4))
            if n:
                lists[f"s{t}"] = np.sort(rng.choice(nd, size=min(n, nd), replace=False))
        if not lists:
            lists["s0"] = np.array([0])
        levels.append(build_level(lid, nd, lists, rng.integers(0, 256, nd).astype(np.uint8)))
    return levels, int(sum(lv["n_docs"] for lv in levels)), len_sum_of(levels)


def random_queries(n: int, vocab, seed: int, lengths=(1, 2, 3, 4), prefix="t"):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        m = int(rng.choice(lengths))
        out.append([f"{prefix}{int(t)}" for t in rng.choice(vocab, size=m, replace=False)])
    return out


# ---------------------------------------------------------------- 4. ties across levels
def tie_levels(n_levels: int = 40, n_docs: int = 500, lift_levels=(38, 39), lift_docs=(3, 7, 11)):
    """Term "all" in every doc of every level with tf 1 and one length byte: every score of ["all"] is the same.  Term "lift" adds to
    a few docs of the LAST levels only, so θ is first set there by high doc ids."""
    levels = []
    for li in range(n_levels):
        lists = {"all": np.arange(n_docs)}
        if li in lift_levels:
            lists["lift"] = np.array(lift_docs)
        levels.append(build_level(li, n_docs, lists, np.full(n_docs, 40, np.uint8), tf_fn=lambda t, d: 1))
    return levels, n_levels * n_docs, len_sum_of(levels)


def near_tie_levels(n_levels: int = 6, n_docs: int = 4096, seed: int = 5):
    """3-term docs whose exact scores (query order a, b, c) are S - 1 ulp, S and S + 1 ulp, for one S, spread over several levels,
    among filler docs that score lower.  The (tf, length byte) triples are searched with the oracle's cache and idfs.
    Returns (levels, n_docs_total, len_sum, near) with near = [(doc_id, score)] of the planted docs."""
    rng = np.random.default_rng(seed)
    per_level = 6
    n_total = n_levels * n_docs
    # list lengths: "a" in every planted doc + fillers, "b"/"c" in the planted docs + fewer fillers -> fixed dfs
    fill = {"a": 600, "b": 300, "c": 150}
    dfs = {t: n_levels * (per_level + f) for t, f in fill.items()}
    lens = np.full(n_docs, 30, np.uint8)
    len_sum = n_levels * sum(synth.byte4_to_int(int(b)) for b in lens)
    cache = O.bm25_cache(n_total, len_sum)
    idf = {t: np.float32(O.lib().orc_idf(n_total, dfs[t])) for t in dfs}
    lb = 30
    tfs = np.arange(1, 300)
    comps = (tfs.astype(np.float32) * K1P) / (tfs.astype(np.float32) + cache[lb])

    def score(ta, tb, tc):
        s = np.float32(0.0)
        for t, tf in (("a", ta), ("b", tb), ("c", tc)):
            s = np.float32(s + np.float32(idf[t] * comps[tf - 1]))
        return s

    # bucket a grid of triples by score bits and find a score S with neighbours at +-1 ulp
    by = {}
    for ta in range(2, 60):                          # tf >= 2 everywhere: every planted doc beats a tf-1 filler
        for tb in range(2, 60):
            for tc in range(2, 40):
                by.setdefault(int(score(ta, tb, tc).view(np.uint32)), []).append((ta, tb, tc))
    best = None
    for u in sorted(by):
        if u - 1 in by and u + 1 in by and len(by[u]) >= 2:
            best = u
            break
    assert best is not None, "no near-tie triple found"
    group = [by[best - 1][0], by[best - 1][-1], by[best][0], by[best][-1], by[best + 1][0], by[best + 1][-1]]
    levels, near = [], []
    for li in range(n_levels):
        planted = rng.choice(np.arange(100, n_docs), size=per_level, replace=False)
        tri = {int(d): group[(li + j) % len(group)] for j, d in enumerate(sorted(planted))}
        others = np.setdiff1d(np.arange(n_docs), planted)
        lists, tfmap = {}, {}
        for ti, t in enumerate(("a", "b", "c")):
            fillers = rng.choice(others, size=fill[t], replace=False)
            ids = np.sort(np.concatenate([planted, fillers]))
            lists[t] = ids
            for d in ids:
                tfmap[(t, int(d))] = tri[int(d)][ti] if int(d) in tri else 1
        lv = build_level(li, n_docs, lists, lens, tf_fn=lambda ti, d, _m=tfmap: _m[("abc"[ti], d)])
        levels.append(lv)
        near += [((li << 16) | d, float(score(*tri[d]))) for d in tri]
    return levels, n_total, len_sum, near


# ---------------------------------------------------------------- the plan's items (lex_plan, bm25.cu: records and the item cut)
def _entries(levels):
    """term key -> [(level index, count, max comp)] with the comps computed later; here the raw posting arrays per (key, level)"""
    out = {}
    for li, lv in enumerate(levels):
        offs = lv["posting_offsets"]
        for i, k in enumerate(lv["term_keys"]):
            out.setdefault(int(k), []).append((li, int(offs[i]), int(offs[i + 1])))
    return out


def plan_items(levels, n_docs: int, len_sum: int, qkeys, is_and: bool, first_lim=FIRST_LIM, gmax=GMAX, item_w=ITEM_W):
    """The records of one query in bound order and their item sizes, as lex_plan builds them: per level the bound Σ idf·max comp in
    query order (f32), levels sorted by bound descending (ties: lower level index first), weight = the count of the list that drives
    (AND: the shortest, ties to the later query slot; OR: the largest upper bound, ties to the earlier slot), then the cut."""
    cache = O.bm25_cache(n_docs, len_sum)
    ents = _entries(levels)
    terms = []
    for k in qkeys:                                                  # unique live terms in query order
        if k in [t[0] for t in terms]:
            continue
        e = ents.get(int(k), [])
        if not e:
            if is_and:
                return [], []
            continue
        df = sum(b - a for _, a, b in e)
        idf = np.float32(O.lib().orc_idf(n_docs, df))
        per = {}
        for li, a, b in e:
            lv = levels[li]
            tf = lv["tfs"][a:b].astype(np.float32)
            c = (tf * K1P) / (tf + cache[lv["doc_len_bytes"][lv["doc_ids"][a:b]]])
            per[li] = (b - a, np.float32(idf * np.float32(c.max())))
        terms.append((int(k), per))
    nl = len(terms)
    recs = []
    for li in range(len(levels)):
        present = [t for t in terms if li in t[1]]
        if (is_and and (nl == 0 or len(present) != nl)) or (not is_and and not present):
            continue
        bound = np.float32(0.0)
        for _, per in terms:
            if li in per:
                bound = np.float32(bound + per[li][1])
        if nl <= 4:
            cs = [t[1][li][0] if li in t[1] else 0 for t in terms]
            us = [t[1][li][1] if li in t[1] else np.float32(0) for t in terms]
            live = [s for s in range(nl) if cs[s]]
            if is_and:
                drv = min(live, key=lambda s: (cs[s], -s))
            else:
                drv = min(live, key=lambda s: (-us[s], s))
            w = cs[drv]
        else:
            w = item_w
        recs.append((float(bound), li, w))
    recs.sort(key=lambda r: (-r[0], r[1]))
    return recs, cut_items([r[2] for r in recs], first_lim, gmax, item_w, why=True)


def cut_items(weights, first_lim=FIRST_LIM, gmax=GMAX, item_w=ITEM_W, why=False):
    """bm25.cu lex_plan: consecutive records form an item; a new item starts when the current one holds `lim` records (first_lim for
    the first item, gmax after) or when adding the next record's weight + 64 would pass item_w.  Returns the item sizes, or with
    why=True (size, cause) pairs: "lim" (record limit), "w" (item_w) or "end" (the last item)."""
    out, acc, nin = [], 0, 0
    for w in weights:
        lim = first_lim if not out else gmax
        ww = w + 64
        if nin > 0 and (nin >= lim or acc + ww > item_w):
            out.append((nin, "lim" if nin >= lim else "w"))
            acc, nin = 0, 0
        acc += ww
        nin += 1
    if nin:
        out.append((nin, "end"))
    return out if why else [n for n, _ in out]


def keys(terms):
    return [key_of(t) for t in terms]
