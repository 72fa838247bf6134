"""N-gram indexes for the tests, restated from the reference: the index-time n-gram generator (tokenizer.rs:672-860, FFR / FRF generated
under the RFF bit), the n-gram posting layout (start positions, own tf, component tfs in word order, index_posting.rs:765-795), the key-head
df bytes of each level (the byte4 code of each component's df over the levels committed so far, compress_postinglist.rs:28-230), and a
float32 scorer of phrase queries (search.rs:3221-3269, add_result.rs:1448-1478) that runs on token sequences, independent of the library."""
import ctypes

import numpy as np

from seekstorm_b200 import NgramSet, NgramType, ngram_key, synth

_libm = ctypes.CDLL("libm.so.6")
_libm.logf.restype = ctypes.c_float
_libm.logf.argtypes = [ctypes.c_float]
F = np.float32


def word(t):
    return f"t{int(t)}"


def index_ngrams(doc, frequent, ngram_set):
    """tokenizer.rs:672-860 on one doc of token ids -> {(words tuple, NgramType): [start positions]} including the single terms"""
    out = {}
    for j, t0 in enumerate(doc):
        out.setdefault(((word(t0),), NgramType.SingleTerm), []).append(j)
        f0 = int(t0) in frequent
        if j >= 1:
            t1 = doc[j - 1]; f1 = int(t1) in frequent
            for bit, ok, ty in ((NgramSet.NgramFF, f1 and f0, NgramType.NgramFF), (NgramSet.NgramRF, (not f1) and f0, NgramType.NgramRF),
                                (NgramSet.NgramFR, f1 and not f0, NgramType.NgramFR)):
                if ngram_set & bit and ok:
                    out.setdefault(((word(t1), word(t0)), ty), []).append(j - 1)
        if j >= 2:
            t2, t1 = doc[j - 2], doc[j - 1]; f2, f1 = int(t2) in frequent, int(t1) in frequent
            # the reference generates FFR and FRF under the RFF bit (tokenizer.rs:817, 850)
            for bit, ok, ty in ((NgramSet.NgramFFF, f2 and f1 and f0, NgramType.NgramFFF),
                                (NgramSet.NgramRFF, (not f2) and f1 and f0, NgramType.NgramRFF),
                                (NgramSet.NgramRFF, f2 and f1 and not f0, NgramType.NgramFFR),
                                (NgramSet.NgramRFF, f2 and (not f1) and f0, NgramType.NgramFRF)):
                if ngram_set & bit and ok:
                    out.setdefault(((word(t2), word(t1), word(t0)), ty), []).append(j - 2)
    return out


def ngram_corpus(n_docs, vocab, seed, frequent, ngram_set, docs_per_level=1000, mean_len=20):
    """-> (docs, levels (neutral dicts with ngram_tfs / ngram_df_bytes), len_sum, stats) where stats = {"df": {key: global df},
    "dfb": {key: [per level df bytes in level order]}, "type": {key: NgramType}}"""
    rng = np.random.default_rng(seed)
    w = 1.0 / (np.arange(vocab) + 2.0)
    w /= w.sum()
    lens = np.clip(rng.geometric(1.0 / mean_len, n_docs), 2, 200)
    docs = [rng.choice(vocab, size=int(n), p=w).astype(np.int64) for n in lens]
    levels, len_sum = [], 0
    word_df = {}                                                    # df of every single term over the levels so far
    df, dfb, types = {}, {}, {}
    for li, base in enumerate(range(0, n_docs, docs_per_level)):
        nd = min(docs_per_level, n_docs - base)
        lists = {}                                                  # key -> [(doc, positions, component tfs)]
        for d in range(nd):
            doc = docs[base + d]
            counts = {}
            for t in doc:
                counts[word(t)] = counts.get(word(t), 0) + 1
            for (ws, ty), pos in index_ngrams(doc, frequent, ngram_set).items():
                key = ngram_key(ws, ty)
                types[key] = ty
                ctf = [counts[x] for x in ws] + [0] * (3 - len(ws)) if ty else [0, 0, 0]
                lists.setdefault(key, (ws, []))[1].append((d, pos, ctf))
        for key, (ws, posts) in lists.items():
            if len(ws) == 1:
                word_df[ws[0]] = word_df.get(ws[0], 0) + len(posts)
        keys = sorted(lists)
        offs, ids, tfs, pos_all, ctfs, dfbytes = [0], [], [], [], [], []
        for key in keys:
            ws, posts = lists[key]
            for d, pos, ctf in posts:
                ids.append(d); tfs.append(len(pos)); pos_all.extend(pos); ctfs.append(ctf)
            offs.append(len(ids))
            b = [synth.int_to_byte4(word_df.get(x, 0)) for x in ws] + [0] * (3 - len(ws)) if types[key] else [0, 0, 0]
            dfbytes.append(b)
            df[key] = df.get(key, 0) + len(posts)
            if types[key]:
                dfb.setdefault(key, []).append(b)
        lb = np.array([synth.int_to_byte4(len(docs[base + d])) for d in range(nd)], dtype=np.uint8)
        len_sum += int(sum(synth.byte4_to_int(int(b)) for b in lb))
        levels.append(dict(level_id=li, n_docs=nd, term_keys=np.array(keys, dtype=np.uint64), posting_offsets=np.array(offs, dtype=np.uint32),
                           doc_ids=np.array(ids, dtype=np.uint16), tfs=np.array(tfs, dtype=np.uint16), doc_len_bytes=lb,
                           positions=np.array(pos_all, dtype=np.uint16), ngram_tfs=np.array(ctfs, dtype=np.uint16).reshape(-1, 3),
                           ngram_df_bytes=np.array(dfbytes, dtype=np.uint8).reshape(-1, 3)))
    return docs, levels, len_sum, dict(df=df, dfb=dfb, type=types)


def single_term_levels(levels):
    """the same levels without the n-gram lists (a SingleTerm-only index of the same corpus)"""
    out = []
    for lv in levels:
        keys, offs = lv["term_keys"], lv["posting_offsets"]
        keep = [t for t in range(len(keys)) if int(keys[t]) & 7 == 0]
        pos_off = np.concatenate([[0], np.cumsum(lv["tfs"].astype(np.int64))])
        n_offs, ids, tfs, pos = [0], [], [], []
        for t in keep:
            a, b = int(offs[t]), int(offs[t + 1])
            ids.append(lv["doc_ids"][a:b]); tfs.append(lv["tfs"][a:b]); pos.append(lv["positions"][pos_off[a]:pos_off[b]])
            n_offs.append(n_offs[-1] + b - a)
        out.append(dict(level_id=lv["level_id"], n_docs=lv["n_docs"], term_keys=keys[keep], posting_offsets=np.array(n_offs, dtype=np.uint32),
                        doc_ids=np.concatenate(ids), tfs=np.concatenate(tfs), doc_len_bytes=lv["doc_len_bytes"], positions=np.concatenate(pos)))
    return out


def bm25_cache(n_docs, len_sum):
    """commit.rs:318-325 in float32"""
    avgdl = F(F(len_sum) / F(n_docs))
    return [F(F(1.2) * F(F(1.0 - 0.75) + F(F(0.75) * F(F(synth.byte4_to_int(b)) / avgdl)))) for b in range(256)]


def idf(n_docs, df):
    """search.rs:3225-3230 with the C library's logf"""
    r = F(F(F(F(n_docs) - F(df)) + F(0.5)) / F(F(df) + F(0.5)))
    return F(_libm.logf(float(F(r + F(1.0)))))


def part(tf, bc):
    t = F(tf)
    return F(F(t * F(2.2)) / F(t + bc))


def ngram_component_sum(idfs, tfs, bc):
    """add_result.rs:1448-1478: idf1*part1 + idf2*part2 (+ idf3*part3), left to right"""
    s = F(F(idfs[0] * part(tfs[0], bc)) + F(idfs[1] * part(tfs[1], bc)))
    if len(idfs) == 3:
        s = F(s + F(idfs[2] * part(tfs[2], bc)))
    return s


def phrase_oracle(docs, levels, len_sum, stats, query_keys, similarity, df_rule, deleted=()):
    """phrase query on the n-gram index -> [(doc id, float32 score)] of every match, best first (score desc, doc id asc).  A doc matches
    when every key's list holds it and some start p has token i at p + i + (1 per earlier bigram, 2 per earlier trigram)."""
    n_docs = sum(lv["n_docs"] for lv in levels)
    cache = bm25_cache(n_docs, len_sum)
    uniq = list(dict.fromkeys(query_keys))
    offs, o = [], 0
    for k in query_keys:
        offs.append(o)
        ty = int(k) & 7
        o += 1 if ty == 0 else (2 if ty <= 3 else 3)
    comp_idf = {}
    for k in uniq:
        ty = int(k) & 7
        if ty and k in stats["dfb"]:
            b = stats["dfb"][k][0 if df_rule == 0 else -1]
            n = 2 if ty <= 3 else 3
            comp_idf[k] = [idf(n_docs, synth.byte4_to_int(int(x))) for x in b[:n]] if similarity == 0 else None
    deleted = set(deleted)
    out = []
    for lv in levels:
        pos_off = np.concatenate([[0], np.cumsum(lv["tfs"].astype(np.int64))])
        keys = {int(x): t for t, x in enumerate(lv["term_keys"])}
        post = {}
        for k in uniq:
            if k not in keys:
                post = None
                break
            t = keys[k]
            a, b = int(lv["posting_offsets"][t]), int(lv["posting_offsets"][t + 1])
            post[k] = {int(lv["doc_ids"][p]): (set(int(x) for x in lv["positions"][pos_off[p]:pos_off[p + 1]]), int(lv["tfs"][p]), lv["ngram_tfs"][p])
                       for p in range(a, b)}
        if post is None:
            continue
        cand = set.intersection(*[set(v) for v in post.values()])
        for d in sorted(cand):
            doc = (lv["level_id"] << 16) | d
            if doc in deleted:
                continue
            if len(query_keys) >= 2:
                p0 = post[query_keys[0]][d][0]
                if not any(all(s + offs[i] in post[query_keys[i]][d][0] for i in range(len(query_keys))) for s in p0):
                    continue
            bc = cache[int(lv["doc_len_bytes"][d])]
            score = F(0.0)
            for k in uniq:
                ty = int(k) & 7
                _, tf, ctf = post[k][d]
                if ty == 0:
                    c = F(idf(n_docs, stats["df"][k]) * part(tf, bc))
                elif comp_idf[k] is None:
                    c = F(0.0)                                  # Bm25fProximity, one field: idf_ngram* stay 0.0
                else:
                    c = ngram_component_sum(comp_idf[k], [int(x) for x in ctf[:len(comp_idf[k])]], bc)
                score = F(score + c)
            out.append((doc, score))
    out.sort(key=lambda x: (-float(x[1]), x[0]))
    return out
