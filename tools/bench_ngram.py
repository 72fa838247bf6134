"""N-gram phrase search: the same C3-law corpus (Zipf token sequences with positions) indexed twice, SingleTerm only and with FF | FFF
n-gram lists of its `--frequent` most frequent terms, then the same phrase queries on both: phrases of 2-3 frequent terms and mixed phrases
(3-4 tokens with at least one rare term), cut out of the documents.  Prints, per index and query set, batched Phrase TopkCount / Topk
queries/s, per-query p50 / p99 latency at batch 1, the lex_generic (dominant kernel) time of the batch from ssb_last_stats, the device
memory each index holds, and the card / power limit read in the same run.  One JSON line per (index, query set), then a summary line.

    python tools/bench_ngram.py [--docs 1000000] [--vocab 50000] [--frequent 100] [--queries 1024]

N-gram keys here are splitmix64 of the token pair / triple (the library only needs distinct keys; the reference hashes the joined
strings).  Nothing is written to disk."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from seekstorm_b200 import Index, LexicalSimilarity, QueryType, ResultType, synth  # noqa: E402



def pair_key(a, b, c=None, ty=1):
    x = a.astype(np.uint64) * np.uint64(1000003) + b.astype(np.uint64) + np.uint64(1 << 40)
    if c is not None:
        x = x * np.uint64(1000003) + c.astype(np.uint64) + np.uint64(1 << 41)
    return (synth.term_keys_np(x) & ~np.uint64(7)) | np.uint64(ty)


def corpus(n_docs, vocab, seed, mean_len=30):
    rng = np.random.default_rng(seed)
    w = 1.0 / (np.arange(vocab) + 2.0)
    w /= w.sum()
    lens = np.clip(rng.geometric(1.0 / mean_len, n_docs), 2, 400).astype(np.int64)
    toks = rng.choice(vocab, size=int(lens.sum()), p=w).astype(np.int64)
    return lens, toks


def levels_of(lens, toks, freq_n, ngrams):
    """neutral levels of 65536 docs; ngrams: also the FF / FFF lists with their component tfs and df bytes"""
    starts = np.concatenate([[0], np.cumsum(lens)])
    word_df = np.zeros(int(toks.max()) + 1, dtype=np.int64)
    out, len_sum = [], 0
    n_docs = len(lens)
    for li, base in enumerate(range(0, n_docs, 65536)):
        nd = min(65536, n_docs - base)
        a, b = starts[base], starts[base + nd]
        tok = toks[a:b]
        doc = np.repeat(np.arange(nd), lens[base:base + nd])
        pos = np.arange(b - a) - (starts[base:base + nd] - a).repeat(lens[base:base + nd])
        # per (doc, word) counts -> component tfs
        dw = doc * (word_df.size) + tok
        u, inv, cnt = np.unique(dw, return_inverse=True, return_counts=True)
        word_df += np.bincount(u % word_df.size, minlength=word_df.size)
        tfw = cnt[inv]
        keys = [synth.term_keys_np(tok)]; docs = [doc]; poss = [pos]; comps = [np.zeros((len(tok), 3), np.int64)]; dfw = [np.zeros((len(tok), 3), np.int64)]
        if ngrams:
            f = tok < freq_n
            same1 = np.zeros(len(tok), bool); same1[:-1] = doc[:-1] == doc[1:]
            same2 = np.zeros(len(tok), bool); same2[:-2] = same1[:-2] & same1[1:-1]
            i2 = np.flatnonzero(same1 & f & np.roll(f, -1))
            keys.append(pair_key(tok[i2], tok[i2 + 1], ty=1)); docs.append(doc[i2]); poss.append(pos[i2])
            comps.append(np.stack([tfw[i2], tfw[i2 + 1], np.zeros_like(i2)], 1))
            dfw.append(np.stack([word_df[tok[i2]], word_df[tok[i2 + 1]], np.zeros_like(i2)], 1))
            i3 = np.flatnonzero(same2 & f & np.roll(f, -1) & np.roll(f, -2))
            keys.append(pair_key(tok[i3], tok[i3 + 1], tok[i3 + 2], ty=4)); docs.append(doc[i3]); poss.append(pos[i3])
            comps.append(np.stack([tfw[i3], tfw[i3 + 1], tfw[i3 + 2]], 1))
            dfw.append(np.stack([word_df[tok[i3]], word_df[tok[i3 + 1]], word_df[tok[i3 + 2]]], 1))
        K, D, P, C, W = (np.concatenate(x) for x in (keys, docs, poss, comps, dfw))
        o = np.lexsort((P, D, K))
        K, D, P, C, W = K[o], D[o], P[o], C[o], W[o]
        newp = np.concatenate([[True], (K[1:] != K[:-1]) | (D[1:] != D[:-1])])
        ps = np.flatnonzero(newp)
        tfs = np.diff(np.concatenate([ps, [len(K)]]))
        pk = K[ps]
        newt = np.concatenate([[True], pk[1:] != pk[:-1]])
        ts = np.flatnonzero(newt)
        wt = W[ps][ts]
        uv, inv = np.unique(wt, return_inverse=True)
        dfb = np.array([synth.int_to_byte4(int(x)) for x in uv], dtype=np.uint8)[inv.ravel()].reshape(wt.shape)
        lb = np.array([synth.int_to_byte4(int(x)) for x in lens[base:base + nd]], dtype=np.uint8)
        len_sum += int(sum(synth.byte4_to_int(int(x)) for x in lb))
        lv = dict(level_id=li, n_docs=nd, term_keys=pk[ts].astype(np.uint64), posting_offsets=np.concatenate([ts, [len(ps)]]).astype(np.uint32),
                  doc_ids=D[ps].astype(np.uint16), tfs=np.minimum(tfs, 65535).astype(np.uint16), doc_len_bytes=lb,
                  positions=np.minimum(P, 65535).astype(np.uint16))
        if ngrams:
            lv["ngram_tfs"] = np.minimum(C[ps], 65535).astype(np.uint16)
            lv["ngram_df_bytes"] = dfb.astype(np.uint8)
        out.append(lv)
    return out, len_sum


def queries(lens, toks, freq_n, n, seed):
    rng = np.random.default_rng(seed)
    starts = np.concatenate([[0], np.cumsum(lens)])
    freq, mixed = [], []
    while len(freq) < n or len(mixed) < n:
        d = int(rng.integers(0, len(lens)))
        m = int(rng.integers(2, 5))
        if lens[d] < m:
            continue
        s = starts[d] + int(rng.integers(0, lens[d] - m + 1))
        ph = toks[s:s + m]
        if (ph < freq_n).all() and m <= 3 and len(freq) < n:
            freq.append(ph)
        elif m >= 3 and (ph < freq_n).sum() >= 2 and (ph >= freq_n).any() and len(mixed) < n:
            mixed.append(ph)
    return freq, mixed


def rewrite(ph, freq_n):
    """greedy FFF, then FF (the rewrite of an FF | FFF index), as keys"""
    out, i = [], 0
    f = ph < freq_n
    while i < len(ph):
        if i + 2 < len(ph) and f[i] and f[i + 1] and f[i + 2]:
            out.append(int(pair_key(ph[i:i + 1], ph[i + 1:i + 2], ph[i + 2:i + 3], ty=4)[0])); i += 3
        elif i + 1 < len(ph) and f[i] and f[i + 1]:
            out.append(int(pair_key(ph[i:i + 1], ph[i + 1:i + 2], ty=1)[0])); i += 2
        else:
            out.append(int(synth.term_keys_np(ph[i:i + 1])[0])); i += 1
    return out


def run(ix, qkeys, reps=5):
    res = {}
    for name, rt in (("topkcount", ResultType.TopkCount), ("topk", ResultType.Topk)):
        ix.search_lexical_batch(qkeys, QueryType.Phrase, 10, rt)
        t = []
        for _ in range(reps):
            t0 = time.perf_counter(); ix.search_lexical_batch(qkeys, QueryType.Phrase, 10, rt); t.append(time.perf_counter() - t0)
        st = ix.last_stats()
        res[name] = dict(qps=round(len(qkeys) / float(np.median(t)), 1), kernel_ms=st["dominant_kernel_ns"] / 1e6)
    lat = []
    for q in qkeys[:256]:
        t0 = time.perf_counter(); ix.search_lexical_batch([q], QueryType.Phrase, 10, ResultType.TopkCount); lat.append(time.perf_counter() - t0)
    res["batch1_p50_us"] = round(float(np.percentile(lat, 50)) * 1e6, 1)
    res["batch1_p99_us"] = round(float(np.percentile(lat, 99)) * 1e6, 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--vocab", type=int, default=50_000)
    ap.add_argument("--frequent", type=int, default=100)
    ap.add_argument("--queries", type=int, default=1024)
    a = ap.parse_args()
    import torch
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    lens, toks = corpus(a.docs, a.vocab, 7)
    freq, mixed = queries(lens, toks, a.frequent, a.queries, 8)
    summary = dict(docs=a.docs, frequent=a.frequent, card=card)
    for ngrams in (False, True):
        levels, len_sum = levels_of(lens, toks, a.frequent, ngrams)
        free0 = torch.cuda.mem_get_info()[0]
        ix = Index(0)
        if ngrams:
            ix.set_ngram_config(similarity=LexicalSimilarity.Bm25f)
        for lv in levels:
            ix.add_lexical_level(lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"], lv["doc_len_bytes"],
                                 lv["positions"], lv.get("ngram_tfs"), lv.get("ngram_df_bytes"))
        ix.commit(a.docs, len_sum)
        hbm = free0 - torch.cuda.mem_get_info()[0]
        name = "FF|FFF" if ngrams else "SingleTerm"
        summary[name] = dict(hbm_bytes=int(hbm), postings=int(sum(len(lv["doc_ids"]) for lv in levels)))
        for qs_name, qs in (("frequent", freq), ("mixed", mixed)):
            qk = [rewrite(q, a.frequent) if ngrams else [int(x) for x in synth.term_keys_np(q)] for q in qs]
            r = run(ix, qk)
            print(json.dumps(dict(index=name, queries=qs_name, card=card, **r)))
            summary[name][qs_name] = r
        ix.close()
        del levels
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
