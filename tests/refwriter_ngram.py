"""TEST INFRASTRUCTURE: the index.bin writer of tests/refwriter.py for shards built with n-gram indexing (a restatement of the reference's
writer, like refwriter.py; no file written by the reference itself can be produced here).

What differs from refwriter.py (paths relative to the reference's seekstorm/src/):
  * key head of 22 (bigrams only) / 23 bytes (trigrams): u64 key, u16 count - 1, u16 max_docid, u16 max_p_docid, the components' df
    bytes posting_count_ngram_{1,2[,3]}_compressed, u16 pivot, u32 compression type << 30 | pointer range  (compress_postinglist.rs:28-230,
    339-409; read at search.rs:2236-2250); single-term keys carry zero bytes there
  * n-gram postings are never embedded in their pointer (index_posting.rs:445) and their blob starts with the VINT component tfs
    tf_ngram1, tf_ngram2[, tf_ngram3] ahead of positions_count (add_result.rs:2076-2089)
"""
import struct

import numpy as np

import refwriter as R


def _key_body(doc_ids, positions, prefixes):
    """refwriter._key_body with a per-posting blob prefix (the component tfs); a posting with a prefix is never embedded"""
    count = len(doc_ids)
    blobs, ptrs, cum, pivot = [], [], 0, None
    for p in range(count):
        deltas = positions[p]
        ptr_size = 2 if (cum < 32768 - 4096 and pivot is None) else 3
        if ptr_size == 3 and pivot is None:
            pivot = p
        if not prefixes[p] and R._embed(deltas, ptr_size):
            ptrs.append(R._embed_bytes(deltas, ptr_size))
            continue
        blob = prefixes[p] + R.vint(len(deltas)) + b"".join(R.vint(int(d)) for d in deltas)
        cum += len(blob)
        blobs.append(blob)
        if ptr_size == 2:
            ptrs.append(struct.pack("<H", cum & 0x7FFF))
        else:
            ptrs.append(bytes([cum & 0xFF, (cum >> 8) & 0xFF, (cum >> 16) & 0x7F]))
    if pivot is None:
        pivot = count
    pos_area = b"".join(reversed(blobs))
    runs = []
    for d in doc_ids:
        if runs and runs[-1][0] + runs[-1][1] + 1 == d:
            runs[-1][1] += 1
        else:
            runs.append([int(d), 0])
    thr = min(count // 2, 65535) if count < 4096 else 2048
    if len(runs) < thr:
        ctype = 3
        cont = struct.pack("<H", len(runs)) + b"".join(struct.pack("<HH", s, l) for s, l in runs)
    elif count < 4096:
        ctype = 1
        cont = np.asarray(doc_ids, dtype="<u2").tobytes()
    else:
        ctype = 2
        bm = np.zeros(8192, dtype=np.uint8)
        ids = np.asarray(doc_ids, dtype=np.int64)
        np.bitwise_or.at(bm, ids >> 3, (1 << (ids & 7)).astype(np.uint8))
        cont = bm.tobytes()
    return pos_area + b"".join(ptrs) + cont, len(pos_area), pivot, ctype


def write_index_bin_ngrams(levels, n_docs_total, key_head_size=23):
    """levels: neutral dicts with positions, ngram_tfs [n_postings, 3] and ngram_df_bytes [n_terms, 3] (tests/helpers_ngram.ngram_corpus),
    level_id ascending from 0, each full (65536 docs) except the last.  Returns (bytes, positions_sum_normalized)."""
    from seekstorm_b200 import synth
    assert key_head_size in (22, 23)
    n_df = key_head_size - 20
    out = [struct.pack("<HH", 6, 1)]
    cum_docs, cum_len = 0, 0
    nseg = 1 << R.SEGMENT_BITS
    for li, lv in enumerate(levels):
        assert lv["level_id"] == li
        if li == 0:
            out.append(struct.pack("<H", 0))
        dl = np.zeros(65536, dtype=np.uint8)
        dl[:lv["n_docs"]] = lv["doc_len_bytes"]
        out.append(dl.tobytes())
        cum_docs += lv["n_docs"]
        cum_len += int(sum(synth.byte4_to_int(int(b)) for b in lv["doc_len_bytes"]))
        out.append(struct.pack("<QQ", cum_docs, cum_len))
        segs = [[] for _ in range(nseg)]
        offs = lv["posting_offsets"]
        pos_all = lv["positions"]
        pos_off = np.concatenate([[0], np.cumsum(lv["tfs"].astype(np.int64))])
        for t, key in enumerate(lv["term_keys"]):
            key = int(key)
            segs[(key >> 40) & (nseg - 1)].append((key, t))
        heads, bodies = [], []
        for s in range(nseg):
            segs[s].sort()
            body, hb = b"", b""
            for key, t in segs[s]:
                a, b = int(offs[t]), int(offs[t + 1])
                ids = lv["doc_ids"][a:b]
                ty = key & 7
                n_comp = 0 if ty == 0 else (2 if ty <= 3 else 3)
                assert n_comp <= n_df
                plist = [R.deltas_of(pos_all[pos_off[j]:pos_off[j + 1]]) for j in range(a, b)]
                prefixes = [b"".join(R.vint(int(c)) for c in lv["ngram_tfs"][j][:n_comp]) for j in range(a, b)]
                kb, rng_off, pivot, ctype = _key_body(ids, plist, prefixes)
                ctp = (ctype << 30) | (len(body) + rng_off)
                dfb = bytes(int(x) for x in lv["ngram_df_bytes"][t][:n_df]) if ty else bytes(n_df)
                hb += struct.pack("<QHHH", key, len(ids) - 1, int(ids[-1]), 0) + dfb + struct.pack("<HI", pivot, ctp)
                body += kb
            heads.append(hb); bodies.append(body)
        out.append(b"".join(struct.pack("<II", len(heads[s]) + len(bodies[s]), len(segs[s])) for s in range(nseg)))
        for s in range(nseg):
            out.append(heads[s]); out.append(bodies[s])
    assert cum_docs == n_docs_total
    return b"".join(out), cum_len


def ngram_checksum(levels, decode_positions):
    """ssb_index_bin_inspect_ngrams' checksums restated over the neutral levels: keys in file order (segment, then key), per key its
    level and df bytes, per posting (doc id, tf, component tfs), and the positions of the n-gram postings"""
    nseg = 1 << R.SEGMENT_BITS
    h, hp = 1469598103934665603, 1469598103934665603
    M = (1 << 64) - 1
    terms = postings = tf_sum = 0

    def mix(h, x):
        return ((h ^ x) * 1099511628211) & M
    for lv in levels:
        offs = lv["posting_offsets"]
        pos_off = np.concatenate([[0], np.cumsum(lv["tfs"].astype(np.int64))])
        order = sorted(((int(k) >> 40) & (nseg - 1), int(k), t) for t, k in enumerate(lv["term_keys"]))
        for _, key, t in order:
            if key & 7 == 0:
                continue
            f = [int(x) for x in lv["ngram_df_bytes"][t]]
            if key & 7 <= 3:
                f[2] = 0
            terms += 1
            h = mix(h, key)
            h = mix(h, (lv["level_id"] << 32) | (f[0] << 16) | (f[1] << 8) | f[2])
            for j in range(int(offs[t]), int(offs[t + 1])):
                c = [int(x) for x in lv["ngram_tfs"][j]]
                tf = int(lv["tfs"][j])
                h = mix(h, (int(lv["doc_ids"][j]) << 48) | (tf << 32) | (c[0] << 16) | c[1])
                h = mix(h, c[2])
                postings += 1; tf_sum += tf
                if decode_positions:
                    for p in lv["positions"][pos_off[j]:pos_off[j + 1]]:
                        hp = mix(hp, int(p))
    return [len(levels), terms, postings, tf_sum, h, hp if decode_positions else 0, 0, 0]
