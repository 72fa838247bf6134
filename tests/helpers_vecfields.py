"""Multi-vector documents: a numpy restatement of the reference's search_vector_shard record loop with the field filter
(vector.rs:1397-1467) and of TopK::push (vector.rs:410-496), plus a vector.bin writer that emits VectorHeader.field_id / chunk_id.

The corpus is given in record order (level by level, cluster by cluster, record by record), as flat per-row arrays, with a precomputed
score matrix S[q, row] (the similarity the scan computes for that row: f32 dot / -squared distance, or the int8 epilogue).
"""
import struct

import numpy as np


def threshold_premap(t, euclidean):
    """TopK::new (vector.rs:388-399): the similarity threshold in score units."""
    if t is None:
        return None
    if euclidean:
        return np.float32(-t)
    return np.float32((np.float32(t) * np.float32(2.0) - np.float32(1.0)) / np.float32(1.0 / 16129.0))


def passes(mask, field):
    """field_filter_set.contains(record.header.field_id) (vector.rs:1411-1412); mask 0 = empty set = no filter."""
    return mask == 0 or (mask >> int(field)) & 1 == 1


def search_fields(S, doc, field, chunk, k, masks, deleted=(), threshold=None, in_scope=None):
    """Per query: the k best docs (score desc, doc id asc), each with the field / chunk of its best row that passes the query's mask
    (the earliest row on equal scores: push replaces only on a strictly better score), and observed = rows in scope whose field passes
    (deleted rows included, as the library counts them).

    S: [nq, n_rows] scores; doc / field / chunk: [n_rows]; masks: [nq]; in_scope: None (AnnMode::All) or [nq, n_rows] bool (the rows of
    the clusters the IVF probe selected).  Returns a list of (hits [(doc, score, field, chunk)], observed) per query."""
    deleted = set(int(d) for d in deleted)
    out = []
    for q in range(S.shape[0]):
        best = {}
        observed = 0
        for r in range(S.shape[1]):
            if in_scope is not None and not in_scope[q, r]:
                continue
            if not passes(int(masks[q]), field[r]):
                continue
            observed += 1
            d = int(doc[r])
            if d in deleted:
                continue
            s = np.float32(S[q, r])
            if s != s or (threshold is not None and s < threshold):
                continue
            if d not in best or s > best[d][0]:
                best[d] = (s, int(field[r]), int(chunk[r]))
        hits = sorted(((d, float(v[0]), v[1], v[2]) for d, v in best.items()), key=lambda h: (-h[1], h[0]))[:k]
        out.append((hits, observed))
    return out


class TopK:
    """TopK::push as the reference writes it (vector.rs:410-496): k slots, per-doc replacement on a strictly better score, the lowest
    slot replaced when a new doc beats it.  Used to show that search_fields is the same list whenever no ties cross the k-th place."""

    def __init__(self, k, threshold=None):
        self.k, self.items, self.lowest = k, [], -np.inf
        self.threshold = -np.inf if threshold is None else threshold
        self.observed = 0

    def push(self, doc, field, chunk, score):
        self.observed += 1
        if score < self.threshold or (len(self.items) == self.k and score <= self.lowest):
            return
        for it in self.items:
            if it[0] == doc:
                if score > it[1]:
                    it[1:] = [score, field, chunk]
                return
        if len(self.items) < self.k:
            self.items.append([doc, score, field, chunk])
            return
        mi = min(range(len(self.items)), key=lambda i: (self.items[i][1], i))
        if score > self.items[mi][1]:
            self.lowest = self.items[mi][1]
            self.items[mi] = [doc, score, field, chunk]

    def result(self):
        return [tuple(it) for it in sorted(self.items, key=lambda it: (-it[1], it[0]))]


def search_fields_topk(S, doc, field, chunk, k, masks, deleted=(), threshold=None):
    """The reference's loop with its TopK (no IVF): per query (hits, observed)."""
    deleted = set(int(d) for d in deleted)
    out = []
    for q in range(S.shape[0]):
        t = TopK(k, threshold)
        for r in range(S.shape[1]):
            if not passes(int(masks[q]), field[r]):
                continue
            if int(doc[r]) in deleted:
                t.observed += 1          # the library counts deleted rows in observed (documented deviation)
                continue
            t.push(int(doc[r]), int(field[r]), int(chunk[r]), np.float32(S[q, r]))
        out.append(([(d, float(s), f, c) for d, s, f, c in t.result()], t.observed))
    return out


def write_vector_bin_fields(levels):
    """levels: list of (local_ids u16, rows f32 [n, dims], field_ids, chunk_ids[, cluster child counts]) — vector.bin with the
    packed 24-byte VectorHeader {u16 doc_id, u32 field_id, u32 chunk_id, f32 scale, f32 norm, i16 zero_point, i32 sum_q} (vector.rs:62-73)."""
    out = []
    for lv in levels:
        ids, rows, fields, chunks = lv[0], lv[1], lv[2], lv[3]
        n = len(ids)
        counts = [n] if len(lv) < 5 or lv[4] is None else [int(c) for c in lv[4]]
        assert sum(counts) == n
        out.append(struct.pack("<I", len(counts)) + b"".join(struct.pack("<I", c) for c in counts))
        for i in range(n):
            out.append(struct.pack("<HIIffhi", int(ids[i]), int(fields[i]), int(chunks[i]), 1.0, 1.0, 0, 0))
            out.append(np.asarray(rows[i], dtype="<f4").tobytes())
    return b"".join(out)


def read_vector_bin_headers(data, dims):
    """(doc_id, field_id, chunk_id) of every record of a vector.bin, in file order."""
    pos, rec, out = 0, 24 + 4 * dims, []
    while pos < len(data):
        (nc,) = struct.unpack_from("<I", data, pos)
        counts = struct.unpack_from("<%dI" % nc, data, pos + 4)
        pos += 4 + 4 * nc
        for _ in range(sum(counts)):
            d, f, c = struct.unpack_from("<HII", data, pos)
            out.append((d, f, c))
            pos += rec
    return out


def tagged_corpus(n_docs, dims, seed, n_fields=3, max_chunks=3):
    """A multi-vector corpus: every doc has 1..max_chunks chunks in each of n_fields fields, in record order (doc by doc, field by field).
    A doc's rows are one base vector plus noise, so they score close together.  Returns (rows f32 [n, dims], doc index, fields, chunks);
    callers split the docs into levels."""
    rng = np.random.default_rng(seed)
    ids, fields, chunks = [], [], []
    for d in range(n_docs):
        for f in range(n_fields):
            for c in range(int(rng.integers(1, max_chunks + 1))):
                ids.append(d); fields.append(f); chunks.append(c)
    base = rng.standard_normal((n_docs, dims)).astype(np.float32)
    ids = np.array(ids, dtype=np.int64)
    rows = base[ids] + np.float32(0.35) * rng.standard_normal((len(ids), dims)).astype(np.float32)
    return rows.astype(np.float32), ids, np.array(fields, dtype=np.uint8), np.array(chunks, dtype=np.uint32)


def search_fields_fast(Sq, doc, field, chunk, k, mask, deleted_rows=None, threshold=None, scope=None):
    """search_fields for one query, vectorised (large corpora): Sq [n_rows] scores.  Each hit also carries the margin of its best row
    over the doc's runner-up passing row (inf when it has one row), so callers can skip best-row checks the scan precision cannot decide."""
    ok = np.ones(Sq.shape[0], dtype=bool) if mask == 0 else ((int(mask) >> field.astype(np.int64)) & 1).astype(bool)
    if scope is not None:
        ok &= scope
    observed = int(ok.sum())
    if deleted_rows is not None:
        ok &= ~deleted_rows
    ok &= Sq == Sq
    if threshold is not None:
        ok &= Sq >= threshold
    idx = np.nonzero(ok)[0]
    if len(idx) == 0:
        return [], observed
    s, d = Sq[idx].astype(np.float64), doc[idx]
    o = np.lexsort((idx, -s, d))                          # per doc: best score first, the earliest row on equal scores
    so, do = s[o], d[o]
    head = np.r_[True, do[1:] != do[:-1]]
    hpos = np.nonzero(head)[0]
    nxt = np.full(len(hpos), -np.inf)
    two = np.r_[~head[1:], False][hpos]                   # the doc has a runner-up row
    nxt[two] = so[hpos[two] + 1]
    margin = so[hpos] - nxt
    first = o[hpos]
    top = np.lexsort((d[first], -s[first]))[:k]
    hits = [(int(d[first[t]]), float(s[first[t]]), int(field[idx[first[t]]]), int(chunk[idx[first[t]]]), float(margin[t])) for t in top]
    return hits, observed
