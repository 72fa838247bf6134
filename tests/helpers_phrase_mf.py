"""Multi-field token-sequence corpora for the phrase tests: every document is F token sequences, one per indexed field, so the ground truth
of a phrase query is a substring search inside one (allowed) field — independent of the oracle's and the GPU's position arithmetic."""
import numpy as np

from oracle import oracle as O
from seekstorm_b200 import synth

# mean token count per field: a short title, a long body, then two middle-sized fields
FIELD_MEAN_LEN = (6, 40, 15, 25)


def levels_from_docs(docs, n_fields, docs_per_level=65536):
    """docs: list of documents, each a sequence of n_fields int token arrays.  -> (levels as neutral dicts: tfs u16 [np, F], doc_len_bytes
    u8 [F, n_docs], positions u16 field-major inside each posting (field 0's run first, each run ascending from 0)), len_sum"""
    levels, len_sum = [], 0
    n_docs = len(docs)
    for li, base in enumerate(range(0, n_docs, docs_per_level)):
        nd = min(docs_per_level, n_docs - base)
        tok, doc_of, fld, pos = [], [], [], []
        lens = np.zeros((n_fields, nd), dtype=np.int64)
        for d in range(nd):
            for f in range(n_fields):
                s = np.asarray(docs[base + d][f], dtype=np.int64)
                lens[f, d] = len(s)
                tok.append(s); doc_of.append(np.full(len(s), d, dtype=np.int64)); fld.append(np.full(len(s), f, dtype=np.int64))
                pos.append(np.arange(len(s), dtype=np.int64))
        tok, doc_of, fld, pos = (np.concatenate(a) for a in (tok, doc_of, fld, pos))
        order = np.lexsort((pos, fld, doc_of, tok))                     # term-major, doc ascending, then field, then position
        tok, doc_of, fld, pos = tok[order], doc_of[order], fld[order], pos[order]
        key = tok * nd + doc_of                                         # postings = runs of equal (term, doc)
        starts = np.flatnonzero(np.concatenate([[True], key[1:] != key[:-1]]))
        p_tok, p_doc = tok[starts], doc_of[starts]
        posting_of = np.repeat(np.arange(len(starts)), np.diff(np.concatenate([starts, [len(key)]])))
        tfs = np.zeros((len(starts), n_fields), dtype=np.int64)
        np.add.at(tfs, (posting_of, fld), 1)
        t_starts = np.flatnonzero(np.concatenate([[True], p_tok[1:] != p_tok[:-1]]))
        terms = p_tok[t_starts]
        offs = np.concatenate([t_starts, [len(p_tok)]]).astype(np.uint32)
        lb = np.vectorize(lambda x: synth.int_to_byte4(int(x)), otypes=[np.uint8])(lens).astype(np.uint8)
        len_sum += int(np.vectorize(lambda b: synth.byte4_to_int(int(b)), otypes=[np.int64])(lb).sum())
        levels.append(dict(level_id=li, n_docs=nd, term_keys=synth.term_keys_np(terms).astype(np.uint64), posting_offsets=offs,
                           doc_ids=p_doc.astype(np.uint16), tfs=np.ascontiguousarray(tfs.astype(np.uint16)),
                           doc_len_bytes=np.ascontiguousarray(lb), positions=pos.astype(np.uint16)))
    return levels, len_sum


def multifield_sequence_corpus(n_docs, vocab, n_fields, seed, docs_per_level=65536):
    """-> (docs: list of [F token arrays], levels, len_sum); field f's lengths are geometric with mean FIELD_MEAN_LEN[f], Zipf-like tokens"""
    rng = np.random.default_rng(seed)
    w = 1.0 / (np.arange(vocab) + 3.0)
    w /= w.sum()
    per_field = []
    for f in range(n_fields):
        lens = np.clip(rng.geometric(1.0 / FIELD_MEAN_LEN[f], n_docs), 1, 400)
        toks = rng.choice(vocab, size=int(lens.sum()), p=w).astype(np.int64)
        per_field.append(np.split(toks, np.cumsum(lens)[:-1]))
    docs = [[per_field[f][d] for f in range(n_fields)] for d in range(n_docs)]
    levels, len_sum = levels_from_docs(docs, n_fields, docs_per_level)
    return docs, levels, len_sum


def phrase_queries_mf(docs, seed, n, vocab):
    """phrases of 2..6 tokens: most cut out of one field of a real document, some shuffled / random (mostly no match), some with a
    repeated bigram"""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        doc = docs[int(rng.integers(0, len(docs)))]
        s_f = doc[int(rng.integers(0, len(doc)))]
        m = int(rng.integers(2, 7))
        if len(s_f) < m:
            continue
        s = int(rng.integers(0, len(s_f) - m + 1))
        ph = [int(x) for x in s_f[s: s + m]]
        r = rng.random()
        if r < 0.2:
            rng.shuffle(ph)
        elif r < 0.3:
            ph = [int(x) for x in rng.integers(0, min(vocab, 30), m)]
        elif r < 0.4:
            ph = ph[:2] + ph[:2] + ph[2:3]
        out.append(ph)
    return out


def contains_phrase_fields(doc, ph, field_mask=0):
    """the phrase occurs as a contiguous substring of one field of the doc that the field filter allows (field_mask 0 = every field)"""
    m = len(ph)
    for f, seq in enumerate(doc):
        if field_mask and not (field_mask >> f) & 1:
            continue
        if any(all(seq[s + i] == ph[i] for i in range(m)) for s in range(len(seq) - m + 1)):
            return True
    return False


class PhraseFieldsOracle:
    """CPU oracle of QueryType::Phrase on an index with one or several indexed fields (add_result.rs:3247-3389), built on the C oracle.

    The C oracle scores the intersection of the phrase's unique terms (BM25F over all fields in first-occurrence order, the term-level
    field-filter rule of field_filter_set, the delete set); the phrase condition is restated here from the levels' own position layout:
    a posting holds sum_f tfs[p][f] positions, one run per field (field 0 first), each run restarting from 0.  Every position is tagged
    with its (doc, field), and a doc matches when some (doc, field, p) has token i at (doc, field, p + i) for every i, in a field the
    field filter allows (field_mask 0 = every field)."""

    def __init__(self, levels, n_docs, len_sum, boosts=None):
        self.orc = O.OracleIndex()
        if boosts is not None and len(boosts) > 1:
            self.orc.set_fields(boosts)
        for lv in levels:
            self.orc.add_level({k: v for k, v in lv.items() if k != "positions"})
        self.orc.commit(n_docs, len_sum)
        self.n_docs = n_docs
        self._cache = {}                                        # phrase matches by (keys, field_mask): independent of the delete set
        self.levels = []
        for lv in levels:
            tfs = np.asarray(lv["tfs"], dtype=np.int64)
            tfs = tfs.reshape(len(tfs), -1)
            nf = tfs.shape[1]
            pos_off = np.concatenate([[0], np.cumsum(tfs.sum(axis=1))])
            assert pos_off[-1] == len(lv["positions"])
            term = {int(k): i for i, k in enumerate(np.asarray(lv["term_keys"], dtype=np.uint64).tolist())}
            self.levels.append((lv["level_id"], term, np.asarray(lv["posting_offsets"], dtype=np.int64), np.asarray(lv["doc_ids"], dtype=np.int64),
                                tfs, pos_off, np.asarray(lv["positions"], dtype=np.int64), nf))

    def set_deleted(self, doc_ids):
        self.orc.set_deleted(doc_ids)

    @staticmethod
    def _occurrences(lvl, t):
        """key = ((doc * F + field) << 16) | position for every occurrence of term index t in the level"""
        _, _, offs, ids, tfs, pos_off, positions, nf = lvl
        j0, j1 = offs[t], offs[t + 1]
        tf = tfs[j0:j1]
        doc = np.repeat(ids[j0:j1], tf.sum(axis=1))
        field = np.repeat(np.tile(np.arange(nf), j1 - j0), tf.ravel())
        return ((doc * nf + field) << 16) | positions[pos_off[j0]:pos_off[j1]]

    def phrase_docs(self, seq_keys, field_mask=0):
        """global ids of the docs where the phrase occurs inside one allowed field"""
        ck = (tuple(int(k) for k in seq_keys), field_mask)
        if ck in self._cache:
            return self._cache[ck]
        out = set()
        for lvl in self.levels:
            level_id, term, nf = lvl[0], lvl[1], lvl[7]
            if any(int(k) not in term for k in seq_keys):
                continue
            occ = {}
            starts = None
            for i, k in enumerate(seq_keys):
                if int(k) not in occ:
                    occ[int(k)] = self._occurrences(lvl, term[int(k)])
                o = occ[int(k)]
                s = o[(o & 0xFFFF) >= i] - i                     # start position p of a phrase with token i at p + i (ascending)
                if starts is None:
                    starts = s
                else:
                    j = np.minimum(np.searchsorted(s, starts), max(len(s) - 1, 0))
                    starts = starts[(s[j] == starts)] if len(s) else s
            dfield = starts >> 16
            field, doc = dfield % nf, dfield // nf
            if field_mask and nf > 1:
                doc = doc[((field_mask >> field) & 1) == 1]
            out.update(int(d) | (level_id << 16) for d in np.unique(doc))
        self._cache[ck] = out
        return out

    def search_phrase(self, seq_keys, k, result_type, field_mask=0):
        """-> (hits [(doc id, score)] in canonical order, at most k; count)"""
        seq_keys = [int(x) for x in seq_keys]
        if len(seq_keys) < 2:                                   # one token: a plain term query
            return self.orc.search(seq_keys, O.QUERY_INTERSECTION, k, result_type, field_mask=field_mask)
        match = self.phrase_docs(seq_keys, field_mask)
        if not match:
            return [], 0
        unique = list(dict.fromkeys(seq_keys))
        hits, _ = self.orc.search(unique, O.QUERY_INTERSECTION, max(self.n_docs, 1), O.RESULT_TOPKCOUNT, field_mask=field_mask)
        keep = [(d, s) for d, s in hits if d in match]
        return ([] if result_type == O.RESULT_COUNT else keep[:k]), len(keep)
