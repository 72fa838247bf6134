"""Sorted lexical search (`result_sort`) restated for the tests: the oracle's exhaustive match list (every match with its exact score) ordered
by a typed restatement of result_ordering_shard (min_heap.rs:574-1051) over the raw facet rows handed to ssb_set_facets — values decoded
and compared in their own FieldType, String facets by their strings' bytes — never through the library's sort keys."""
import ctypes as C
import functools
import math
import struct

import numpy as np

from oracle import oracle as O
from seekstorm_b200 import _lib


def _cmp(a, b):
    return int(a > b) - int(a < b)


def _cmp_value(x, y):
    """one facet value against another in the facet's type; floats by PartialOrd with -0.0 == +0.0, and NaN (where the reference's
    partial_cmp yields Equal, i.e. an arrival-order dependent result) above +inf — the library's documented total order"""
    if isinstance(x, float):
        nx, ny = math.isnan(x), math.isnan(y)
        if nx or ny:
            return _cmp(nx, ny)
        return _cmp(x, y)
    return _cmp(x, y)


class FacetRows:
    """the shard's facet file as handed to ssb_set_facets / the oracle: rows [n_docs, row_bytes] u8 of doc ids first_doc.., each facet a
    (FieldType, byte offset) inside the row.  Values are decoded from those bytes in the facet's own type, the way result_ordering_shard
    reads facets_file_mmap; a String facet's id is looked up in its value strings (`facet.values`) and compared as UTF-8 bytes (Rust String
    order = memcmp order)."""
    _DT = {_lib.FACET_U8: "<u1", _lib.FACET_U16: "<u2", _lib.FACET_U32: "<u4", _lib.FACET_U64: "<u8", _lib.FACET_I8: "<i1",
           _lib.FACET_I16: "<i2", _lib.FACET_I32: "<i4", _lib.FACET_I64: "<i8", _lib.FACET_TIMESTAMP: "<i8", _lib.FACET_F32: "<f4",
           _lib.FACET_F64: "<f8", _lib.FACET_STRING16: "<u2", _lib.FACET_STRING32: "<u4"}

    def __init__(self, rows, first_doc, fields, strings=None):
        """fields: name -> (FieldType, offset); strings: name -> value strings by id (String facets)"""
        self.rows, self.first, self.fields, self.strings = np.asarray(rows, dtype=np.uint8), int(first_doc), dict(fields), dict(strings or {})
        self._ranks = {}

    @staticmethod
    def of_index(ix, strings=None):
        """the rows an Index handed to ssb_set_facets"""
        rows, fields, first, n, _ = ix._facet_rows
        return FacetRows(rows[:n], first, {name: (t, fields[i].offset) for name, (i, t) in ix._facet_schema.items()}, strings)

    @staticmethod
    def pack(cols, first_doc=0, string_facets=(), timestamp_facets=(), strings=None):
        """a facet file of typed columns, packed field after field (the reference's facet file layout)"""
        kinds = {"uint8": _lib.FACET_U8, "uint16": _lib.FACET_U16, "uint32": _lib.FACET_U32, "uint64": _lib.FACET_U64, "int8": _lib.FACET_I8,
                 "int16": _lib.FACET_I16, "int32": _lib.FACET_I32, "int64": _lib.FACET_I64, "float32": _lib.FACET_F32, "float64": _lib.FACET_F64}
        n = len(next(iter(cols.values())))
        width = sum(np.asarray(c).dtype.itemsize for c in cols.values())
        rows, fields, off = np.zeros((n, width), dtype=np.uint8), {}, 0
        for name, c in cols.items():
            c = np.ascontiguousarray(c)
            t = kinds[c.dtype.name]
            if name in string_facets:
                t = _lib.FACET_STRING16 if c.dtype.itemsize == 2 else _lib.FACET_STRING32
            if name in timestamp_facets:
                t = _lib.FACET_TIMESTAMP
            rows[:, off:off + c.dtype.itemsize] = c.view(np.uint8).reshape(n, c.dtype.itemsize)
            fields[name] = (t, off)
            off += c.dtype.itemsize
        return FacetRows(rows, first_doc, fields, strings)

    def _raw(self, name):
        t, off = self.fields[name]
        w = np.dtype(self._DT[t]).itemsize
        return t, w, off

    def value(self, name, doc):
        """the typed value the reference compares: int, float, or a String facet's value as UTF-8 bytes"""
        t, w, off = self._raw(name)
        b = self.rows[doc - self.first, off:off + w].tobytes()
        if t in (_lib.FACET_STRING16, _lib.FACET_STRING32):
            return self.strings[name][int.from_bytes(b, "little")].encode("utf-8")
        if t == _lib.FACET_F32:
            return struct.unpack("<f", b)[0]
        if t == _lib.FACET_F64:
            return struct.unpack("<d", b)[0]
        return int.from_bytes(b, "little", signed=t in (_lib.FACET_I8, _lib.FACET_I16, _lib.FACET_I32, _lib.FACET_I64, _lib.FACET_TIMESTAMP))

    def rank(self, name):
        """per row the dense rank of its value in the facet's type (floats: -0.0 == +0.0, NaN last; strings by their UTF-8 bytes)"""
        if name not in self._ranks:
            t, w, off = self._raw(name)
            c = np.frombuffer(np.ascontiguousarray(self.rows[:, off:off + w]).tobytes(), dtype=self._DT[t])
            if t in (_lib.FACET_STRING16, _lib.FACET_STRING32):
                enc = [v.encode("utf-8") for v in self.strings[name]]
                pos = {x: i for i, x in enumerate(sorted(set(enc)))}
                r = np.asarray([pos[x] for x in enc], dtype=np.int64)[c.astype(np.int64)]
            elif t in (_lib.FACET_F32, _lib.FACET_F64):
                r = np.unique(c.astype(np.float64) + 0.0, return_inverse=True, equal_nan=True)[1]   # -0.0 -> +0.0; NaN sorts last
            else:
                r = np.unique(c, return_inverse=True)[1]
            self._ranks[name] = np.asarray(r, dtype=np.int64).reshape(-1)
        return self._ranks[name]


def compare(a, b, criteria, facets):
    """> 0: hit a ranks before hit b.  criteria: [(name, descending)] with name a facet, "_id" or "_score"; _id / _score end the
    comparison (min_heap.rs:580-604); all criteria equal -> score desc (:1043-1050), then doc id asc"""
    (da, sa), (db, sb) = a, b
    for name, desc in criteria:
        if name == "_id":
            o = _cmp(da, db)
            return o if desc else -o
        if name == "_score":
            o = _cmp(np.float32(sa), np.float32(sb))
            if o:
                return o if desc else -o
            return _cmp(db, da)
        o = _cmp_value(facets.value(name, da), facets.value(name, db))
        if o:
            return o if desc else -o
    o = _cmp(np.float32(sa), np.float32(sb))
    return o if o else _cmp(db, da)


def sort_hits_cmp(hits, criteria, facets):
    """sorted by `compare` (one Python comparison per pair: the restatement itself, for small lists)"""
    return sorted(hits, key=functools.cmp_to_key(lambda a, b: -compare(a, b, criteria, facets)))


_HIT = np.dtype([("doc_id", "<u8"), ("score", "<f4"), ("pad", "<u4")])


def all_matches(orc, n_docs, term_keys, query_type, phrase=False, not_keys=None, filters=None, set_values=None):
    """every match of one query with its exact score: the oracle's exhaustive top-n_docs search (the same C entry points
    OracleIndex.search / search_phrase call), its hit buffer read as a structured array (doc_id, score).  -> (hits, count)"""
    L = O.lib()
    keys = np.ascontiguousarray(np.array(term_keys, dtype=np.uint64))
    buf = (O.OrcHit * max(n_docs, 1))()
    n, tot = C.c_uint32(0), C.c_uint64(0)
    out = (buf, C.byref(n), C.byref(tot))
    if phrase:
        f = L.orc_search_lexical_phrase
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]
        rc = f(orc._h, O._ptr(keys), len(keys), n_docs, O.RESULT_TOPKCOUNT, *out)
    elif filters:
        nk = np.ascontiguousarray(np.array(not_keys if not_keys else [0], dtype=np.uint64))
        fa = (O.OrcFacetFilter * len(filters))(*[O.OrcFacetFilter(*[int(x) for x in f]) for f in filters])
        sv = np.ascontiguousarray(np.array(set_values if set_values else [0], dtype=np.uint64))
        f = L.orc_search_lexical_ex
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                      C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]
        rc = f(orc._h, O._ptr(keys), len(keys), O._ptr(nk), len(not_keys) if not_keys else 0, fa, len(filters), O._ptr(sv), 0,
               query_type, n_docs, O.RESULT_TOPKCOUNT, *out)
    elif not_keys:
        nk = np.ascontiguousarray(np.array(not_keys, dtype=np.uint64))
        rc = L.orc_search_lexical_not(orc._h, O._ptr(keys), len(keys), O._ptr(nk), len(nk), query_type, n_docs, O.RESULT_TOPKCOUNT, *out)
    else:
        rc = L.orc_search_lexical(orc._h, O._ptr(keys), len(keys), query_type, n_docs, O.RESULT_TOPKCOUNT, *out)
    assert rc == 0, rc
    return np.frombuffer(buf, dtype=_HIT, count=n.value).copy(), int(tot.value)


def sort_hits(hits, criteria, facets, k=None):
    """the order of `compare` (test_sort_cpu pins the two together), by one np.lexsort over typed ranks: fast on long match lists.
    hits: [(doc, score)] or an all_matches array; returns the first k as [(doc, score)]"""
    if len(hits) == 0:
        return []
    if isinstance(hits, np.ndarray):
        docs, scores = hits["doc_id"].astype(np.int64), hits["score"].astype(np.float64)
        hits = None
    else:
        docs = np.asarray([d for d, _ in hits], dtype=np.int64)
        scores = np.asarray([s for _, s in hits], dtype=np.float32).astype(np.float64)
    keys, tail = [], -scores                                           # fallback: score desc
    for name, desc in criteria:
        if name == "_id":
            keys.append(-docs if desc else docs)
            tail = None
            break
        if name == "_score":
            tail = -scores if desc else scores
            break
        r = facets.rank(name)[docs - facets.first]
        keys.append(-r if desc else r)
    order = [docs] + ([tail] if tail is not None else []) + keys[::-1]   # lexsort: last key is primary
    idx = np.lexsort(order)[:k]
    return [(int(docs[i]), float(np.float32(scores[i]))) for i in idx] if hits is None else [hits[i] for i in idx]


def search_sorted(orc, n_docs, term_keys, query_type, k, result_type, criteria, facets, phrase=False, **kw):
    """the sorted search of one query: (first k hits in sort order, count).  Count ignores the sort (search.rs:2498); k = 0 is Count."""
    if result_type == O.RESULT_COUNT or k == 0:
        if phrase:
            return orc.search_phrase(term_keys, 0, O.RESULT_COUNT)
        return orc.search(term_keys, query_type, 0, O.RESULT_COUNT, **kw)
    if phrase:
        hits, tot = orc.search_phrase(term_keys, n_docs, O.RESULT_TOPKCOUNT)
    else:
        hits, tot = orc.search(term_keys, query_type, n_docs, O.RESULT_TOPKCOUNT, **kw)
    return sort_hits(hits, criteria, facets, k), tot


def sort_criteria(criteria):
    """[(name, descending)] -> the ResultSort list of the Python mirror"""
    from seekstorm_b200 import ResultSort, SortOrder
    return [ResultSort(n, SortOrder.Descending if d else SortOrder.Ascending) for n, d in criteria]
