"""Host-side mirror of the reference's search interface for the hot path, on top of the C-ABI.

Mirrors (names, argument meaning, error behaviour) of /root/reference/seekstorm/src/:
  * `Search::search`                        search.rs:1134-1150 (impl 1153-2131)  -> Index.search
  * `QueryType`, `ResultType`, `SearchMode`, `AnnMode`   search.rs:120-185, vector_similarity.rs:43-67
  * `ResultObject` / `Result`               search.rs:186-213, min_heap.rs:17-40
  * per-shard seams search_lexical_shard (search.rs:2427-2458) / search_vector_shard (vector.rs:1105-1115)
    -> Index.search_lexical_batch / Index.search_vector_batch (batched: the GPU path amortises launches)

The reference's `search` is infallible by type: failures yield an empty `ResultObject` (search.rs:1630-1631).
The same holds here for "term not in dictionary"/empty queries; programming errors (k > 32, no GPU,
library missing) raise `SsbError` — there is no CPU fallback.

The tokenizer (tokenizer.rs) is out of scope: query strings are split on whitespace, a leading '+' marks a
mandatory term (tokenizer.rs:546-563); terms are mapped to 64-bit keys by `term_key_fn`.
"""
from __future__ import annotations

import bisect
import ctypes as C
import enum
from dataclasses import dataclass, field
from typing import Callable, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import SsbConfig, SsbHit, SsbLevelDesc, SsbLevelNgrams, SsbLexBatch, SsbStats, check, lib


class QueryType(enum.IntEnum):
    """search.rs `QueryType`.  Phrase: the query's terms in phrase order, repeats included; needs levels loaded with positions."""
    Union = 0
    Intersection = 1
    Phrase = 2


class ResultType(enum.IntEnum):
    """search.rs:150-175."""
    Count = 0
    Topk = 1
    TopkCount = 2


class VectorSimilarity(enum.IntEnum):
    """vector_similarity.rs:20-30."""
    Dot = 0
    Cosine = 1
    Euclidean = 2


@dataclass(frozen=True)
class AnnMode:
    """vector_similarity.rs:43-67: which IVF clusters of each level are searched (vector.rs:1300-1392)."""
    kind: int = 0                 # SSB_ANN_*: 0 All, 1 Nprobe, 2 Similaritythreshold, 3 NprobeSimilaritythreshold
    n_probe: int = 0
    threshold: float = 0.0

    @staticmethod
    def Nprobe(n):
        return AnnMode(1, int(n))

    @staticmethod
    def Similaritythreshold(t):
        return AnnMode(2, 0, float(t))

    @staticmethod
    def NprobeSimilaritythreshold(n, t):
        return AnnMode(3, int(n), float(t))


AnnMode.All = AnnMode()


@dataclass
class SearchMode:
    """search.rs `SearchMode::{Lexical, Vector{..}, Hybrid{..}}`."""
    kind: str = "Lexical"
    similarity_threshold: Optional[float] = None
    ann_mode: AnnMode = AnnMode.All

    @staticmethod
    def Lexical():
        return SearchMode("Lexical")

    @staticmethod
    def Vector(similarity_threshold=None, ann_mode=AnnMode.All):
        return SearchMode("Vector", similarity_threshold, ann_mode)

    @staticmethod
    def Hybrid(similarity_threshold=None, ann_mode=AnnMode.All):
        return SearchMode("Hybrid", similarity_threshold, ann_mode)


class DistanceUnit(enum.IntEnum):
    """`DistanceUnit` (index.rs) of a geo filter."""
    Kilometers = 0
    Miles = 1


@dataclass(frozen=True)
class FacetFilter:
    """`FacetFilter` (search.rs:735-860): a range filter `start <= value < end` (Rust `Range<T>`) on a numeric / timestamp facet field, or a
    value-id set on a String16 / String32 facet (values = the ids the reference resolves the filter strings to, FilterSparse::String16/32),
    or the strings of a StringSet16 / StringSet32 facet (values = [str, ...]: a doc passes when its set holds one of them, resolved like
    search.rs:2643-2710), or on a Point facet (`FacetFilter::Point`, base = (lat, lon)) the docs whose distance to base lies in start..end,
    in unit.
    field: the facet's name (Index.set_facets) or its index."""
    field: object
    start: object = None
    end: object = None
    values: Optional[Sequence[int]] = None
    base: Optional[Sequence[float]] = None
    unit: DistanceUnit = DistanceUnit.Kilometers


class RangeType(enum.IntEnum):
    """`RangeType` (search.rs:216-228) of a range facet: the count within each range, or the running sum from the top / the bottom."""
    CountWithinRange = 0
    CountAboveRange = 1
    CountBelowRange = 2


@dataclass(frozen=True)
class QueryFacet:
    """`QueryFacet` (search.rs:234-…): facet counts of the query's matches on one facet field.  A String16 / String32 field takes `prefix`
    and `length` (the `length` values with the most matches whose string starts with prefix; 0 = not collected); a numeric / Timestamp /
    F32 / F64 field takes `range_type` and `ranges` = [(label, start), ...] (start ascending; a range runs up to the next start); a Point
    field also takes `base` (lat, lon) and `unit`, and ranges over the distance to base.  A request whose shape does not fit the field's
    type, or an unknown field, is ignored as the reference does."""
    field: str
    prefix: str = ""
    length: int = 0
    range_type: RangeType = RangeType.CountWithinRange
    ranges: Sequence = ()
    base: Optional[Sequence[float]] = None
    unit: DistanceUnit = DistanceUnit.Kilometers


_VALUE_FACETS = (_lib.FACET_STRING16, _lib.FACET_STRING32, _lib.FACET_STRINGSET16, _lib.FACET_STRINGSET32)   # counted per value id
_SET_FACETS = (_lib.FACET_STRINGSET16, _lib.FACET_STRINGSET32)


@dataclass
class StringSetFacet:
    """A multi-value string facet as the reference ingests it (index.rs:5763-5801).  combos[i]: the sorted member list stored for
    combination i (the FIRST doc's list of its joined key, repeats kept); by_key: joined key -> combination id; members: the distinct
    member strings as bytes in byte-wise order (member id = position); offsets / member_ids: the CSR of ssb_set_facet_string_sets."""
    ids: np.ndarray
    combos: list
    by_key: dict
    members: list
    offsets: np.ndarray
    member_ids: np.ndarray

    def filter_values(self, strings):
        """FacetFilter::StringSet16 / 32 (search.rs:2643-2710) -> filter_set_values: per string v its member id, and the id of the
        combination whose joined key is v, flagged (SET_COMBINATION), when that combination does not hold v itself (["a", "b"] for "a_b")"""
        pos = {m: i for i, m in enumerate(self.members)}
        out = []
        for v in strings:
            m = pos.get(v.encode("utf-8"))
            if m is not None:
                out.append(m)
            c = self.by_key.get(v)
            if c is not None and v not in self.combos[c]:
                out.append(c | _lib.SET_COMBINATION)
        return out


def string_set_facet(docs, bits: int = 16) -> StringSetFacet:
    """Ingest of a StringSet16 / StringSet32 column (index.rs:5763-5801): each doc's list sorted byte-wise (Rust Vec<String>::sort) and
    joined with "_"; the joined key gets the next id on first sight and keeps that first list.  Past 65,535 (StringSet16) / 2^32 - 1
    combinations the reference writes no id for the remaining docs; this raises ValueError instead."""
    limit = 65535 if bits == 16 else (1 << 32) - 1
    by_key, combos = {}, []
    ids = np.zeros(len(docs), dtype=np.uint16 if bits == 16 else np.uint32)
    for d, lst in enumerate(docs):
        if len(combos) >= limit:
            raise ValueError(f"StringSet{bits}: more than {limit} combinations (the reference stops writing ids there)")
        key = sorted((str(x) for x in lst), key=lambda x: x.encode("utf-8"))
        c = by_key.setdefault("_".join(key), len(combos))
        if c == len(combos):
            combos.append(key)
        ids[d] = c
    members = sorted({m.encode("utf-8") for k in combos for m in k})
    pos = {m: i for i, m in enumerate(members)}
    offsets = np.zeros(len(combos) + 1, dtype=np.uint64)
    flat = []
    for c, k in enumerate(combos):
        flat.extend(pos[m.encode("utf-8")] for m in k)
        offsets[c + 1] = len(flat)
    return StringSetFacet(ids, combos, by_key, members, offsets, np.asarray(flat, dtype=np.uint32))


def prefix_rank_interval(order, prefix: bytes):
    """[lo, hi) of the ranks (positions in `order`, the sorted distinct strings as bytes) of the strings that start with prefix"""
    lo = bisect.bisect_left(order, prefix)
    succ = prefix.rstrip(b"\xff")
    if not succ:
        return lo, len(order)
    succ = succ[:-1] + bytes([succ[-1] + 1])
    return lo, bisect.bisect_left(order, succ)


def assemble_range_facet(counts, labels, range_type, prefix=""):
    """One range facet of one shard (search.rs:3660-3745): the bins with a nonzero count, RangeType applied (the running sum over those
    bins from the top or the bottom), in range order, labels attached, filtered by the label prefix."""
    vals = {i: int(c) for i, c in enumerate(counts) if c}
    rt = RangeType(range_type)
    if rt != RangeType.CountWithinRange:
        s = 0
        for i in sorted(vals, reverse=rt == RangeType.CountAboveRange):
            s += vals[i]
            vals[i] = s
    return [(labels[i], vals[i]) for i in sorted(vals) if not prefix or labels[i].startswith(prefix)]


def merge_facets(per_field, lengths):
    """Search::search's final step (search.rs:1932-1936, 2038-2048): per field, the counts of equal labels summed, then the (label, count)
    pairs by count descending (stable: ties keep their order), at most `length` of them"""
    out = {}
    for f, v in per_field.items():
        acc = {}
        for label, c in v:
            acc[label] = acc.get(label, 0) + c
        out[f] = sorted(acc.items(), key=lambda x: -x[1])[:lengths[f]]
    return out


class SortOrder(enum.IntEnum):
    """search.rs:885-890."""
    Ascending = 0
    Descending = 1


@dataclass(frozen=True)
class ResultSort:
    """`ResultSort` (search.rs:893-901): sort the hits by a facet field (name given to set_facets), "_id" or "_score".  base: the
    `FacetValue::Point` (lat, lon) of geo proximity sorting on a Point facet: the hits are ordered by their distance to it (ascending =
    nearest first); a Point facet without a base is skipped like the reference does.  A base on any other field raises
    NotImplementedError."""
    field: str
    order: SortOrder = SortOrder.Descending
    base: object = None


@dataclass
class Result:
    """min_heap.rs:17-40."""
    doc_id: int
    score: float


@dataclass
class ResultObject:
    """search.rs:186-213 (suggestions are outside the hot path).  facets: {field: [(string or range label, count), ...]}."""
    original_query: str = ""
    query: str = ""
    query_terms: list = field(default_factory=list)
    result_count: int = 0
    result_count_total: int = 0
    results: list = field(default_factory=list)
    observed_vector_count: int = 0
    observed_cluster_count: int = 0
    facets: dict = field(default_factory=dict)


def fnv1a64(term: str) -> int:
    h = 0xCBF29CE484222325
    for b in term.encode("utf-8"):
        h = ((h ^ b) * 0x100000001B3) & ((1 << 64) - 1)
    return h & ~7


def synthetic_term_key(term: str) -> int:
    """Key of a synthetic term 't<id>' (synth.py) or FNV-1a of any other string; low 3 bits clear
    (reserved for the n-gram type in the reference, index.rs:4165-4225)."""
    from .synth import splitmix64
    if len(term) > 1 and term[0] == "t" and term[1:].isdigit():
        return splitmix64(int(term[1:])) & ~7
    return fnv1a64(term)


class LexicalSimilarity(enum.IntEnum):
    """index.rs:559-566 (the reference's default is Bm25fProximity).  The two score identically unless the index holds n-gram lists."""
    Bm25f = 0
    Bm25fProximity = 1


class NgramSet(enum.IntFlag):
    """index.rs:1834-1851: the n-gram types an index is built with (F = frequent term, R = rare term)"""
    SingleTerm = 0
    NgramFF = 1
    NgramFR = 2
    NgramRF = 4
    NgramFFF = 8
    NgramRFF = 16
    NgramFFR = 32
    NgramFRF = 64


class NgramType(enum.IntEnum):
    """index.rs:1854-1872: the low 3 bits of an n-gram key"""
    SingleTerm = 0
    NgramFF = 1
    NgramFR = 2
    NgramRF = 3
    NgramFFF = 4
    NgramRFF = 5
    NgramFFR = 6
    NgramFRF = 7


def ngram_key(words: Sequence[str], ngram_type: int, term_key_fn: Callable[[str], int] = synthetic_term_key) -> int:
    """hash64("a b" / "a b c") | NgramType (tokenizer.rs:678-685), with the index's term hash; a single word is its term key"""
    if int(ngram_type) == 0:
        return term_key_fn(words[0])
    return (term_key_fn(" ".join(words)) & ~7 & ((1 << 64) - 1)) | int(ngram_type)


def ngram_rewrite(terms: Sequence[str], frequent, ngram_set: int):
    """The query-time rewrite of a phrase (tokenizer.rs:898-1387): greedy, left to right, each position tries FFF, RFF, FFR, FRF, then
    FF, RF, FR under their own NgramSet bits, else keeps the single term.  -> [(words tuple, NgramType)]"""
    out, i, n = [], 0, len(terms)
    f = [t in frequent for t in terms]
    while i < n:
        if i + 2 < n:
            tri = ((NgramSet.NgramFFF, f[i] and f[i + 1] and f[i + 2], NgramType.NgramFFF),
                   (NgramSet.NgramRFF, (not f[i]) and f[i + 1] and f[i + 2], NgramType.NgramRFF),
                   (NgramSet.NgramFFR, f[i] and f[i + 1] and not f[i + 2], NgramType.NgramFFR),
                   (NgramSet.NgramFRF, f[i] and (not f[i + 1]) and f[i + 2], NgramType.NgramFRF))
            hit = next((ty for bit, ok, ty in tri if ngram_set & bit and ok), None)
            if hit is not None:
                out.append((tuple(terms[i:i + 3]), hit))
                i += 3
                continue
        if i + 1 < n:
            bi = ((NgramSet.NgramFF, f[i] and f[i + 1], NgramType.NgramFF),
                  (NgramSet.NgramRF, (not f[i]) and f[i + 1], NgramType.NgramRF),
                  (NgramSet.NgramFR, f[i] and not f[i + 1], NgramType.NgramFR))
            hit = next((ty for bit, ok, ty in bi if ngram_set & bit and ok), None)
            if hit is not None:
                out.append((tuple(terms[i:i + 2]), hit))
                i += 2
                continue
        out.append(((terms[i],), NgramType.SingleTerm))
        i += 1
    return out


def _morton_spread(v):
    x = v.astype(np.uint64)
    for sh, m in ((16, 0x0000FFFF0000FFFF), (8, 0x00FF00FF00FF00FF), (4, 0x0F0F0F0F0F0F0F0F), (2, 0x3333333333333333), (1, 0x5555555555555555)):
        x = (x | (x << np.uint64(sh))) & np.uint64(m)
    return x


def _rust_as_i32(v):
    """Rust `f64 as i32` on an array: truncation toward zero, saturating at the i32 limits, NaN -> 0"""
    v = np.asarray(v, dtype=np.float64)
    out = np.trunc(np.clip(np.where(np.isnan(v), 0.0, v), -2147483648.0, 2147483647.0))
    return out.astype(np.int64).astype(np.int32)


def encode_morton_2d(lat, lon):
    """encode_morton_2_d (geo_search.rs:27-42) on arrays: x = ((lat * 1e7) as i32) as u32 in the even bits, y = the same of lon in the odd
    bits -> uint64 codes"""
    x = _rust_as_i32(np.asarray(lat, dtype=np.float64) * 10000000.0).view(np.uint32)
    y = _rust_as_i32(np.asarray(lon, dtype=np.float64) * 10000000.0).view(np.uint32)
    return _morton_spread(x) | (_morton_spread(y) << np.uint64(1))


def decode_morton_2d(codes):
    """decode_morton_2_d (geo_search.rs:58-79) on an array of codes: (x_u32 as i32) as f64 / 1e7 of the even (lat) and odd (lon) bits"""
    def compact(c):
        x = c & np.uint64(0x5555555555555555)
        for sh, m in ((1, 0x3333333333333333), (2, 0x0F0F0F0F0F0F0F0F), (4, 0x00FF00FF00FF00FF), (8, 0x0000FFFF0000FFFF), (16, 0xFFFFFFFF)):
            x = (x ^ (x >> np.uint64(sh))) & np.uint64(m)
        return x.astype(np.uint32).view(np.int32).astype(np.float64) / 10000000.0
    c = np.asarray(codes, dtype=np.uint64)
    return compact(c), compact(c >> np.uint64(1))


def point_column(points):
    """a Point facet's column as the reference writes it (index.rs:5803-5819): [n, 2] (lat, lon) -> the Morton codes; a coordinate outside
    [-90, 90] x [-180, 180] (or NaN) is not written, its row stays 0"""
    p = np.asarray(points, dtype=np.float64).reshape(-1, 2)
    lat, lon = p[:, 0], p[:, 1]
    ok = (lat >= -90.0) & (lat <= 90.0) & (lon >= -180.0) & (lon <= 180.0)
    return np.where(ok, encode_morton_2d(np.where(ok, lat, 0.0), np.where(ok, lon, 0.0)), np.uint64(0)).astype(np.uint64)


def _addr(x):
    """Address of a numpy array / torch tensor (host or device) or None."""
    if x is None:
        return None
    if isinstance(x, np.ndarray):
        return x.ctypes.data
    return x.data_ptr()  # torch.Tensor


def _hits_array(n):
    return np.zeros(n, dtype=np.dtype([("doc_id", "<u8"), ("score", "<f4"), ("pad", "<u4")]))


def vector_field_mask(field_mask: int, n_lexical_fields: int) -> int:
    """The field filter of the vector search: the reference builds field_filter_set from the indexed lexical fields only
    (vector.rs:1228-1231), so bits past the lexical fields (or beyond the 32 a mask holds) name no field and are dropped; a mask left
    empty filters nothing."""
    return int(field_mask) & ((1 << min(max(int(n_lexical_fields), 0), 32)) - 1)


class Index:
    """One shard's GPU-resident mirror: committed lexical levels + vector levels on one H100."""

    def __init__(self, device: int = 0, vector_dims: int = 0,
                 vector_similarity: VectorSimilarity = VectorSimilarity.Cosine, max_batch: int = 4096,
                 term_key_fn: Callable[[str], int] = synthetic_term_key, vector_kernel: int = 0,
                 vector_quantization: int = 0):
        """vector_kernel: SSB_VEC_KERNEL_* (0 = auto, 1 = FP32 FFMA scan, 2/3 = wgmma 3xTF32, 4/5/6 = wgmma 3xBF16 with 128/64/256
        queries per pass, 7/8 = fp16 filter scan + exact f32 refine with 128/256 queries per pass, 9 = the 256-query filter scan on
        CTA pairs).  include/seekstorm_b200.h states what AUTO picks and when the filter scans fall back."""
        self._h = C.c_void_p()
        cfg = SsbConfig(device, max_batch, vector_dims, int(vector_similarity), vector_kernel, int(vector_quantization),
                        (C.c_uint32 * 2)(0, 0))
        check(lib().ssb_create(C.byref(cfg), C.byref(self._h)))
        self.vector_dims = vector_dims
        self.vector_similarity = VectorSimilarity(vector_similarity)
        self.term_key_fn = term_key_fn
        self.indexed_doc_count = 0
        self._keep = []
        self.vector_fields = False          # vector rows carry field ids (add_vector_level(field_ids=...), load_vector_bin(keep_fields=True))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().ssb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ load
    def set_field_boosts(self, boosts):
        """Several indexed fields (BM25F, add_result.rs:1171-1426): per-field boosts, before the first level.  Levels then carry
        tfs [n_postings, n_fields] (0 = term not in that field) and doc_len_bytes [n_fields, n_docs]."""
        b = np.ascontiguousarray(np.asarray(boosts, dtype=np.float32))
        check(lib().ssb_lexical_set_field_boosts(self._h, len(b), b.ctypes.data))
        self._n_fields = len(b)
        if len(getattr(self, "field_names", [])) != len(b):
            self.field_names = [f"field{f}" for f in range(len(b))]      # names of the indexed fields in schema order (Index.search field_filter)

    def set_ngram_config(self, frequent_terms=(), ngram_set: int = 0, similarity: LexicalSimilarity = LexicalSimilarity.Bm25fProximity,
                         df_rule: int = _lib.NGRAM_DF_FIRST_LEVEL):
        """An index built with n-gram lists (NGRAM_SEARCH.md), before the first level: the frequent-term set and NgramSet bits of the
        query rewrite, the LexicalSimilarity, and which level's key-head df bytes an n-gram list keeps (NGRAM_DF_FIRST_LEVEL: the
        reference's Ram access, NGRAM_DF_LAST_LEVEL: its Mmap access)."""
        check(lib().ssb_lexical_set_ngram_config(self._h, int(similarity), int(df_rule)))
        self.frequent_terms = frozenset(frequent_terms)
        self.ngram_set = int(ngram_set)
        self.lexical_similarity = LexicalSimilarity(similarity)

    def add_lexical_level(self, level_id: int, n_docs: int, term_keys, posting_offsets, doc_ids, tfs, doc_len_bytes, positions=None,
                          ngram_tfs=None, ngram_df_bytes=None):
        """One committed 64K-doc level in the neutral layout (arrays: numpy on host or torch on the device).  positions: u16 [sum of tfs], the
        term positions of every posting in posting order (phrase queries), or None.  With several indexed fields (tfs [n_postings, F]) a
        posting holds the sum of its F tfs positions, one run per field in field order (field 0's first), each run ascending and starting
        again from 0 in every field; a phrase matches inside one field only.
        ngram_tfs u16 [n_postings, 3] / ngram_df_bytes u8 [n_terms, 3]: the component tfs and key-head df bytes of the n-gram lists (keys
        with low bits set) of an index with n-gram lists (ssb_lexical_add_level_ngrams)."""
        if positions is not None:
            n_pos = positions.size if isinstance(positions, np.ndarray) else positions.numel()
            want = int(tfs.astype(np.int64).sum()) if isinstance(tfs, np.ndarray) else int((tfs.long() & 0xFFFF).sum())
            if n_pos != want:
                raise _lib.SsbError(f"add_lexical_level {level_id}: positions holds {n_pos} values, the postings' tfs add up to {want}")
        n_terms = int(term_keys.shape[0])
        d = SsbLevelDesc(level_id, n_docs, n_terms, getattr(self, "_n_fields", 1), _addr(term_keys), _addr(posting_offsets), _addr(doc_ids),
                         _addr(tfs), _addr(doc_len_bytes), _addr(positions))
        if ngram_tfs is not None or ngram_df_bytes is not None:
            ng = SsbLevelNgrams(_addr(ngram_tfs), _addr(ngram_df_bytes))
            check(lib().ssb_lexical_add_level_ngrams(self._h, C.byref(d), C.byref(ng)))
        else:
            check(lib().ssb_lexical_add_level(self._h, C.byref(d)))

    def add_synth_level(self, lv):
        """Convenience: a seekstorm_b200.synth.Level (tensors on CPU or on this index's device)."""
        if lv.term_keys.is_cuda:
            self.add_lexical_level(lv.level_id, lv.n_docs, lv.term_keys, lv.posting_offsets, lv.doc_ids, lv.tfs,
                                   lv.doc_len_bytes, getattr(lv, "positions", None))
        else:
            n = lv.to_numpy()
            self.add_lexical_level(n["level_id"], n["n_docs"], n["term_keys"], n["posting_offsets"], n["doc_ids"],
                                   n["tfs"], n["doc_len_bytes"], n.get("positions"))

    def load_index_bin(self, data, indexed_field_count: int = 1, key_head_size: int = 20, segment_number_bits: int = 11, decode_positions: bool = False,
                       ngrams: bool = False) -> int:
        """Load one shard's index.bin (bytes / mmap / numpy uint8 array, the reference's own format, index.rs:3253-3516) and commit.
        ngrams: also load its n-gram posting lists (22 / 23-byte key heads; ssb_load_index_bin_ngrams, set_ngram_config first).
        Returns indexed_doc_count."""
        from ._lib import SsbIndexBinParams
        buf = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data, dtype=np.uint8)
        prm = SsbIndexBinParams(indexed_field_count, key_head_size, segment_number_bits, 1 if decode_positions else 0)   # positions: phrase queries
        n = C.c_uint64(0)
        load = lib().ssb_load_index_bin_ngrams if ngrams else lib().ssb_load_index_bin
        check(load(self._h, buf.ctypes.data, buf.size, C.byref(prm), C.byref(n)))
        self.indexed_doc_count = n.value
        return n.value

    def load_vector_bin(self, data, keep_fields: bool = False) -> int:
        """Load one shard's vector.bin (vector.rs:1066-1094, f32 records).  Returns the number of vectors.  keep_fields: also keep every
        record's VectorHeader.field_id / chunk_id (ssb_load_vector_bin_fields): the vector search then applies field filters and
        reports each hit's best field / chunk."""
        buf = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data, dtype=np.uint8)
        n = C.c_uint64(0)
        load = lib().ssb_load_vector_bin_fields if keep_fields else lib().ssb_load_vector_bin
        check(load(self._h, buf.ctypes.data, buf.size, C.byref(n)))
        if keep_fields and n.value:
            self.vector_fields = True
        return n.value

    def commit(self, n_docs: int, len_sum_normalized: int):
        """Global statistics of the whole shard (commit.rs:318-319) + directory / block-max build."""
        check(lib().ssb_lexical_commit(self._h, n_docs, len_sum_normalized))
        self.indexed_doc_count = n_docs

    def dict_export(self):
        n = C.c_uint64(0)
        check(lib().ssb_lexical_dict_size(self._h, C.byref(n)))
        keys = np.zeros(n.value, dtype=np.uint64)
        dfs = np.zeros(n.value, dtype=np.uint32)
        check(lib().ssb_lexical_dict_export(self._h, keys.ctypes.data, dfs.ctypes.data, n.value))
        return keys, dfs

    def set_global_df(self, keys: np.ndarray, dfs: np.ndarray):
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        dfs = np.ascontiguousarray(dfs, dtype=np.uint32)
        check(lib().ssb_lexical_set_global_df(self._h, keys.ctypes.data, dfs.ctypes.data, len(keys)))

    # ------------------------------------------------------------------ sharded index (one process per GPU)
    def comm_unique_id(self) -> np.ndarray:
        """ncclGetUniqueId through the library (rank 0); ship the 128 bytes to the other ranks and call comm_init everywhere."""
        ident = np.zeros(128, dtype=np.uint8)
        check(lib().ssb_comm_unique_id(ident.ctypes.data))
        return ident

    def comm_init(self, ident: np.ndarray, rank: int, world: int):
        """Collective.  From here on every search_* call returns the GLOBAL result on every rank: the library all-gathers the
        per-shard top-k keys over NCCL and merges them (all-reduces the counts) on the search stream."""
        ident = np.ascontiguousarray(ident, dtype=np.uint8)
        assert ident.size == 128
        check(lib().ssb_comm_init(self._h, ident.ctypes.data, rank, world))

    def comm_destroy(self):
        check(lib().ssb_comm_destroy(self._h))

    def sync_df(self):
        """Collective: install the index-wide document frequencies (idf of the whole index on every shard)."""
        check(lib().ssb_lexical_sync_df(self._h))

    def set_deleted(self, doc_ids):
        """shard.delete_hashset: these docs are neither scored nor counted (lexical, vector, hybrid); [] clears the set."""
        a = np.ascontiguousarray(np.asarray(list(doc_ids), dtype=np.uint64))
        check(lib().ssb_set_deleted(self._h, a.ctypes.data if a.size else None, a.size))

    def set_facets(self, columns: dict, first_doc_id: int = 0, string_facets: Sequence[str] = (), timestamp_facets: Sequence[str] = (),
                   string_values: Optional[dict] = None, point_facets: Sequence[str] = (), string_set_facets: Sequence[str] = (),
                   string_set32_facets: Sequence[str] = ()):
        """The shard's facet file (`facets_file_mmap`, add_result.rs:343-347): one typed value per doc and facet field.  columns: name ->
        numpy array [n_docs] (dtype = the facet's FieldType; names in string_facets are String16 / String32 value ids, names in
        timestamp_facets Timestamp); rows are packed field after field like the reference's facet file and handed to ssb_set_facets.
        string_values: name -> the String facet's value strings by id (`facet.values`); sorting by that facet orders by the strings
        (result_ordering_shard, min_heap.rs:861-898), so their byte-wise order is sent along (ssb_set_facet_value_order).
        point_facets: names whose column is an [n_docs, 2] float64 array of (lat, lon): Point facets, stored as their Morton codes
        (point_column: invalid coordinates are stored as 0).
        string_set_facets / string_set32_facets: names whose column is a per-doc list of strings: StringSet16 / StringSet32 facets, ingested
        like the reference (string_set_facet) and sent with their member lists (ssb_set_facet_string_sets)."""
        from ._lib import SsbFacetField
        kinds = {"uint8": _lib.FACET_U8, "uint16": _lib.FACET_U16, "uint32": _lib.FACET_U32, "uint64": _lib.FACET_U64, "int8": _lib.FACET_I8,
                 "int16": _lib.FACET_I16, "int32": _lib.FACET_I32, "int64": _lib.FACET_I64, "float32": _lib.FACET_F32, "float64": _lib.FACET_F64}
        for name in (*point_facets, *string_set_facets, *string_set32_facets):
            if name not in columns:
                raise ValueError(f"point_facets / string_set_facets: {name!r} is not a column")
        sets = {name: string_set_facet(columns[name], 16 if name in string_set_facets else 32)
                for name in (*string_set_facets, *string_set32_facets)}
        columns = {name: (point_column(c) if name in point_facets else sets[name].ids if name in sets else c) for name, c in columns.items()}
        names = list(columns)
        n = len(next(iter(columns.values()))) if names else 0
        fields, off, self._facet_schema = (SsbFacetField * max(len(names), 1))(), 0, {}
        for i, name in enumerate(names):
            a = np.asarray(columns[name])
            t = kinds[a.dtype.name]
            if name in string_facets:
                t = {"uint16": _lib.FACET_STRING16, "uint32": _lib.FACET_STRING32}[a.dtype.name]
            if name in timestamp_facets:
                t = {"int64": _lib.FACET_TIMESTAMP}[a.dtype.name]
            if name in point_facets:
                t = _lib.FACET_POINT
            if name in sets:
                t = _lib.FACET_STRINGSET16 if name in string_set_facets else _lib.FACET_STRINGSET32
            fields[i] = SsbFacetField(t, off)
            self._facet_schema[name] = (i, t)
            off += a.dtype.itemsize
        rows = np.zeros((max(n, 1), max(off, 1)), dtype=np.uint8)
        for i, name in enumerate(names):
            a = np.ascontiguousarray(columns[name])
            rows[:n, fields[i].offset:fields[i].offset + a.dtype.itemsize] = a.view(np.uint8).reshape(n, a.dtype.itemsize)
        self._facet_rows = (rows, fields, int(first_doc_id), n, off)      # also what the tests hand to the oracle
        self._string_values, self._string_order = {}, {}
        check(lib().ssb_set_facets(self._h, rows.ctypes.data, int(first_doc_id), n, off, fields, len(names)))
        self._string_sets = sets
        for name, ss in sets.items():
            if n:
                check(lib().ssb_set_facet_string_sets(self._h, self._facet_schema[name][0], ss.offsets.ctypes.data, ss.member_ids.ctypes.data,
                                                      len(ss.combos), len(ss.members)))
            self._string_values[name] = [m.decode("utf-8") for m in ss.members]      # facet counts name member ids
            self._string_order[name] = ss.members                                   # prefixes are member-id intervals
        for name, values in (string_values or {}).items():
            t = self._facet_schema.get(name, (None, None))[1]
            if t not in (_lib.FACET_STRING16, _lib.FACET_STRING32):
                raise ValueError(f"string_values: {name!r} is not a String16 / String32 facet (facets: {list(self._facet_schema)})")
            enc = [str(v).encode("utf-8") for v in values]
            order = sorted(set(enc))                                        # Rust String order: byte-wise lexicographic
            pos = {b: i for i, b in enumerate(order)}
            rank = np.ascontiguousarray([pos[b] for b in enc], dtype=np.uint32)
            check(lib().ssb_set_facet_value_order(self._h, self._facet_schema[name][0], rank.ctypes.data, rank.size))
            self._string_values[name], self._string_order[name] = [str(v) for v in values], order

    def _sort_criteria(self, result_sort):
        """ResultSort list -> ssb_sort_criterion array (ResultSortIndex, search.rs:2497-2525): "_id" / "_score", facet names resolved to
        their index; unknown names are dropped like the reference does (facets_map.get, :2517).  A base is accepted on a Point facet
        only (the bases themselves travel separately, _sort_bases)."""
        from ._lib import SsbSortCriterion
        out = []
        for rs in result_sort:
            if rs.base is not None and getattr(self, "_facet_schema", {}).get(rs.field, (None, None))[1] != _lib.FACET_POINT:
                raise NotImplementedError("a ResultSort base (FacetValue::Point) is only read on a Point facet; other bases are not built")
            order = _lib.SORT_DESCENDING if SortOrder(rs.order) == SortOrder.Descending else _lib.SORT_ASCENDING
            if rs.field == "_id":
                out.append(SsbSortCriterion(_lib.SORT_ID, 0, order, 0))
            elif rs.field == "_score":
                out.append(SsbSortCriterion(_lib.SORT_SCORE, 0, order, 0))
            elif rs.field in getattr(self, "_facet_schema", {}):
                out.append(SsbSortCriterion(_lib.SORT_FACET, self._facet_schema[rs.field][0], order, 0))
        return (SsbSortCriterion * max(len(out), 1))(*out), len(out)

    def _sort_bases(self, result_sort, nq, sort_bases=None):
        """the bases array of ssb_search_lexical_sorted_ex: sort_bases ([nq] (lat, lon) per query) or else the base of the sort's Point
        criterion for every query; None when neither exists (a Point criterion is then dropped)"""
        if sort_bases is None:
            base = next((rs.base for rs in result_sort if rs.base is not None), None)
            if base is None:
                return None
            sort_bases = [base] * nq
        b = np.ascontiguousarray(np.asarray(sort_bases, dtype=np.float64).reshape(-1, 2))
        if len(b) != nq:
            raise ValueError(f"sort_bases: {len(b)} bases for {nq} queries")
        return b

    def _encode_filters(self, filters):
        """filters: per query a list of FacetFilter -> (filter_offsets, ssb_facet_filter array, set values)"""
        from ._lib import SsbFacetFilter
        offs = np.zeros(len(filters) + 1, dtype=np.uint32)
        flat, sets = [], []
        for i, fl in enumerate(filters):
            for f in fl or ():
                idx, t = self._facet_schema[f.field] if isinstance(f.field, str) else (int(f.field), None)
                if t is None:
                    t = next((v[1] for v in getattr(self, "_facet_schema", {}).values() if v[0] == idx), _lib.FACET_U64)
                if f.base is not None:                                        # FacetFilter::Point: (base, start..end, unit)
                    f64 = lambda x: int(np.float64(x).view(np.uint64))
                    flat.append(SsbFacetFilter(idx, _lib.FILTER_POINT, f64(f.start), f64(f.end), len(sets), 3))
                    sets.extend([f64(f.base[0]), f64(f.base[1]), int(DistanceUnit(f.unit))])
                elif f.values is not None and t in _SET_FACETS:            # strings -> member ids and flagged combination ids
                    ss = self._string_sets[next(n for n, v in self._facet_schema.items() if v[0] == idx)]
                    vals = ss.filter_values([v for v in f.values if isinstance(v, str)]) + [int(v) for v in f.values if not isinstance(v, str)]
                    flat.append(SsbFacetFilter(idx, _lib.FILTER_SET, 0, 0, len(sets), len(vals)))
                    sets.extend(vals)
                elif f.values is not None:
                    flat.append(SsbFacetFilter(idx, _lib.FILTER_SET, 0, 0, len(sets), len(f.values)))
                    sets.extend(int(v) for v in f.values)
                else:
                    if t in (_lib.FACET_F32, _lib.FACET_F64):
                        enc = lambda x: int(np.float64(x).view(np.uint64))
                    elif t in (_lib.FACET_I8, _lib.FACET_I16, _lib.FACET_I32, _lib.FACET_I64, _lib.FACET_TIMESTAMP):
                        enc = lambda x: int(np.int64(x).view(np.uint64))
                    else:
                        enc = lambda x: int(np.uint64(x))
                    flat.append(SsbFacetFilter(idx, _lib.FILTER_RANGE, enc(f.start), enc(f.end), 0, 0))
            offs[i + 1] = len(flat)
        arr = (SsbFacetFilter * max(len(flat), 1))(*flat)
        sv = np.asarray(sets if sets else [0], dtype=np.uint64)
        return offs, arr, sv

    def _facet_requests(self, query_facets):
        """QueryFacet list -> (ssb_facet_request array, kept buffers, [(field, kind, QueryFacet)] per request).  The reference keeps one
        request per facet field (the last one wins) and ignores requests whose shape does not fit the field's type (search.rs:2729-3012)."""
        from ._lib import SsbFacetRequest
        by_field = {}
        for qf in query_facets:
            idx, t = getattr(self, "_facet_schema", {}).get(qf.field, (None, None))
            if idx is None:
                continue
            string = t in _VALUE_FACETS
            if string == bool(qf.ranges):
                continue
            by_field[qf.field] = (idx, t, qf)
        reqs, keep, meta = [], [], []
        for name, (idx, t, qf) in by_field.items():
            if t in _VALUE_FACETS:
                lo = hi = has = 0
                if qf.prefix:
                    if name not in self._string_order:
                        raise ValueError(f"query facet {name!r}: a prefix needs the facet's string_values (set_facets)")
                    lo, hi = prefix_rank_interval(self._string_order[name], qf.prefix.encode("utf-8"))
                    has = 1
                reqs.append(SsbFacetRequest(idx, _lib.FACET_COUNT_VALUES, int(qf.length), has, lo, hi, 0, 0, None))
            else:
                starts = [r[1] for r in qf.ranges]
                if t in (_lib.FACET_F32, _lib.FACET_F64, _lib.FACET_POINT):
                    a = np.asarray(starts, dtype=np.float64).view(np.uint64)
                elif t in (_lib.FACET_I8, _lib.FACET_I16, _lib.FACET_I32, _lib.FACET_I64, _lib.FACET_TIMESTAMP):
                    a = np.asarray(starts, dtype=np.int64).view(np.uint64)
                else:
                    a = np.asarray(starts, dtype=np.uint64)
                a = np.ascontiguousarray(a)
                keep.append(a)
                reqs.append(SsbFacetRequest(idx, _lib.FACET_COUNT_RANGES, 0, 0, 0, 0, len(starts), int(DistanceUnit(qf.unit)), a.ctypes.data))
            meta.append((name, t, qf))
        arr = (SsbFacetRequest * max(len(reqs), 1))(*reqs)
        return arr, len(reqs), keep, meta

    def search_lexical_facets(self, queries_keys, query_type: QueryType, query_facets, not_keys=None, filters=None, field_masks=None,
                              facet_bases=None):
        """Facet counts of a lexical batch (ssb_search_lexical_facets): the docs result_count_total counts for the same arguments, per query
        {field: raw} with raw = [(value id, count), ...] (String facets: count desc, id asc, at most `length`) or the counts of every range
        (zeros included).  facet_bases: per query the (lat, lon) base of each Point request in request order (default: QueryFacet.base)."""
        nq = len(queries_keys)
        b, keep = self._lex_batch(queries_keys, query_type, not_keys, filters, field_masks)
        arr, n_req, keep2, meta = self._facet_requests(query_facets)
        if n_req == 0 or nq == 0:
            return [{} for _ in range(nq)]
        points = [qf for _, t, qf in meta if t == _lib.FACET_POINT]
        bases = None
        if points:
            if facet_bases is None:
                facet_bases = [[qf.base for qf in points]] * nq
            bases = np.ascontiguousarray(np.asarray(facet_bases, dtype=np.float64).reshape(nq, len(points), 2))
        caps = [qf.length if t in _VALUE_FACETS else len(qf.ranges) for _, t, qf in meta]
        stride = sum(caps)
        out = np.zeros(max(nq * stride, 1), dtype=[("value", np.uint32), ("pad", np.uint32), ("count", np.uint64)])
        n_out = np.zeros(max(nq * n_req, 1), dtype=np.uint32)
        check(lib().ssb_search_lexical_facets(self._h, C.byref(b), C.addressof(arr), n_req, bases.ctypes.data if bases is not None else None,
                                              out.ctypes.data, n_out.ctypes.data))
        res = []
        for i in range(nq):
            d, o = {}, i * stride
            for r, (name, t, qf) in enumerate(meta):
                m = int(n_out[i * n_req + r])
                e = out[o:o + m]
                d[name] = ([(int(v), int(c)) for v, c in zip(e["value"], e["count"])] if t in _VALUE_FACETS
                           else [int(c) for c in e["count"]])
                o += caps[r]
            res.append(d)
        return res

    def assemble_facets(self, raw, query_facets):
        """One query's raw counts (search_lexical_facets) -> ResultObject.facets: per field the shard's assembly (search.rs:3598-3750: the
        strings of the counted ids; for ranges RangeType, labels, the label prefix, no zero bins), then Search::search's ordering by count
        and truncation to `length` (search.rs:2038-2048).  A field whose list comes out empty is left out."""
        per_field, lengths = {}, {}
        reqs = {qf.field: qf for qf in query_facets if qf.field in raw}
        for name, qf in reqs.items():
            t = self._facet_schema[name][1]
            if t in _VALUE_FACETS:
                sv = getattr(self, "_string_values", {}).get(name)
                v = [(sv[i] if sv is not None else i, c) for i, c in raw[name]]
                lengths[name] = int(qf.length)
            else:
                v = assemble_range_facet(raw[name], [r[0] for r in qf.ranges], qf.range_type, qf.prefix)
                lengths[name] = 65535
            if v:
                per_field[name] = v
        return merge_facets(per_field, lengths)

    def add_vector_level(self, level_id: int, rows, local_ids=None, cluster_counts=None, field_ids=None, chunk_ids=None):
        """rows: [n, dims] f32 (numpy or torch, host or device), n <= 65536.  cluster_counts: the level's IVF cluster table (rows in
        cluster order, medoid = first row of each cluster; vector.rs:1066-1094) or None = one cluster.  field_ids (u8, < 32) / chunk_ids
        (u32): each row's indexed field and chunk (multi-vector documents, ssb_vector_add_level_fields) — every level of an index carries
        them or none does."""
        n, dims = int(rows.shape[0]), int(rows.shape[1])
        stride = rows.strides[0] // 4 if isinstance(rows, np.ndarray) else rows.stride(0)
        if field_ids is not None or chunk_ids is not None:
            if field_ids is None or chunk_ids is None:
                raise ValueError("field_ids and chunk_ids go together")
            fi = np.ascontiguousarray(field_ids, dtype=np.uint8)
            ci = np.ascontiguousarray(chunk_ids, dtype=np.uint32)
            if fi.size != n or ci.size != n:
                raise ValueError("field_ids / chunk_ids need one entry per row")
            cc = None if cluster_counts is None else np.ascontiguousarray(cluster_counts, dtype=np.uint32)
            check(lib().ssb_vector_add_level_fields(self._h, level_id, _addr(rows), stride, _addr(local_ids), n, dims,
                                                    None if cc is None else cc.ctypes.data, 0 if cc is None else len(cc),
                                                    fi.ctypes.data, ci.ctypes.data))
            if n:
                self.vector_fields = True
        elif cluster_counts is None:
            check(lib().ssb_vector_add_level(self._h, level_id, _addr(rows), stride, _addr(local_ids), n, dims))
        else:
            cc = np.ascontiguousarray(cluster_counts, dtype=np.uint32)
            check(lib().ssb_vector_add_level_clustered(self._h, level_id, _addr(rows), stride, _addr(local_ids), n, dims, cc.ctypes.data, len(cc)))

    def set_turboquant_mask(self, seed_mask):
        """TurboQuantI8 indexes (vector_quantization = 2): the index's +-1 sign mask (TurboQuant.seed_mask, next_power_of_two(dims) values)"""
        m = np.ascontiguousarray(seed_mask, dtype=np.float32)
        check(lib().ssb_vector_set_turboquant_mask(self._h, m.ctypes.data, m.size))

    def reserve_vectors(self, n_rows: int):
        """Capacity hint (ssb_vector_reserve): one allocation for n_rows rows instead of geometric growth while loading."""
        check(lib().ssb_vector_reserve(self._h, int(n_rows)))

    def add_vectors(self, rows, first_level: int = 0):
        """Split a big [N, dims] matrix into 64K-row levels (doc_id = row index when first_level = 0)."""
        n = int(rows.shape[0])
        self.reserve_vectors(self.vector_count + n)
        for s in range(0, n, 65536):
            self.add_vector_level(first_level + s // 65536, rows[s:min(n, s + 65536)])

    def set_vector_kernel(self, kernel: int):
        """SSB_VEC_KERNEL_*, as `vector_kernel` of the constructor."""
        check(lib().ssb_set_vector_kernel(self._h, kernel))

    @property
    def vector_count(self) -> int:
        n = C.c_uint64(0)
        check(lib().ssb_vector_count(self._h, C.byref(n)))
        return n.value

    # ------------------------------------------------------------------ batched shard-level search
    def _lex_batch(self, queries_keys: Sequence[Sequence[int]], query_type: QueryType, not_keys: Optional[Sequence[Sequence[int]]] = None,
                   filters: Optional[Sequence[Sequence["FacetFilter"]]] = None, field_masks: Optional[Sequence[int]] = None):
        """not_keys: per query the keys of its '-' terms (not_query_list, add_result.rs:3440-3496) or None.
        filters: per query its FacetFilter list (facet_filter of search_lexical_shard) or None."""
        nots = not_keys if not_keys is not None else [[] for _ in queries_keys]
        offs = np.zeros(len(queries_keys) + 1, dtype=np.uint32)
        for i, q in enumerate(queries_keys):
            if len(q) > _lib.MAX_QUERY_TERMS:
                raise _lib.SsbError(f"query {i} has {len(q)} terms (> {_lib.MAX_QUERY_TERMS})")
            offs[i + 1] = offs[i] + len(q) + len(nots[i])
        keys = np.zeros(max(int(offs[-1]), 1), dtype=np.uint64)
        flags = np.zeros(max(int(offs[-1]), 1), dtype=np.uint8)
        p = 0
        for q, nq_ in zip(queries_keys, nots):
            for t in q:
                keys[p] = t
                p += 1
            for t in nq_:
                keys[p] = t
                flags[p] = 1
                p += 1
        b = SsbLexBatch(len(queries_keys), int(query_type), offs.ctypes.data, keys.ctypes.data,
                        flags.ctypes.data if not_keys is not None else None, None, None, None, None)
        keep = [offs, keys, flags]
        if filters is not None:
            foffs, farr, fsets = self._encode_filters(filters)
            b.filter_offsets, b.filters, b.filter_set_values = foffs.ctypes.data, C.addressof(farr), fsets.ctypes.data
            keep += [foffs, farr, fsets]
        if field_masks is not None:       # field_filter: per query a bitmask of indexed fields (0 = none)
            fm = np.ascontiguousarray(np.asarray(list(field_masks), dtype=np.uint32))
            b.field_masks = fm.ctypes.data
            keep.append(fm)
        return b, tuple(keep)

    def search_lexical_batch(self, queries_keys, query_type: QueryType, k: int,
                             result_type: ResultType = ResultType.TopkCount, not_keys=None, filters=None, field_masks=None, sort=None,
                             sort_bases=None):
        """Batched search_lexical_shard.  Returns (list of [(doc_id, score)...], counts ndarray).  not_keys: '-' terms per query;
        filters: FacetFilter list per query (needs set_facets); sort: ResultSort list for the whole batch (ssb_search_lexical_sorted_ex);
        sort_bases: per query the (lat, lon) base of the sort's Point criterion (default: that criterion's ResultSort.base)."""
        nq = len(queries_keys)
        b, keep = self._lex_batch(queries_keys, query_type, not_keys, filters, field_masks)
        hits = _hits_array(max(nq * max(k, 1), 1))
        n_hits = np.zeros(max(nq, 1), dtype=np.uint32)
        counts = np.zeros(max(nq, 1), dtype=np.uint64)
        if sort is not None:
            crit, n_crit = self._sort_criteria(sort)
            bases = self._sort_bases(sort, nq, sort_bases)
            check(lib().ssb_search_lexical_sorted_ex(self._h, C.byref(b), C.addressof(crit), n_crit, bases.ctypes.data if bases is not None else None,
                                                     k, int(result_type), hits.ctypes.data, n_hits.ctypes.data, counts.ctypes.data))
        else:
            check(lib().ssb_search_lexical(self._h, C.byref(b), k, int(result_type), hits.ctypes.data, n_hits.ctypes.data,
                                           counts.ctypes.data))
        out = []
        for i in range(nq):
            h = hits[i * k: i * k + int(n_hits[i])]
            out.append([(int(d), float(s)) for d, s in zip(h["doc_id"], h["score"])])
        return out, counts[:nq]

    def search_empty_batch(self, n_queries: int, k: int, result_type: ResultType = ResultType.TopkCount, filters=None, sort=None,
                           sort_bases=None):
        """The empty query for a batch of n_queries filter-only queries (ssb_search_empty): every live doc of the lexical levels through
        each query's FacetFilter list (filters: per query a list, or None), in the order of the ResultSort list `sort` (a leading "_score"
        orders by doc id; ties and no sort: doc id descending).  Returns (list of [(doc_id, 0.0)...], counts ndarray)."""
        nq = int(n_queries)
        b, keep = self._lex_batch([[] for _ in range(nq)], QueryType.Union, None, filters)
        b.term_offsets = None
        hits = _hits_array(max(nq * max(k, 1), 1))
        n_hits = np.zeros(max(nq, 1), dtype=np.uint32)
        counts = np.zeros(max(nq, 1), dtype=np.uint64)
        crit, n_crit = self._sort_criteria(sort or [])
        bases = self._sort_bases(sort or [], nq, sort_bases)
        check(lib().ssb_search_empty(self._h, C.byref(b), C.addressof(crit), n_crit, bases.ctypes.data if bases is not None else None,
                                     k, int(result_type), hits.ctypes.data, n_hits.ctypes.data, counts.ctypes.data))
        out = []
        for i in range(nq):
            h = hits[i * k: i * k + int(n_hits[i])]
            out.append([(int(d), float(s)) for d, s in zip(h["doc_id"], h["score"])])
        return out, counts[:nq]

    def search_empty_facets(self, query_facets):
        """Facet counts of the empty query (ssb_search_empty_facets, get_index_string_facets_shard index.rs:4441-4569): per String facet
        of query_facets [(value id, count), ...] over every facet row, count desc, id asc, at most `length`, prefix applied before the
        cut.  Range facets are left out."""
        arr, n_req, keep, meta = self._facet_requests(query_facets)
        if n_req == 0:
            return {}
        caps = [qf.length if t in _VALUE_FACETS else len(qf.ranges) for _, t, qf in meta]
        out = np.zeros(max(sum(caps), 1), dtype=[("value", np.uint32), ("pad", np.uint32), ("count", np.uint64)])
        n_out = np.zeros(n_req, dtype=np.uint32)
        check(lib().ssb_search_empty_facets(self._h, C.addressof(arr), n_req, out.ctypes.data, n_out.ctypes.data))
        res, o = {}, 0
        for r, (name, t, qf) in enumerate(meta):
            if t in _VALUE_FACETS:
                e = out[o:o + int(n_out[r])]
                res[name] = [(int(v), int(c)) for v, c in zip(e["value"], e["count"])]
            o += caps[r]
        return res

    def _search_empty(self, offset, length, result_type, query_facets, facet_filter, result_sort) -> ResultObject:
        """Search::search("", enable_empty_query = true, ..) on one shard.  Without facet filter and query_facets and with at most one
        "_id" / "_score" criterion, the index route (search.rs:1413-1432, search_iterator_index iterator.rs:360-413): the live doc ids from
        the largest (ascending when that criterion is Ascending), result_count_total = the live docs for every result type.  Otherwise the
        shard route (search_iterator_shard, iterator.rs:316-358): every doc through the facet filters and the sort, counted under Count /
        TopkCount (Topk counts nothing: total 0), and the index-wide String facet counts (search.rs:3598-3602) for every result type."""
        ro = ResultObject()
        rt = ResultType(result_type)
        index_route = not query_facets and not facet_filter and (not result_sort or (len(result_sort) == 1 and result_sort[0].field in ("_id", "_score")))
        if index_route:
            _, counts = self.search_empty_batch(1, 0, ResultType.Count)
            ro.result_count_total = int(counts[0])
            if rt != ResultType.Count and length > 0:
                asc = bool(result_sort) and SortOrder(result_sort[0].order) == SortOrder.Ascending
                res, _ = self.search_empty_batch(1, offset + length, ResultType.Topk, sort=[ResultSort("_id", SortOrder.Ascending)] if asc else None)
                ro.results = [Result(d, s) for d, s in res[0][offset:offset + length]]
        else:
            if length == 0 and rt != ResultType.Count:           # search.rs:2472-2478
                if rt == ResultType.Topk:
                    return ro
                rt = ResultType.Count
            heap = offset + length
            res, counts = self.search_empty_batch(1, heap if rt != ResultType.Count else 0, rt, [list(facet_filter)] if facet_filter else None,
                                                  list(result_sort) if result_sort and rt != ResultType.Count else None)
            ro.result_count_total = int(counts[0]) if rt != ResultType.Topk else 0
            ro.results = [Result(d, s) for d, s in res[0][offset:offset + length]]
            if query_facets:
                ro.facets = self.assemble_facets(self.search_empty_facets(list(query_facets)), list(query_facets))
        ro.result_count = len(ro.results)
        return ro

    def search_vector_batch(self, queries, k: int):
        """Batched search_vector_shard (AnnMode::All).  queries: [nq, dims] f32 numpy/torch."""
        nq = int(queries.shape[0])
        if isinstance(queries, np.ndarray):
            queries = np.ascontiguousarray(queries, dtype=np.float32)
        hits = _hits_array(max(nq * k, 1))
        n_hits = np.zeros(max(nq, 1), dtype=np.uint32)
        check(lib().ssb_search_vector(self._h, _addr(queries), nq, k, hits.ctypes.data, n_hits.ctypes.data))
        out = []
        for i in range(nq):
            h = hits[i * k: i * k + int(n_hits[i])]
            out.append([(int(d), float(s)) for d, s in zip(h["doc_id"], h["score"])])
        return out

    # ---- raw C-ABI calls with caller-owned numpy buffers (no per-hit Python objects; what a Rust shim would do) ----
    def make_lex_batch(self, queries_keys, query_type: QueryType):
        """Build the host-side ssb_lex_batch once; returns (struct, keepalive)."""
        return self._lex_batch(queries_keys, query_type)

    def search_lexical_raw(self, batch_struct, k: int, result_type: ResultType, hits, n_hits, counts):
        """ssb_search_lexical with preallocated outputs: hits = structured array [nq*k] (doc_id u8, score f4, pad u4)."""
        check(lib().ssb_search_lexical(self._h, C.byref(batch_struct), k, int(result_type), hits.ctypes.data,
                                       n_hits.ctypes.data, counts.ctypes.data if counts is not None else None))

    def search_vector_raw(self, queries, k: int, hits, n_hits):
        """ssb_search_vector with preallocated outputs; queries: host or device [nq, dims] f32."""
        check(lib().ssb_search_vector(self._h, _addr(queries), int(queries.shape[0]), k, hits.ctypes.data, n_hits.ctypes.data))

    @staticmethod
    def hits_buffer(n):
        return _hits_array(n)

    def search_vector_ex(self, queries, k: int, similarity_threshold=None, int8_queries: bool = False, ann_mode: int = 0, n_probe: int = 0,
                         cluster_threshold: float = 0.0, field_masks=None):
        """ssb_search_vector_ex: threshold (vector.rs:388-399), int8 query codes, vb result fields, observed_vector_count.
        field_masks: per query a bitmask of indexed fields (0 = no filter; ssb_search_vector_fields) — needs field-tagged rows.
        Returns (hits per query, ext structured array [nq, k], observed [nq]); on a field-tagged index ext carries each hit's best
        field_id / chunk_id."""
        from ._lib import SsbHitExt, SsbVecQuery
        nq = int(queries.shape[0])
        if isinstance(queries, np.ndarray):
            queries = np.ascontiguousarray(queries, dtype=np.int8 if int8_queries else np.float32)
        hits = _hits_array(max(nq * k, 1))
        n_hits = np.zeros(max(nq, 1), dtype=np.uint32)
        ext = (SsbHitExt * max(nq * k, 1))()
        observed = np.zeros(max(nq, 1), dtype=np.uint64)
        vq = SsbVecQuery(_addr(queries), nq, k, 1 if int8_queries else 0, 0 if similarity_threshold is None else 1,
                         0.0 if similarity_threshold is None else float(similarity_threshold), int(ann_mode), int(n_probe), float(cluster_threshold))
        if field_masks is None:
            check(lib().ssb_search_vector_ex(self._h, C.byref(vq), hits.ctypes.data, n_hits.ctypes.data, C.addressof(ext), observed.ctypes.data))
        else:
            fm = np.ascontiguousarray(np.asarray(list(field_masks), dtype=np.uint32))
            if fm.size != nq:
                raise ValueError("field_masks needs one mask per query")
            check(lib().ssb_search_vector_fields(self._h, C.byref(vq), fm.ctypes.data, hits.ctypes.data, n_hits.ctypes.data, C.addressof(ext),
                                                 observed.ctypes.data))
        out = []
        for i in range(nq):
            h = hits[i * k: i * k + int(n_hits[i])]
            out.append([(int(d), float(s)) for d, s in zip(h["doc_id"], h["score"])])
        return out, ext, observed[:nq]

    def search_hybrid_batch(self, queries_keys, query_type: QueryType, queries, k: int, field_masks=None):
        """ssb_search_hybrid.  field_masks: per query a bitmask of indexed fields (0 = none) — the lexical half's field filter, and the
        vector half's too when the vector rows carry field ids."""
        nq = len(queries_keys)
        b, keep = self._lex_batch(queries_keys, query_type, field_masks=field_masks)
        if isinstance(queries, np.ndarray):
            queries = np.ascontiguousarray(queries, dtype=np.float32)
        hits = _hits_array(max(nq * k, 1))
        n_hits = np.zeros(max(nq, 1), dtype=np.uint32)
        check(lib().ssb_search_hybrid(self._h, C.byref(b), _addr(queries), k, hits.ctypes.data, n_hits.ctypes.data))
        out = []
        for i in range(nq):
            h = hits[i * k: i * k + int(n_hits[i])]
            out.append([(int(d), float(s)) for d, s in zip(h["doc_id"], h["score"])])
        return out

    def last_stats(self) -> dict:
        s = SsbStats()
        check(lib().ssb_last_stats(self._h, C.byref(s)))
        return dict(kernel_launches=s.kernel_launches, algorithmic_bytes=s.algorithmic_bytes, h2d_bytes=s.h2d_bytes,
                    d2h_bytes=s.d2h_bytes, postings_visited=s.postings_visited, probes=s.probes,
                    items_processed=s.items_processed, items_skipped=s.items_skipped,
                    dominant_kernel_ns=s.dominant_kernel_ns, scan_bytes_read=s.scan_bytes_read,
                    filter_fallbacks=s.filter_fallbacks)

    # ------------------------------------------------------------------ device-resident API (bench / multi-GPU)
    def search_vector_keys(self, queries_dev, k: int, keys_out_dev):
        check(lib().ssb_search_vector_keys(self._h, _addr(queries_dev), int(queries_dev.shape[0]), k, _addr(keys_out_dev)))

    def search_lexical_keys(self, batch_struct, k: int, result_type: ResultType, keys_out_dev, counts_dev=None):
        check(lib().ssb_search_lexical_keys(self._h, C.byref(batch_struct), k, int(result_type), _addr(keys_out_dev),
                                            _addr(counts_dev)))

    def merge_keys(self, keys_dev, n_lists: int, nq: int, k: int):
        hits = _hits_array(max(nq * k, 1))
        n_hits = np.zeros(max(nq, 1), dtype=np.uint32)
        check(lib().ssb_merge_keys(self._h, _addr(keys_dev), n_lists, nq, k, hits.ctypes.data, n_hits.ctypes.data))
        return [[(int(d), float(s)) for d, s in zip(hits[i * k: i * k + int(n_hits[i])]["doc_id"],
                                                     hits[i * k: i * k + int(n_hits[i])]["score"])] for i in range(nq)]

    def merge_keys_raw(self, keys_dev, n_lists: int, nq: int, k: int, hits, n_hits):
        """ssb_merge_keys into caller-owned numpy buffers (no per-hit Python objects)."""
        check(lib().ssb_merge_keys(self._h, _addr(keys_dev), n_lists, nq, k, hits.ctypes.data, n_hits.ctypes.data))

    def sync(self):
        check(lib().ssb_sync(self._h))

    @property
    def stream(self) -> int:
        return lib().ssb_stream(self._h) or 0

    def set_stream(self, cuda_stream):
        """Run on a caller-owned CUDA stream handle (e.g. torch.cuda.current_stream().cuda_stream; 0 = the CUDA legacy
        default stream); None restores the index's own stream."""
        check(lib().ssb_set_stream(self._h, C.c_void_p(-1 if cuda_stream is None else cuda_stream)))

    # ------------------------------------------------------------------ the reference's public call
    def search(self, query_string: str, query_vector=None, query_type_default: QueryType = QueryType.Union,
               search_mode: SearchMode = None, enable_empty_query: bool = False, offset: int = 0, length: int = 10,
               result_type: ResultType = ResultType.TopkCount, include_uncommitted: bool = False,
               field_filter: Sequence[str] = (), query_facets: Sequence = (), facet_filter: Sequence = (),
               result_sort: Sequence = (), query_rewriting=None) -> ResultObject:
        """`Search::search` (search.rs:1134-1150) for committed data, 1-shard semantics.

        facet_filter: FacetFilter objects (range / value-set / geo distance filters on the facet fields given to set_facets) — applied to
        the lexical search like the reference does (the vector search takes no facet filter, vector.rs:1105-1115).
        result_sort: ResultSort objects — lexical search only (the hits in sort order, ssb_search_lexical_sorted_ex; a Point facet's
        ResultSort.base sorts by the distance to it).
        query_facets: QueryFacet objects — facet counts of the lexical matches in ResultObject.facets (ssb_search_lexical_facets), unless
        the result type is Topk (search.rs:1748).
        enable_empty_query with query_string "" and no query_vector (Lexical mode): every live doc through facet_filter, result_sort and
        the paging, the index-wide String facet counts in `facets` (_search_empty).
        field_filter: names (or indices) of indexed lexical fields (field_names).  It filters the lexical search, and the vector search
        when the vector rows carry field ids (add_vector_level(field_ids=...), load_vector_bin(keep_fields=True)): a row counts only if its
        field is in the filter, as the reference builds the filter from the lexical fields alone (vector.rs:1228-1231).  A filter that names
        no indexed field — an index past the lexical fields, or no lexical fields at all — filters no vector row (vector_field_mask); on a
        vector index without field ids the vector search is unfiltered.
        Unsupported reference features (facet counts of vector-only queries or of an empty query without enable_empty_query, sorting
        vector / hybrid results, a base on a non-Point facet, uncommitted, rewriting) raise NotImplementedError rather than being silently
        ignored."""
        if include_uncommitted:
            raise NotImplementedError("uncommitted search is outside the GPU hot path")
        search_mode = search_mode or SearchMode.Lexical()
        if query_facets and search_mode.kind == "Vector":
            raise NotImplementedError("facet counts of a vector search are not built")
        if any(not isinstance(qf, QueryFacet) for qf in query_facets):
            raise NotImplementedError("query_facets takes QueryFacet requests; other forms (bare field names) are not built")
        if result_sort and search_mode.kind != "Lexical":
            raise NotImplementedError("result_sort on vector / hybrid search is not built")
        if result_sort:
            self._sort_criteria(result_sort)                     # a base on a non-Point facet raises before any search runs
        if enable_empty_query and query_string == "" and query_vector is None and search_mode.kind == "Lexical":
            return self._search_empty(offset, length, result_type, query_facets, facet_filter, result_sort)
        # field_filter: names of indexed fields (self.field_names, in schema order) or their indices -> one bitmask
        fmask = 0
        for f in field_filter:
            names = getattr(self, "field_names", [])
            if isinstance(f, str) and f not in names:
                raise ValueError(f"field_filter: unknown indexed field {f!r} (indexed fields: {names})")
            fmask |= 1 << (names.index(f) if isinstance(f, str) else int(f))
        ro = ResultObject(original_query=query_string, query=query_string)
        heap = offset + length                       # search.rs:1708 per-shard length = offset+length
        # tokenizer stand-in: whitespace, '+' = mandatory (tokenizer.rs:546-563); unique terms (search.rs:3023-3039)
        toks = query_string.split()
        phrase = query_type_default == QueryType.Phrase
        if len(query_string) >= 2 and query_string.startswith('"') and query_string.endswith('"'):     # "..." = a phrase (tokenizer.rs:546-563)
            phrase, toks = True, query_string[1:-1].split()
        elif any(t.startswith('"') for t in toks):
            raise NotImplementedError("a phrase mixed with other terms is outside the GPU hot path")
        not_terms = [t[1:] for t in toks if t.startswith("-") and len(t) > 1]          # '-' operator: not_query_list (tokenizer.rs:546-563)
        toks = [t for t in toks if not t.startswith("-")]
        qt = query_type_default
        if toks and all(t.startswith("+") for t in toks):
            qt = QueryType.Intersection
        terms = []
        for t in toks:
            t = t.lstrip("+")
            if t and (phrase or t not in terms):       # a phrase keeps its repeated terms: their order is the query
                terms.append(t)
        if phrase and len(terms) >= 2:
            qt = QueryType.Phrase
            if not_terms:
                raise NotImplementedError("NOT terms next to a phrase are outside the GPU hot path")
        elif phrase:
            qt = QueryType.Intersection
        ro.query_terms = list(dict.fromkeys(terms))    # the component terms, also of a phrase rewritten to n-grams (search.rs:3333-3357)
        if qt == QueryType.Phrase and getattr(self, "ngram_set", 0):
            keys = [ngram_key(w, ty, self.term_key_fn) for w, ty in ngram_rewrite(terms, self.frequent_terms, self.ngram_set)]
        else:
            keys = [self.term_key_fn(t) for t in terms]
        nkeys = [self.term_key_fn(t) for t in dict.fromkeys(not_terms)]
        lex, vec, total = [], [], 0
        want_lex = search_mode.kind in ("Lexical", "Hybrid") and len(keys) > 0
        want_vec = search_mode.kind in ("Vector", "Hybrid") and query_vector is not None
        rt = ResultType(result_type)
        if length == 0 and rt == ResultType.TopkCount:   # search.rs:2472-2478
            rt = ResultType.Count
        if want_lex:
            res, counts = self.search_lexical_batch([keys], qt, heap if rt != ResultType.Count else 0, rt, [nkeys] if nkeys else None,
                                                    [list(facet_filter)] if facet_filter else None, [fmask] if fmask else None,
                                                    list(result_sort) if result_sort else None)
            lex, total = res[0], int(counts[0])
            if query_facets and rt != ResultType.Topk:
                raw = self.search_lexical_facets([keys], qt, list(query_facets), [nkeys] if nkeys else None,
                                                 [list(facet_filter)] if facet_filter else None, [fmask] if fmask else None)
                ro.facets = self.assemble_facets(raw[0], list(query_facets))
        elif query_facets and rt != ResultType.Topk and search_mode.kind != "Vector":
            raise NotImplementedError("facet counts of the empty query (get_index_string_facets_shard) are not built")
        if want_vec:
            qv = np.asarray(query_vector, dtype=np.float32).reshape(1, -1)
            # similarity_threshold (TopK::new, vector.rs:388-399) and observed_vector_count are handled behind the C-ABI
            am = search_mode.ann_mode or AnnMode.All
            # field_filter on the vector rows (vector.rs:1226-1238): only on an index whose rows carry field ids
            vm = vector_field_mask(fmask, len(getattr(self, "field_names", [])))
            vmask = [vm] if vm and self.vector_fields else None
            res, _, observed = self.search_vector_ex(qv, max(heap, 1), search_mode.similarity_threshold, ann_mode=am.kind, n_probe=am.n_probe,
                                                     cluster_threshold=am.threshold, field_masks=vmask)
            vec = res[0][:heap]
            ro.observed_vector_count = int(observed[0])
        if search_mode.kind == "Lexical":
            fused = lex
            ro.result_count_total = total
        elif search_mode.kind == "Vector":
            fused = vec
            ro.result_count_total = len(vec)       # vector.rs:1509 (scan-order dependent in the reference)
        else:
            a = _hits_array(max(len(lex), 1)); b = _hits_array(max(len(vec), 1)); o = _hits_array(len(lex) + len(vec) + 1)
            for i, (d, s) in enumerate(lex):
                a[i] = (d, s, 0)
            for i, (d, s) in enumerate(vec):
                b[i] = (d, s, 0)
            n = C.c_uint32(0)
            check(lib().ssb_rrf_fuse(a.ctypes.data, len(lex), b.ctypes.data, len(vec), o.ctypes.data, C.byref(n)))
            fused = [(int(o[i]["doc_id"]), float(o[i]["score"])) for i in range(n.value)]
            ro.result_count_total = total
        # search.rs:2108-2121: drop offset, truncate length
        fused = fused[offset:offset + length] if offset < len(fused) else []
        ro.results = [Result(d, s) for d, s in fused]
        ro.result_count = len(ro.results)
        return ro
