"""ctypes loader for libseekstorm_b200.so (the C-ABI in include/seekstorm_b200.h).

There is NO CPU fallback: if the shared library is missing or no H100 is visible, calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# SSB_LIB: A/B experiments with an alternative in-tree build of the same sources (e.g. a compile-time switch); never a fallback
LIB_PATH = os.environ.get("SSB_LIB") or os.path.join(_HERE, "libseekstorm_b200.so")

SSB_OK = 0
K_MAX = 32
MAX_QUERY_TERMS = 32

QUERY_UNION, QUERY_INTERSECTION, QUERY_PHRASE = 0, 1, 2
RESULT_COUNT, RESULT_TOPK, RESULT_TOPKCOUNT = 0, 1, 2
SIM_DOT, SIM_COSINE, SIM_EUCLIDEAN = 0, 1, 2


class SsbHit(C.Structure):
    _fields_ = [("doc_id", C.c_uint64), ("score", C.c_float), ("pad", C.c_uint32)]


class SsbConfig(C.Structure):
    _fields_ = [("device", C.c_int32), ("max_batch", C.c_uint32), ("vector_dims", C.c_uint32),
                ("vector_similarity", C.c_uint32), ("vector_kernel", C.c_uint32), ("vector_quantization", C.c_uint32),
                ("reserved", C.c_uint32 * 2)]


class SsbHitExt(C.Structure):
    _fields_ = [("field_id", C.c_uint32), ("chunk_id", C.c_uint32), ("level_id", C.c_uint32), ("shard_id", C.c_uint32),
                ("cluster_id", C.c_uint32), ("cluster_score", C.c_float), ("vector_score", C.c_float),
                ("lexical_score", C.c_float), ("source", C.c_uint32), ("pad", C.c_uint32 * 3)]


class SsbVecQuery(C.Structure):
    _fields_ = [("queries", C.c_void_p), ("n_queries", C.c_uint32), ("k", C.c_uint32), ("query_format", C.c_uint32),
                ("has_threshold", C.c_uint32), ("similarity_threshold", C.c_float), ("ann_mode", C.c_uint32), ("n_probe", C.c_uint32),
                ("cluster_threshold", C.c_float)]


class SsbIndexBinParams(C.Structure):
    _fields_ = [("indexed_field_count", C.c_uint32), ("key_head_size", C.c_uint32), ("segment_number_bits", C.c_uint32),
                ("decode_positions", C.c_uint32)]


class SsbLevelDesc(C.Structure):
    _fields_ = [("level_id", C.c_uint32), ("n_docs", C.c_uint32), ("n_terms", C.c_uint32), ("n_fields", C.c_uint32),
                ("term_keys", C.c_void_p), ("posting_offsets", C.c_void_p), ("doc_ids", C.c_void_p),
                ("tfs", C.c_void_p), ("doc_len_bytes", C.c_void_p), ("positions", C.c_void_p)]


class SsbLevelNgrams(C.Structure):
    _fields_ = [("component_tfs", C.c_void_p), ("component_df_bytes", C.c_void_p)]


# SSB_LEXSIM_* (LexicalSimilarity), SSB_NGRAM_DF_* (which level's df bytes an n-gram list keeps), SSB_NGRAM_* (NgramType, key low bits)
LEXSIM_BM25F, LEXSIM_BM25F_PROXIMITY = 0, 1
NGRAM_DF_FIRST_LEVEL, NGRAM_DF_LAST_LEVEL = 0, 1
NGRAM_FF, NGRAM_FR, NGRAM_RF, NGRAM_FFF, NGRAM_RFF, NGRAM_FFR, NGRAM_FRF = 1, 2, 3, 4, 5, 6, 7


class SsbLexBatch(C.Structure):
    _fields_ = [("n_queries", C.c_uint32), ("query_type", C.c_uint32), ("term_offsets", C.c_void_p),
                ("term_keys", C.c_void_p), ("term_flags", C.c_void_p),
                ("filter_offsets", C.c_void_p), ("filters", C.c_void_p), ("filter_set_values", C.c_void_p),
                ("field_masks", C.c_void_p)]


class SsbFacetField(C.Structure):
    _fields_ = [("type", C.c_uint32), ("offset", C.c_uint32)]


class SsbFacetFilter(C.Structure):
    _fields_ = [("facet", C.c_uint32), ("kind", C.c_uint32), ("start", C.c_uint64), ("end", C.c_uint64),
                ("set_first", C.c_uint32), ("set_count", C.c_uint32)]


# SSB_FACET_* (FieldType of a facet field) and SSB_FILTER_*
FACET_U8, FACET_U16, FACET_U32, FACET_U64, FACET_I8, FACET_I16, FACET_I32, FACET_I64, FACET_TIMESTAMP, FACET_F32, FACET_F64, \
    FACET_STRING16, FACET_STRING32, FACET_POINT, FACET_STRINGSET16, FACET_STRINGSET32 = range(16)
FILTER_RANGE, FILTER_SET, FILTER_POINT = 0, 1, 2
SET_COMBINATION = 1 << 63           # SSB_SET_COMBINATION: a StringSet filter value that is a combination id, not a member id
UNIT_KILOMETERS, UNIT_MILES = 0, 1


class SsbSortCriterion(C.Structure):
    _fields_ = [("source", C.c_uint32), ("facet", C.c_uint32), ("order", C.c_uint32), ("pad", C.c_uint32)]


class SsbFacetRequest(C.Structure):
    _fields_ = [("facet", C.c_uint32), ("kind", C.c_uint32), ("length", C.c_uint32), ("has_prefix", C.c_uint32),
                ("rank_lo", C.c_uint32), ("rank_hi", C.c_uint32), ("n_ranges", C.c_uint32), ("unit", C.c_uint32),
                ("range_starts", C.c_void_p)]


class SsbFacetCount(C.Structure):
    _fields_ = [("value", C.c_uint32), ("pad", C.c_uint32), ("count", C.c_uint64)]


# SSB_FACET_COUNT_* (kind of a facet request) and the request limits
FACET_COUNT_VALUES, FACET_COUNT_RANGES = 0, 1
MAX_FACET_RANGES, MAX_FACET_LENGTH, MAX_FACET_REQUESTS = 256, 1024, 16


# SSB_SORT_* (source of a sort criterion) and SSB_SORT_ASCENDING / DESCENDING
SORT_FACET, SORT_ID, SORT_SCORE = 0, 1, 2
SORT_ASCENDING, SORT_DESCENDING = 0, 1


class SsbStats(C.Structure):
    _fields_ = [("kernel_launches", C.c_uint64), ("algorithmic_bytes", C.c_uint64), ("h2d_bytes", C.c_uint64),
                ("d2h_bytes", C.c_uint64), ("postings_visited", C.c_uint64), ("probes", C.c_uint64),
                ("items_processed", C.c_uint64), ("items_skipped", C.c_uint64), ("dominant_kernel_ns", C.c_uint64),
                ("scan_bytes_read", C.c_uint64), ("filter_fallbacks", C.c_uint64), ("reserved", C.c_uint64 * 1)]


# every symbol include/seekstorm_b200.h declares
EXPORTS = [
    "ssb_abi_version", "ssb_last_error", "ssb_create", "ssb_destroy", "ssb_lexical_add_level",
    "ssb_vector_add_level_clustered", "ssb_lexical_set_field_boosts", "ssb_lexical_set_ngram_config", "ssb_lexical_add_level_ngrams", "ssb_lexical_commit", "ssb_lexical_dict_size", "ssb_lexical_dict_export", "ssb_lexical_set_global_df",
    "ssb_load_index_bin", "ssb_load_index_bin_ngrams", "ssb_load_vector_bin", "ssb_index_bin_inspect", "ssb_index_bin_inspect_ngrams", "ssb_set_deleted", "ssb_set_facets", "ssb_set_facet_value_order", "ssb_set_facet_string_sets", "ssb_vector_set_turboquant_mask", "ssb_vector_add_level", "ssb_vector_count", "ssb_vector_reserve", "ssb_set_vector_kernel", "ssb_search_lexical", "ssb_search_lexical_sorted", "ssb_search_lexical_sorted_ex", "ssb_search_lexical_facets", "ssb_search_empty", "ssb_search_empty_facets", "ssb_search_vector", "ssb_search_vector_ex", "ssb_search_hybrid",
    "ssb_vector_add_level_fields", "ssb_load_vector_bin_fields", "ssb_search_vector_fields",
    "ssb_rrf_fuse", "ssb_comm_unique_id", "ssb_comm_init", "ssb_comm_attach", "ssb_comm_destroy", "ssb_lexical_sync_df",
    "ssb_search_vector_keys", "ssb_search_lexical_keys", "ssb_merge_keys", "ssb_sync",
    "ssb_stream", "ssb_set_stream", "ssb_last_stats",
]

_lib = None


class SsbError(RuntimeError):
    pass


def lib():
    """Load the library (raises if it has not been built: run `python -c 'import __graft_entry__ as g; g.build()'`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SsbError(f"{LIB_PATH} not found — build it with __graft_entry__.build(); there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int32
    L.ssb_abi_version.restype = u32
    L.ssb_last_error.restype = C.c_char_p
    sigs = {
        "ssb_create": [C.POINTER(SsbConfig), C.POINTER(vp)],
        "ssb_destroy": [vp],
        "ssb_lexical_add_level": [vp, C.POINTER(SsbLevelDesc)],
        "ssb_lexical_commit": [vp, u64, u64],
        "ssb_lexical_set_field_boosts": [vp, u32, vp],
        "ssb_lexical_set_ngram_config": [vp, u32, u32],
        "ssb_lexical_add_level_ngrams": [vp, C.POINTER(SsbLevelDesc), C.POINTER(SsbLevelNgrams)],
        "ssb_lexical_dict_size": [vp, C.POINTER(u64)],
        "ssb_lexical_dict_export": [vp, vp, vp, u64],
        "ssb_lexical_set_global_df": [vp, vp, vp, u64],
        "ssb_vector_add_level": [vp, u32, vp, u64, vp, u32, u32],
        "ssb_vector_add_level_clustered": [vp, u32, vp, u64, vp, u32, u32, vp, u32],
        "ssb_load_index_bin": [vp, vp, u64, C.POINTER(SsbIndexBinParams), C.POINTER(u64)],
        "ssb_load_vector_bin": [vp, vp, u64, C.POINTER(u64)],
        "ssb_index_bin_inspect": [vp, u64, C.POINTER(SsbIndexBinParams), vp],
        "ssb_load_index_bin_ngrams": [vp, vp, u64, C.POINTER(SsbIndexBinParams), C.POINTER(u64)],
        "ssb_index_bin_inspect_ngrams": [vp, u64, C.POINTER(SsbIndexBinParams), vp],
        "ssb_set_deleted": [vp, vp, u64],
        "ssb_set_facets": [vp, vp, u64, u64, u32, vp, u32],
        "ssb_set_facet_value_order": [vp, u32, vp, u32],
        "ssb_set_facet_string_sets": [vp, u32, vp, vp, u32, u32],
        "ssb_vector_set_turboquant_mask": [vp, vp, u32],
        "ssb_vector_count": [vp, C.POINTER(u64)],
        "ssb_vector_reserve": [vp, u64],
        "ssb_set_vector_kernel": [vp, u32],
        "ssb_search_lexical": [vp, C.POINTER(SsbLexBatch), u32, u32, vp, vp, vp],
        "ssb_search_lexical_sorted": [vp, C.POINTER(SsbLexBatch), vp, u32, u32, u32, vp, vp, vp],
        "ssb_search_lexical_sorted_ex": [vp, C.POINTER(SsbLexBatch), vp, u32, vp, u32, u32, vp, vp, vp],
        "ssb_search_lexical_facets": [vp, C.POINTER(SsbLexBatch), vp, u32, vp, vp, vp],
        "ssb_search_empty": [vp, C.POINTER(SsbLexBatch), vp, u32, vp, u32, u32, vp, vp, vp],
        "ssb_search_empty_facets": [vp, vp, u32, vp, vp],
        "ssb_search_vector": [vp, vp, u32, u32, vp, vp],
        "ssb_search_vector_ex": [vp, C.POINTER(SsbVecQuery), vp, vp, vp, vp],
        "ssb_search_hybrid": [vp, C.POINTER(SsbLexBatch), vp, u32, vp, vp],
        "ssb_vector_add_level_fields": [vp, u32, vp, u64, vp, u32, u32, vp, u32, vp, vp],
        "ssb_load_vector_bin_fields": [vp, vp, u64, C.POINTER(u64)],
        "ssb_search_vector_fields": [vp, C.POINTER(SsbVecQuery), vp, vp, vp, vp, vp],
        "ssb_rrf_fuse": [vp, u32, vp, u32, vp, C.POINTER(u32)],
        "ssb_search_vector_keys": [vp, vp, u32, u32, vp],
        "ssb_search_lexical_keys": [vp, C.POINTER(SsbLexBatch), u32, u32, vp, vp],
        "ssb_merge_keys": [vp, vp, u32, u32, u32, vp, vp],
        "ssb_sync": [vp],
        "ssb_comm_unique_id": [vp],
        "ssb_comm_init": [vp, vp, u32, u32],
        "ssb_comm_attach": [vp, vp, u32, u32],
        "ssb_comm_destroy": [vp],
        "ssb_lexical_sync_df": [vp],
        "ssb_set_stream": [vp, vp],
        "ssb_last_stats": [vp, C.POINTER(SsbStats)],
    }
    for name, args in sigs.items():
        f = getattr(L, name)
        f.argtypes = args
        f.restype = i32
    L.ssb_stream.argtypes = [vp]
    L.ssb_stream.restype = vp
    _lib = L
    return L


def check(rc: int):
    if rc != SSB_OK:
        msg = lib().ssb_last_error().decode("utf-8", "replace")
        raise SsbError(f"libseekstorm_b200 error {rc}: {msg}")
