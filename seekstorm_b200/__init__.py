"""seekstorm_b200 — H100-native (sm_90a) drop-in for the two query-time hot paths behind SeekStorm's
Index::search(): BM25 AND/OR top-k and the brute-force f32 vector scan (+ RRF hybrid).

The compute lives in libseekstorm_b200.so (hand-written CUDA, C-ABI in include/seekstorm_b200.h);
this package is the host-side mirror of the reference's search interface.  No CPU fallback.
"""
from .index import (AnnMode, DistanceUnit, FacetFilter, Index, LexicalSimilarity, NgramSet, NgramType, QueryFacet, QueryType, RangeType, Result, ResultObject, ResultSort, ResultType, SearchMode, SortOrder,
                    VectorSimilarity, ngram_key, ngram_rewrite, synthetic_term_key)
from ._lib import SsbError, lib, LIB_PATH

__all__ = ["AnnMode", "DistanceUnit", "FacetFilter", "Index", "LexicalSimilarity", "NgramSet", "NgramType", "QueryFacet", "QueryType", "RangeType", "Result", "ResultObject", "ResultSort", "ResultType", "SearchMode", "SortOrder",
           "VectorSimilarity", "SsbError", "lib", "LIB_PATH", "ngram_key", "ngram_rewrite", "synthetic_term_key"]
