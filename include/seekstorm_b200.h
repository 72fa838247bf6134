/*
 * seekstorm_b200.h — C ABI of libseekstorm_b200.so, the H100 (sm_90a) drop-in for the two query-time hot
 * paths behind SeekStorm's Index::search():
 *   (a) BM25 top-k over block-partitioned posting lists (AND / OR with block-max pruning), and
 *   (b) the brute-force f32 dot / cosine / Euclidean vector scan with fused top-k,
 * plus their RRF hybrid.  Plain pointers and sizes only; every pointer argument may be a HOST pointer or a
 * DEVICE pointer of the index's device (detected with cudaPointerGetAttributes) unless stated otherwise.
 *
 * The reference has no FFI for this path; the seams this ABI replaces are (all paths relative to
 * /root/reference/seekstorm/src/):
 *   ssb_search_lexical  <- SearchLexicalShard::search_lexical_shard  search.rs:2427-2458 (body 2445-3767),
 *                          i.e. the kernel-level calls single_blockid / union_docid_2 / union_docid_3 /
 *                          union_blockid / intersection_blockid dispatched at search.rs:3370-3563
 *   ssb_search_vector   <- SearchVectorShard::search_vector_shard    vector.rs:1105-1115 (body 1202-1514)
 *   ssb_search_hybrid   <- Search::search, SearchMode::Hybrid        search.rs:1134-1150, RRF 1962-2035
 *   ssb_lexical_add_level / ssb_lexical_commit <- the committed level as written by commit.rs:203-467 and
 *                          read back by index.rs:3253-3830 (postings, tf = positions_count, byte4 doc lengths)
 *   ssb_vector_add_level <- vector.bin level records written by vector.rs:969-1100
 * INTEGRATION.md shows the Rust `extern "C"` block + shim a maintainer would add.
 *
 * Conventions: every call returns int32_t status (0 = OK, <0 = SSB_E_*), never unwinds, never aborts.
 * Outputs are caller-allocated.  search_* calls on one handle may run CONCURRENTLY from many threads: each takes a
 * search context (CUDA stream + workspaces) from an internal pool, the committed index data is immutable and shared.
 * Index mutation (add_level / commit / set_global_df / set_stream) takes the handle exclusively, like the reference's
 * RwLock around a shard (commit.rs:142, index.rs:5508).
 * Doc ids on the ABI are the reference's shard-local ids: (level << 16) | local (vector.rs:1448,
 * add_result.rs docid = block_id<<16 | local), widened to u64.
 */
#ifndef SEEKSTORM_B200_H
#define SEEKSTORM_B200_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SSB_ABI_VERSION 3
#define SSB_K_MAX 32u            /* top-k capacity of one kernel pass (lane-distributed lists); *_keys calls */
#define SSB_K_LIMIT 1024u        /* ssb_search_lexical / ssb_search_vector page beyond 32 internally         */
#define SSB_MAX_QUERY_TERMS 32u  /* unique terms per lexical query (<= 4: record path; 5..32: one term per lane)  */

enum { SSB_OK = 0, SSB_E_INVALID = -1, SSB_E_CUDA = -2, SSB_E_NOMEM = -3, SSB_E_STATE = -4,
       SSB_E_UNSUPPORTED = -5, SSB_E_NO_DEVICE = -6 };

/* QueryType (search.rs, enum QueryType): Union / Intersection / Phrase.  A PHRASE batch lists every query's terms in phrase order,
 * repeated terms included ("to be or not to be" = 6 keys); a doc matches when it contains all of them and token i occurs at position
 * p + i for some p (add_result.rs:3586-3684); scores and counts as for an intersection of the unique terms.  Needs levels loaded with
 * ssb_level_desc.positions; NOT terms are not accepted in a phrase batch.  Several indexed fields (add_result.rs:3247-3389): positions
 * restart in every field and the phrase must occur inside ONE field; with a field filter (ssb_lex_batch.field_masks) only the fields of
 * the filter are searched. */
enum { SSB_QUERY_UNION = 0, SSB_QUERY_INTERSECTION = 1, SSB_QUERY_PHRASE = 2 };
/* ResultType (search.rs:150-175): Count / Topk / TopkCount (default) */
enum { SSB_RESULT_COUNT = 0, SSB_RESULT_TOPK = 1, SSB_RESULT_TOPKCOUNT = 2 };
/* VectorSimilarity (vector_similarity.rs:20-30) */
enum { SSB_SIM_DOT = 0, SSB_SIM_COSINE = 1, SSB_SIM_EUCLIDEAN = 2 };
/* Quantization (vector_similarity.rs `Quantization`): SCALAR_I8 = ScalarQuantizationI8.
 *   Cosine   : rows and queries are normalised, then quantised round(v*127) clamped to [-127,127] (vector_similarity.rs:1226-1232,
 *              vector.rs:585-640); score = the exact int32 dot product as f32 (vector_similarity.rs:193-206, 1011-1016).
 *   Dot      : per-vector scale = max|x|/127, codes round(x/scale) (QuantizedVector::new_scale, vector_similarity.rs:1340-1353);
 *              score = dot_i32 as f32 * query_scale * row_scale (dot_i8_quantized, :1754-1758).
 *   Euclidean: new_scale_norm (:1356-1371), the NON-AFFINE variant the reference uses for non-integer data (vector.rs:651-660);
 *              score = -max(0, query_norm + row_norm - 2*dot) (euclidean_i8_quantized, :1721-1734).  When the FIRST vector of the index is
 *              integer-valued in 0..255 (SIFT-like data) the reference switches the shard to its AFFINE quantiser for good
 *              (new_scale_norm_affine, :1414-1463: codes = round(x / scale) + zero_point with scale / zero point from the running min / max
 *              of everything indexed so far; euclidean_i8_quantized_affine, :1770-1795) — so does this library: rows must then be added
 *              in the reference's ingestion order, queries are quantised with the state the index has reached.
 * All three are bit-exact with the scalar CPU arithmetic (integer accumulation on s8 wgmma, reference operation order). */
enum { SSB_QUANT_NONE = 0, SSB_QUANT_SCALAR_I8 = 1,
       /* TurboQuantI8 (vector_similarity.rs:1825-2093): every vector (after normalize_f32 for Cosine) is zero-padded to the next power of
        * two, sign-flipped by the index's seed mask, rotated by the normalised fast Walsh-Hadamard transform and quantised with
        * scale = max(||x|| / sqrt(dim) / 32, 1e-8); rows are stored at next_power_of_two(dims) bytes.  Scores as in the reference:
        * Dot / Cosine = -(dot_i32 as f32 * query_scale * row_scale) (it negates the estimate, :161-176, 220-235), Euclidean =
        * -max(0, query_norm + row_norm - 2 * dot_i32 as f32 * query_scale * row_scale) (:2058-2069).  Bit-exact with the scalar CPU
        * arithmetic.  Needs ssb_vector_set_turboquant_mask before the first level. */
       SSB_QUANT_TURBO_I8 = 2 };
/* which vector scan kernel to use.  FFMA: FP32 scan, 16 queries per corpus pass (HBM-bound).  TCGEN05[_N64]: tensor-core scan with
 * the 3xTF32 split, 128 (64) queries per pass.  TCGEN05_BF16[_N64|_N256]: the 3xBF16 split (half the operand bytes; score error ~1e-5
 * relative, inside the 1e-4 tolerance), 128 (64, 256) queries per pass.  FILTER[_N256]: one fp16 product over a 2-byte plane of the
 * corpus selects, with a proven error margin, the <= 32 rows that can be in the top-k; those are re-scored with the plain f32 dot product
 * and queries whose candidate set did not fit are re-run by an exact f32 scan on the device: the exact f32 top-k, 128 (256) queries per
 * pass; FILTER_N256_PAIR: the 256-query filter scan on CTA pairs sharing one copy of the query block (TMA multicast).  The filter scans
 * run for k <= 16 without paging; other calls take TCGEN05_BF16 (FILTER) or the cheaper of TCGEN05_BF16 and _N256 (the 256-query ones).
 * AUTO: the filter scan whenever it can run (FILTER up to 128 queries, FILTER_N256 above), else FFMA up to 16 queries and the cheaper of
 * TCGEN05_BF16 and _N256 above.  Euclidean f32 indexes always take FFMA, int8 indexes the s8 tensor-core scan (128 queries per pass). */
enum { SSB_VEC_KERNEL_AUTO = 0, SSB_VEC_KERNEL_FFMA = 1, SSB_VEC_KERNEL_TCGEN05 = 2, SSB_VEC_KERNEL_TCGEN05_N64 = 3,
       SSB_VEC_KERNEL_TCGEN05_BF16 = 4, SSB_VEC_KERNEL_TCGEN05_BF16_N64 = 5, SSB_VEC_KERNEL_TCGEN05_BF16_N256 = 6,
       SSB_VEC_KERNEL_TCGEN05_FILTER = 7, SSB_VEC_KERNEL_TCGEN05_FILTER_N256 = 8, SSB_VEC_KERNEL_TCGEN05_FILTER_N256_PAIR = 9 };

typedef struct ssb_index ssb_index;

/* min_heap.rs:17-40 `Result` {doc_id, score}; 16 bytes */
typedef struct { uint64_t doc_id; float score; uint32_t pad; } ssb_hit;
/* the `vb`-feature fields of `Result` (min_heap.rs:21-39), parallel to an ssb_hit array; 48 bytes.
 * source: ResultSource (Lexical / Vector / Hybrid). */
enum { SSB_SOURCE_LEXICAL = 0, SSB_SOURCE_VECTOR = 1, SSB_SOURCE_HYBRID = 2 };
typedef struct {
    uint32_t field_id, chunk_id, level_id, shard_id, cluster_id;
    float cluster_score, vector_score, lexical_score;
    uint32_t source; uint32_t pad[3];
} ssb_hit_ext;

typedef struct {
    int32_t  device;             /* CUDA device ordinal                                                  */
    uint32_t max_batch;          /* max queries per search_* call (workspace sizing); 0 -> 4096          */
    uint32_t vector_dims;        /* 0 = no vector index                                                   */
    uint32_t vector_similarity;  /* SSB_SIM_*  (meta.inference similarity)                               */
    uint32_t vector_kernel;      /* SSB_VEC_KERNEL_*                                                      */
    uint32_t vector_quantization;/* SSB_QUANT_* (0 = f32 corpus)                                           */
    uint32_t reserved[2];
} ssb_config;

/* One committed level = one 64K-doc block of the shard, in a neutral (decoded) layout.
 * Replaces the per-level bytes the reference keeps in index.bin (ARCHITECTURE.md:77-82):
 *   doc_ids / tfs : per term, ascending local doc ids and positions_count (tf), what
 *                   intersection.rs:199-247 + add_result.rs:2036-2197 decode per candidate
 *   doc_len_bytes : the level's byte4 field-length array (index.rs:770-776)                    */
typedef struct {
    uint32_t level_id;                /* block id; doc_id = level_id<<16 | local                         */
    uint32_t n_docs;                  /* <= 65536                                                         */
    uint32_t n_terms;
    uint32_t n_fields;                /* indexed fields: 0 / 1 = one field; F > 1 needs ssb_lexical_set_field_boosts(ix, F, ..) first  */
    const uint64_t* term_keys;        /* [n_terms] 64-bit term hash (reference key_hash), any order       */
    const uint32_t* posting_offsets;  /* [n_terms+1]                                                      */
    const uint16_t* doc_ids;          /* [n_postings] ascending within a term                            */
    const uint16_t* tfs;              /* [n_postings]; F fields: [n_postings][F], 0 = the term does not occur in that field; the     */
                                      /* per-field tfs also give the lengths of a posting's per-field position runs (positions)      */
    const uint8_t*  doc_len_bytes;    /* [n_docs];     F fields: [F][n_docs] (document_length_compressed_array[field], index.rs:770-776) */
    const uint16_t* positions;        /* [sum of tfs] or NULL: the term positions of every posting, in posting order, ascending inside a   */
                                      /* posting (what get_next_position_singlefield decodes, add_result.rs:2036-2197); needed by          */
                                      /* SSB_QUERY_PHRASE only; either every level carries them or none.  F fields: a posting holds        */
                                      /* Σ_f tfs[p][f] positions, one run per field in field order (field 0's tfs[p][0] first), each run   */
                                      /* strictly ascending and starting again from 0 (add_result.rs:3258-3283)                             */
} ssb_level_desc;

/* ---- facets and facet filters (SURVEY.md §8f row 4) ---------------------------------------------------- */
/* FieldType of a facet field (index.rs `FieldType`; FilterSparse search.rs:863-881).  POINT (geo, index.rs:5803-5819): the row holds
 * the u64 Morton code encode_morton_2_d([lat, lon]) (geo_search.rs:27-42): x = ((lat * 1e7) as i32) as u32 in the even bits, y = the
 * same of lon in the odd bits, Rust's saturating `as i32` (NaN -> 0).  The reference writes no code for a coordinate outside
 * [-90, 90] x [-180, 180]: that row stays 0, which decodes to (0.0, 0.0).  Decode: (x as i32) as f64 / 1e7 (geo_search.rs:58-79).
 * STRINGSET16 / STRINGSET32 (multi-value string facets, index.rs:5763-5801): the row holds the u16 / u32 id of the doc's COMBINATION —
 * its strings sorted byte-wise and joined with "_", numbered in first-insertion order; the member lists of the combinations are given
 * by ssb_set_facet_string_sets. */
enum { SSB_FACET_U8 = 0, SSB_FACET_U16 = 1, SSB_FACET_U32 = 2, SSB_FACET_U64 = 3, SSB_FACET_I8 = 4, SSB_FACET_I16 = 5,
       SSB_FACET_I32 = 6, SSB_FACET_I64 = 7, SSB_FACET_TIMESTAMP = 8, SSB_FACET_F32 = 9, SSB_FACET_F64 = 10,
       SSB_FACET_STRING16 = 11, SSB_FACET_STRING32 = 12, SSB_FACET_POINT = 13, SSB_FACET_STRINGSET16 = 14, SSB_FACET_STRINGSET32 = 15 };
/* DistanceUnit (index.rs) of a POINT filter */
enum { SSB_UNIT_KILOMETERS = 0, SSB_UNIT_MILES = 1 };
/* one facet field of the shard's facet file: its type and its byte offset inside a doc's row (`facet.offset`, add_result.rs:345) */
typedef struct { uint32_t type; uint32_t offset; } ssb_facet_field;
/* One filter of one query.  RANGE = Rust `Range<T>::contains`: start <= value < end, compared in the facet's own type (floats by
 * PartialOrd: NaN is never inside).  start / end carry the bound widened to 8 bytes: unsigned types as u64, signed types and
 * Timestamp as i64 (two's complement), F32 / F64 as the bits of the f64 value.  SET (String16 / String32) = `values.contains(id)`
 * over filter_set_values[set_first .. set_first + set_count).  A facet without a filter entry is FilterSparse::None.
 * POINT (POINT facets only; FacetFilter::Point {field, (base, start..end, unit)} -> FilterSparse::Point, search.rs:2712-2723,
 * add_result.rs:462-478): start / end are the distance range as f64 bits; set_count = 3 values at filter_set_values[set_first ..]: the
 * base's lat and lon as f64 bits, then the unit (SSB_UNIT_*).  A doc passes when morton_min <= code < morton_max, the interval of
 * point_distance_to_morton_range(base, end, unit) (geo_search.rs:109-144, computed by the host), AND start <= euclidian_distance(base,
 * decode(code), unit) < end: the equirectangular R * sqrt(x*x + y*y), R = 6371.0087714 km or 3958.761315801475 mi.  The reference's
 * quirks are kept: the interval is a Z-order range of u32-cast signed coordinates, so a box that crosses latitude 0 or longitude 0
 * usually has min > max and no doc passes; near the poles the longitude delta explodes and the encode saturates; a NaN in the base or
 * the bounds rejects every doc.
 * Precision: the integer decode, /1e7, + - * and sqrt are IEEE round-to-nearest in the reference's operation order without FMA
 * contraction, bit for bit; the Morton interval is computed on the host with the C library's cos.  The device evaluates the distance's
 * cos with CUDA's double cos (within 2 ulp, not guaranteed equal to the host libm): a filter decision can differ from the reference only
 * for a distance within a few ulp of a bound.
 * SET on a STRINGSET facet (FacetFilter::StringSet16 / 32, search.rs:2643-2710): the values are MEMBER ids (ssb_set_facet_string_sets),
 * or, with bit 63 (SSB_SET_COMBINATION) set, a combination id that must match exactly.  A doc passes when its combination id equals a
 * flagged id or when one of its combination's members is listed.  The reference accepts, per filter string v, every combination whose
 * members contain v (string_set_to_single_term_id, index.rs:4282-4297) plus the combination whose joined key equals v: the host sends
 * v's member id, and the flagged id of that combination when it does not already hold v (["a", "b"] for v = "a_b").  A member id
 * >= n_values or a flagged id >= n_sets is SSB_E_INVALID; a STRINGSET facet without string sets is SSB_E_STATE. */
enum { SSB_FILTER_RANGE = 0, SSB_FILTER_SET = 1, SSB_FILTER_POINT = 2 };
#define SSB_SET_COMBINATION (1ull << 63)
typedef struct ssb_facet_filter {
    uint32_t facet;                   /* index into the fields given to ssb_set_facets                    */
    uint32_t kind;                    /* SSB_FILTER_*                                                     */
    uint64_t start, end;              /* RANGE bounds (see above)                                         */
    uint32_t set_first, set_count;    /* SET / POINT: slice of ssb_lex_batch.filter_set_values            */
} ssb_facet_filter;
#define SSB_MAX_FACETS 16u
#define SSB_MAX_FILTERS_PER_QUERY 16u

/* A batch of lexical queries, already tokenised by the host (tokenizer.rs is out of scope): unique terms
 * per query as 64-bit keys, CSR layout; at most SSB_MAX_QUERY_TERMS per query (checked for host arrays; with device
 * arrays extra terms are ignored).  Repeated keys inside a query count once, as in the reference's unique_terms. */
#define SSB_TERM_NOT 1u            /* term_flags bit 0: the '-' operator — docs containing the term are excluded (not_query_list,  */
                                  /* add_result.rs:3440-3496); NOT terms neither score nor count towards the 32-term limit       */
#define SSB_MAX_NOT_TERMS 4u
typedef struct {
    uint32_t n_queries;
    uint32_t query_type;              /* SSB_QUERY_* (applies to the whole batch)                         */
    const uint32_t* term_offsets;     /* [n_queries+1]                                                    */
    const uint64_t* term_keys;        /* [term_offsets[n_queries]]                                        */
    const uint8_t*  term_flags;       /* [term_offsets[n_queries]] SSB_TERM_* per term, or NULL (all positive); at most        */
                                      /* SSB_MAX_NOT_TERMS NOT terms per query                                                 */
    /* facet filters (ABI v3; `facet_filter: Vec<FacetFilter>` of search_lexical_shard, search.rs:2427-2458, resolved to one      */
    /* FilterSparse per facet, search.rs:863-881): HOST arrays or NULL.  A doc enters neither the top-k nor the counts unless      */
    /* every filter of its query accepts its facet value (is_facet_filter, add_result.rs:340-478).  Needs ssb_set_facets.          */
    const uint32_t* filter_offsets;           /* [n_queries+1] or NULL (no query is filtered)                                      */
    const struct ssb_facet_filter* filters;   /* [filter_offsets[n_queries]]                                                       */
    const uint64_t* filter_set_values;        /* value ids of the SSB_FILTER_SET filters (String16 / String32), the payloads of    */
                                              /* the SSB_FILTER_POINT filters, or NULL                                              */
    /* field filter (`field_filter: Vec<String>` -> field_filter_set, add_result.rs:3124-3137, 3558-3571): HOST array [n_queries] or   */
    /* NULL; bit f = indexed field f is in the query's filter, 0 = no field filter.  A doc is dropped when a query term it contains    */
    /* occurs in none of the filter's fields (tested like the reference only when term fields + filter fields <= indexed fields);      */
    /* scores still sum every field.  Indexes with one indexed field ignore it (the reference's test can never fire there).            */
    const uint32_t* field_masks;
} ssb_lex_batch;

uint32_t    ssb_abi_version(void);
const char* ssb_last_error(void);                              /* thread-local, never NULL              */

int32_t ssb_create(const ssb_config* cfg, ssb_index** out);
int32_t ssb_destroy(ssb_index* ix);

/* ---- lexical index: add immutable levels, then commit global statistics --------------------------- */
int32_t ssb_lexical_add_level(ssb_index* ix, const ssb_level_desc* level);
/* n_docs = indexed_doc_count, len_sum_normalized = positions_sum_normalized (commit.rs:318-319) of the
 * WHOLE shard (all GPUs' levels).  Builds the dictionary, bm25_component_cache (commit.rs:321-325),
 * per-(term,block) block-max (index.rs:2938-3049) and the bitmap containers for dense lists. */
/* Several indexed fields (BM25F, get_bm25f_multiterm_multifield add_result.rs:1171-1426): n_fields <= 4 and the per-field boosts
 * (indexed_schema_vec[f].boost; NULL = 1.0) — before the first ssb_lexical_add_level.  Score of a doc = sum over query terms (query
 * order) and over the fields the term occurs in (ascending) of boost_f * idf_t * tf_tf*(K+1)/(tf_tf + cache[len_byte_f(doc)]),
 * accumulated left to right like the reference.  Pruning bounds use an upper bound of the boost-weighted per-posting sum; such an
 * index is searched by the general (one term per lane) kernel. */
int32_t ssb_lexical_set_field_boosts(ssb_index* ix, uint32_t n_fields, const float* boosts);
/* ---- n-gram posting lists (NGRAM_SEARCH.md; keys tokenizer.rs:678-685) ---------------------------------------------------------
 * An n-gram key is hash64("a b" / "a b c") | NgramType: the low 3 bits name the type (index.rs:1854-1872).  Its postings are the docs
 * holding the n-gram, its tf the n-gram's own count, its positions the n-gram's start positions.  A PHRASE batch may list n-gram keys
 * between single-term keys: token i must then sit at p + i + (1 per earlier bigram) + (2 per earlier trigram) (search.rs:3305-3330).
 * LexicalSimilarity (index.rs:559-566): BM25F scores an n-gram list as the sum of its components, component c = the c-th word of the
 * n-gram: idf_c * tf_c*(K+1)/(tf_c + cache[len]), idf_c from the component's df decoded from the key head's byte4 code
 * (add_result.rs:1448-1478, search.rs:3231-3269).  BM25F_PROXIMITY (the reference's default) leaves the component idfs at 0 on a
 * single-field index: an n-gram list then adds 0 to a doc's score (it still selects the docs).  With single-term keys only the two
 * similarities score identically. */
enum { SSB_LEXSIM_BM25F = 0, SSB_LEXSIM_BM25F_PROXIMITY = 1 };
/* which level's key-head df bytes an n-gram list takes when it occurs in several levels: the FIRST level's (open_shard with
 * AccessType::Ram, index.rs:3633-3664) or the LAST level's (AccessType::Mmap, decode_posting_list_counts, search.rs:2224-2277) */
enum { SSB_NGRAM_DF_FIRST_LEVEL = 0, SSB_NGRAM_DF_LAST_LEVEL = 1 };
/* NgramType: the low 3 bits of an n-gram key (F = frequent term, R = rare term) */
enum { SSB_NGRAM_FF = 1, SSB_NGRAM_FR = 2, SSB_NGRAM_RF = 3, SSB_NGRAM_FFF = 4, SSB_NGRAM_RFF = 5, SSB_NGRAM_FFR = 6, SSB_NGRAM_FRF = 7 };
/* before the first level (else SSB_E_STATE); without it an index scores n-gram lists with BM25F_PROXIMITY and the first level's df bytes */
int32_t ssb_lexical_set_ngram_config(ssb_index* ix, uint32_t lexical_similarity, uint32_t df_level_rule);
/* the n-gram data of one level: HOST or DEVICE arrays.  component_tfs [n_postings][3]: per posting the tfs of the n-gram's components in
 * word order (tf_ngram1..3, add_result.rs:2076-2089; the third is ignored for bigrams, all three for single-term lists);
 * component_df_bytes [n_terms][3]: per term the key head's posting_count_ngram_{1,2,3}_compressed bytes (compress_postinglist.rs:28-230),
 * byte4 codes decoded like the document lengths (ignored for single-term keys). */
typedef struct {
    const uint16_t* component_tfs;
    const uint8_t*  component_df_bytes;
} ssb_level_ngrams;
/* ssb_lexical_add_level, where every key whose low 3 bits are not 0 is an n-gram list.  ngrams NULL = ssb_lexical_add_level.  One indexed
 * field only (several: SSB_E_UNSUPPORTED); not on a handle with a communicator, and ssb_comm_init / ssb_comm_attach / ssb_lexical_sync_df
 * refuse an index holding n-gram lists (SSB_E_UNSUPPORTED): which level's df bytes an n-gram takes is not defined once its levels are
 * split across GPUs.  ssb_lexical_set_global_df leaves n-gram keys alone: their dictionary idf is 1.0, the components carry the idfs.
 * Once the index holds n-gram lists, every level must come through this call: ssb_lexical_add_level refuses a level whose keys have low
 * bits set (SSB_E_INVALID), and this call refuses such keys when an earlier plain level carried them. */
int32_t ssb_lexical_add_level_ngrams(ssb_index* ix, const ssb_level_desc* level, const ssb_level_ngrams* ngrams);
int32_t ssb_lexical_commit(ssb_index* ix, uint64_t n_docs, uint64_t len_sum_normalized);
/* dictionary export / global document-frequency override (multi-GPU block-range sharding: idf uses the
 * global df, search.rs:3225).  keys/dfs are host pointers. */
int32_t ssb_lexical_dict_size(const ssb_index* ix, uint64_t* n_terms);
int32_t ssb_lexical_dict_export(const ssb_index* ix, uint64_t* keys, uint32_t* dfs, uint64_t cap);
int32_t ssb_lexical_set_global_df(ssb_index* ix, const uint64_t* keys, const uint32_t* dfs, uint64_t n);

/* ---- loading the reference's own shard files (SURVEY.md §8f row 1) ------------------------------------ */
/* index.bin of ONE shard as written by commit.rs:203-467 / read by open_shard (index.rs:3253-3516): header, then per 64K-doc level
 * the byte4 length array, the cumulative statistics, the segment table, key heads (compress_postinglist.rs:339-409) and key bodies
 * (Array / Bitmap / RLE doc-id containers, compress_postinglist.rs:694-977; tf from the rank-position pointers,
 * add_result.rs:2036-2197).  Adds every level and commits with the file's own indexed_doc_count / positions_sum_normalized.
 * bytes: HOST memory (e.g. the mmap of the file).  params come from the shard's index.json / schema.json. */
typedef struct {
    uint32_t indexed_field_count;   /* schema: indexed fields; only 1 is supported by the loader (multi-field BM25F: neutral layout, ssb_lexical_set_field_boosts)        */
    uint32_t key_head_size;         /* 20 without n-gram indexing, 22 / 23 with bigram / trigram df bytes                      */
    uint32_t segment_number_bits;   /* 11 (create_shard(.., 11, ..), index.rs:3295): 2048 dictionary segments per level        */
    uint32_t decode_positions;      /* != 0: also decode every posting's term positions (embedded layouts index_posting.rs:590-640, VINT delta  */
                                    /* blobs compress_postinglist.rs:946-977) and load them for SSB_QUERY_PHRASE; positions above 65535 fail   */
} ssb_index_bin_params;
int32_t ssb_load_index_bin(ssb_index* ix, const void* bytes, uint64_t len, const ssb_index_bin_params* params, uint64_t* n_docs_out);
/* host-only walk of an index.bin (no GPU needed): out = {levels, single-term keys, postings, sum of tf, indexed_doc_count,
 * positions_sum_normalized, FNV checksum over every (key, level, doc id, tf) in file order, FNV checksum over every decoded
 * position (decode_positions) or 0} */
int32_t ssb_index_bin_inspect(const void* bytes, uint64_t len, const ssb_index_bin_params* params, uint64_t out[8]);
/* ssb_load_index_bin that also loads the n-gram posting lists of a shard built with n-gram indexing (key_head_size 22 / 23): the key heads'
 * df bytes 14..16, the component tfs ahead of positions_count in every n-gram posting's blob (add_result.rs:2076-2089), its tf and (with
 * decode_positions) its start positions, fed through ssb_lexical_add_level_ngrams (ssb_lexical_set_ngram_config first, if at all).
 * ssb_load_index_bin keeps skipping n-gram keys. */
int32_t ssb_load_index_bin_ngrams(ssb_index* ix, const void* bytes, uint64_t len, const ssb_index_bin_params* params, uint64_t* n_docs_out);
/* host-only walk of the n-gram keys of an index.bin: out = {levels, n-gram keys, n-gram postings, sum of their tfs, FNV checksum over every
 * n-gram key, level and df bytes and every posting's (doc id, tf, component tfs) in file order, FNV checksum over their positions
 * (decode_positions) or 0, 0, 0} */
int32_t ssb_index_bin_inspect_ngrams(const void* bytes, uint64_t len, const ssb_index_bin_params* params, uint64_t out[8]);
/* vector.bin of one shard (vector.rs:1066-1094; Precision::F32 records of 24 + 4*dims bytes); dims = the index's vector_dims */
int32_t ssb_load_vector_bin(ssb_index* ix, const void* bytes, uint64_t len, uint64_t* n_vectors_out);
/* ssb_load_vector_bin that also keeps each record's VectorHeader.field_id / chunk_id (vector.rs:62-73) and adds the levels through
 * ssb_vector_add_level_fields.  A field id >= 32 -> SSB_E_INVALID; a handle with a communicator -> SSB_E_UNSUPPORTED. */
int32_t ssb_load_vector_bin_fields(ssb_index* ix, const void* bytes, uint64_t len, uint64_t* n_vectors_out);

/* ---- delete set ---------------------------------------------------------------------------------------- */
/* shard.delete_hashset (index.rs:1594; delete_document index.rs:5110): deleted docs are neither scored nor counted, in the
 * lexical path (add_result.rs:3435, union_count union.rs:975-1000) and in the vector scan (vector.rs:1450-1451).  doc_ids: host
 * array of shard-local ids (level << 16 | local); replaces the current set; n = 0 clears it.  Exclusive like a commit. */
int32_t ssb_set_deleted(ssb_index* ix, const uint64_t* doc_ids, uint64_t n);

/* ---- facets ---------------------------------------------------------------------------------------------- */
/* The shard's facet file (`facets_file_mmap`: one row of `facets_size_sum` bytes per doc, doc id = level << 16 | local;
 * is_facet_filter reads `row_bytes * docid + field.offset`, add_result.rs:343-347).  rows: HOST array [n_docs * row_bytes] holding
 * the rows of doc ids first_doc_id .. first_doc_id + n_docs (a shard of a sharded index passes the rows of its own level range).
 * Every value is converted once into an order-preserving 64-bit key and kept as one column per facet in HBM (8 bytes per doc and
 * facet); a doc outside the covered range fails every filter.  Replaces the current facets; n_docs = 0 clears them.  Exclusive. */
int32_t ssb_set_facets(ssb_index* ix, const void* rows, uint64_t first_doc_id, uint64_t n_docs, uint32_t row_bytes,
                       const ssb_facet_field* fields, uint32_t n_fields);
/* String16 / String32 facets sort by the value's STRING (result_ordering_shard, min_heap.rs:861-898, `values.get_index(id)`; Rust
 * String order = byte-wise lexicographic), which the library does not hold: rank_of_id[id] = position of id's string in that order
 * (equal strings, equal rank), computed by the host.  HOST array [n_ids].  ssb_set_facets clears it.  Needed by sorted searches only. */
int32_t ssb_set_facet_value_order(ssb_index* ix, uint32_t facet, const uint32_t* rank_of_id, uint32_t n_ids);
/* The member lists of a STRINGSET facet's combinations (facet.values of index.rs:5763-5801: per combination the FIRST doc's sorted list,
 * repeats and the empty list included), CSR over MEMBER ids: combination c holds members[set_offsets[c] .. set_offsets[c + 1]).  Member
 * ids are the ranks of the distinct member strings in byte-wise order (Rust String order), so a string prefix is an id interval and id
 * order is string order.  HOST arrays set_offsets [n_sets + 1] (ascending, from 0), members [set_offsets[n_sets]].  SSB_E_INVALID when a
 * member id is >= n_values, the facet's column holds an id >= n_sets, or a STRINGSET16 facet gets more than 65,535 sets (the reference's
 * ingest bound).  The sort rank of a combination is derived from its first member
 * (the empty combination below every string), with the facet's zones in those ranks: no ssb_set_facet_value_order for these facets.
 * ssb_set_facets clears it; filters, counts and sorting on the facet need it (else SSB_E_STATE).  Exclusive. */
int32_t ssb_set_facet_string_sets(ssb_index* ix, uint32_t facet, const uint64_t* set_offsets, const uint32_t* members, uint32_t n_sets,
                                  uint32_t n_values);

/* ---- vector index -------------------------------------------------------------------------------- */
/* rows: [n, dims] row-major f32 (row_stride_floats >= dims, 0 = dims); local_ids: [n] u16 or NULL (= 0..n-1).
 * Cosine: rows are L2-normalised on load (vector.rs:585-596 does this at index time). */
int32_t ssb_vector_add_level(ssb_index* ix, uint32_t level_id, const float* rows, uint64_t row_stride_floats,
                             const uint16_t* local_ids, uint32_t n, uint32_t dims);
/* The same level with its IVF cluster table (vector.bin: `u32 clusters; u32 child_count x clusters; records`, vector.rs:1066-1094): rows
 * are in cluster order, cluster c holds the next cluster_counts[c] rows, its medoid is its FIRST row (vector.rs:1316-1320).  Levels added
 * without a table are one cluster (what the reference writes below 100 vectors or with Clustering::None, vector.rs:1048-1062).  The
 * clusters only matter to ssb_search_vector_ex calls with ann_mode != SSB_ANN_ALL.  f32 indexes only. */
int32_t ssb_vector_add_level_clustered(ssb_index* ix, uint32_t level_id, const float* rows, uint64_t row_stride_floats,
                                       const uint16_t* local_ids, uint32_t n, uint32_t dims,
                                       const uint32_t* cluster_counts, uint32_t n_clusters);
/* Multi-vector documents: the level with each row's indexed field (field_ids, u8 [n], the reference's indexed_field_id, < 32 else
 * SSB_E_INVALID) and chunk id (chunk_ids, u32 [n]); cluster_counts as in _clustered, or NULL for one cluster.  Every vector level of an
 * index carries field ids or none does (mixing -> SSB_E_STATE).  The field filter of ssb_search_vector_fields / ssb_search_hybrid then
 * applies to the rows (search_vector_shard, vector.rs:1226-1238, 1411-1412), and ssb_hit_ext.field_id / chunk_id name each hit's best
 * row (TopK::push, vector.rs:436-470).  A handle with a communicator -> SSB_E_UNSUPPORTED (another rank's best row cannot be resolved). */
int32_t ssb_vector_add_level_fields(ssb_index* ix, uint32_t level_id, const float* rows, uint64_t row_stride_floats,
                                    const uint16_t* local_ids, uint32_t n, uint32_t dims, const uint32_t* cluster_counts,
                                    uint32_t n_clusters, const uint8_t* field_ids, const uint32_t* chunk_ids);
/* TurboQuantI8 indexes: the index's sign mask `TurboQuant.seed_mask` (dim = next_power_of_two(vector_dims) values of +1 / -1).  The
 * reference draws it once per index from ChaCha8Rng::seed_from_u64(1234) (vector_similarity.rs:1845-1859, index.rs:2215-2216) — a
 * third-party generator (rand_chacha) that this library does not restate: the host hands over the mask it holds.  Before the first level. */
int32_t ssb_vector_set_turboquant_mask(ssb_index* ix, const float* seed_mask, uint32_t dim);
int32_t ssb_vector_count(const ssb_index* ix, uint64_t* n_rows);
/* capacity hint: size the vector arenas for n_rows rows up front (loading level by level otherwise grows them geometrically) */
int32_t ssb_vector_reserve(ssb_index* ix, uint64_t n_rows);
/* switch the scan kernel (SSB_VEC_KERNEL_*) of an existing index */
int32_t ssb_set_vector_kernel(ssb_index* ix, uint32_t vector_kernel);

/* ---- search ---------------------------------------------------------------------------------------- */
/* hits: [n_queries * k] best-first (score desc, doc id asc); n_hits: [n_queries]; count_total: [n_queries] or
 * NULL (result_count_total: exact for Count/TopkCount, unspecified for Topk — search.rs:196-198). */
int32_t ssb_search_lexical(ssb_index* ix, const ssb_lex_batch* q, uint32_t k, uint32_t result_type,
                           ssb_hit* hits, uint32_t* n_hits, uint64_t* count_total);
/* `result_sort: Vec<ResultSort>` of Search::search (search.rs:1004-1013, ResultSort :893-901, resolved by ResultSortIndex :2497-2525):
 * the same search with the hits ordered by the criteria, compared left to right (result_ordering_shard, min_heap.rs:574-1051): a facet
 * in its own type (String16 / String32 by the value order of ssb_set_facet_value_order), the doc id (SSB_SORT_ID) or the score
 * (SSB_SORT_SCORE).  _id and _score end the comparison (min_heap.rs:580-604): criteria after them are ignored.  Ties on every criterion
 * fall back to score desc (:1043-1050), then doc id asc.  Deviations: a NaN facet value orders above +inf (descending puts it first), the
 * reference's partial_cmp makes it equal to everything; -0.0 == +0.0 as in the reference.  Hits carry the BM25 score; counts are those
 * of ssb_search_lexical (Count ignores the sort, search.rs:2498).  One sort for the whole batch; n_sort = 0, or criteria that reduce to
 * "_score desc", is ssb_search_lexical.  The facet criteria with their natural widths (8 bits U8 / I8, 16 bits U16 / I16 / String16,
 * 32 bits U32 / I32 / F32 / String32 / _id, 64 bits U64 / I64 / Timestamp / F64) must fit 64 bits in total (else SSB_E_UNSUPPORTED).
 * Needs ssb_set_facets rows for every doc of the lexical levels.  Not on a handle with a communicator (SSB_E_UNSUPPORTED).
 * STRINGSET16 / 32 (16 / 32 bits) sort by the combination's FIRST member string (min_heap.rs:393-420, 900-925); equal first members
 * tie.  Deviation: the empty combination, on which the reference panics, sorts below every string. */
enum { SSB_SORT_FACET = 0, SSB_SORT_ID = 1, SSB_SORT_SCORE = 2 };
enum { SSB_SORT_ASCENDING = 0, SSB_SORT_DESCENDING = 1 };          /* SortOrder, search.rs:885-890 */
typedef struct { uint32_t source, facet, order, pad; } ssb_sort_criterion;   /* facet: index into ssb_set_facets' fields (SSB_SORT_FACET) */
#define SSB_MAX_SORT_CRITERIA 4u
int32_t ssb_search_lexical_sorted(ssb_index* ix, const ssb_lex_batch* q, const ssb_sort_criterion* sort, uint32_t n_sort,
                                  uint32_t k, uint32_t result_type, ssb_hit* hits, uint32_t* n_hits, uint64_t* count_total);
/* The same with the bases of a POINT criterion (ResultSort on a Point facet with a FacetValue::Point base, min_heap.rs:510-529,
 * 1017-1037): bases is a HOST array [n_queries][2] (lat, lon), one base per query.  The criterion compares simplified_distance(decode(code),
 * base) = ((base.lon - p.lon) * cos(DEG2RAD * (p.lat + base.lat) / 2))^2 + (base.lat - p.lat)^2 in degrees (geo_search.rs:82-107):
 * ascending = nearest first.  A NaN distance orders like a NaN F64 value.  bases = NULL: a POINT criterion has no base and is dropped, as
 * the reference skips it; the bases are ignored by every other criterion.  A POINT criterion takes 64 bits, so only `_score` may follow it
 * (else SSB_E_UNSUPPORTED).  Precision: as for SSB_FILTER_POINT, every operation but cos is IEEE bit-exact; with CUDA's cos two docs at
 * DIFFERENT coordinates whose distances lie within a few ulp may order differently from the host libm; equal coordinates always tie.
 * ssb_search_lexical_sorted is this call with bases = NULL. */
int32_t ssb_search_lexical_sorted_ex(ssb_index* ix, const ssb_lex_batch* q, const ssb_sort_criterion* sort, uint32_t n_sort,
                                     const double* bases, uint32_t k, uint32_t result_type, ssb_hit* hits, uint32_t* n_hits,
                                     uint64_t* count_total);
/* Facet counts of a lexical batch (`query_facets` of Search::search, QueryFacet search.rs:234-…, facet_count add_result.rs:487-640): per
 * query and request, how many of the query's matches fall on each value (VALUES) or into each range (RANGES).  The docs counted are
 * exactly those result_count_total counts under Count / TopkCount for the same batch (delete set, NOT terms, facet filters, field filter
 * and phrase check applied).  The call computes the counts only: a caller runs it next to whichever search it makes on the batch.
 * One request set for the whole batch (as one sort is); a RANGES request on a POINT facet reads one base per query.
 *   VALUES (String16 / String32 facets): the `length` value ids with the most matches, count descending, then id ascending (the reference
 *     orders ties by hash-map arrival); ids with count 0 are left out.  has_prefix: only ids whose rank in the facet's value order
 *     (ssb_set_facet_value_order, else SSB_E_STATE) lies in [rank_lo, rank_hi) — the ids whose string starts with a prefix form one such
 *     interval.  length = 0: the facet is not collected (n_out 0).  length <= SSB_MAX_FACET_LENGTH.
 *   RANGES (numeric, Timestamp, F32 / F64 facets; POINT facets by the distance to the query's base in `unit`): bin i holds the docs whose
 *     value v has range_starts[i] <= v < range_starts[i + 1] (the last range is open above): the reference's binary search over the
 *     starts.  range_starts: n_ranges strictly ascending starts widened like SSB_FILTER_RANGE bounds (unsigned as u64, signed and
 *     Timestamp as i64, F32 / F64 and POINT distances as f64 bits); a NaN start or a list that does not ascend is SSB_E_INVALID.  All
 *     n_ranges raw counts are written, zeros included; RangeType (CountAboveRange / CountBelowRange), labels and the label prefix belong
 *     to the caller.  A value below the first start, a NaN value or distance and a doc without a facet row are not counted (the
 *     reference panics or reads out of bounds on them).
 * Counts are over every match: the reference counts only the docs it visits under Topk pruning and, for multi-term Union queries, only
 * the docs of blocks with one valid term.  out: HOST [n_queries][sum of caps], cap = length (VALUES) or n_ranges (RANGES), requests in
 * order; n_out: HOST [n_queries][n_req] entries written per request.  bases: HOST [n_queries][number of POINT requests][2] (lat, lon), or
 * NULL when no request is on a POINT facet.  The value histograms take n_queries x (sum over VALUES requests of the facet's largest id
 * + 1) x 4 bytes; the batch runs in query chunks within a 256 MiB workspace per search context (one query above it: SSB_E_UNSUPPORTED).
 * Not on a handle with a communicator (SSB_E_UNSUPPORTED).
 *   STRINGSET16 / 32 facets take VALUES only (RANGES: SSB_E_INVALID) and need ssb_set_facet_string_sets (else SSB_E_STATE): a doc counts
 *     once under every member occurrence of its combination (search.rs:3615-3640), `value` is a MEMBER id, [rank_lo, rank_hi) a member-id
 *     interval, ties go to the smaller id, and the histogram takes n_values words. */
enum { SSB_FACET_COUNT_VALUES = 0, SSB_FACET_COUNT_RANGES = 1 };
#define SSB_MAX_FACET_RANGES 256u
#define SSB_MAX_FACET_LENGTH 1024u
#define SSB_MAX_FACET_REQUESTS 16u
typedef struct {
    uint32_t facet;                  /* index into ssb_set_facets' fields                                                */
    uint32_t kind;                   /* SSB_FACET_COUNT_*                                                                */
    uint32_t length;                 /* VALUES: at most this many (id, count); 0 = not collected                         */
    uint32_t has_prefix;             /* VALUES: restrict to value-order ranks in [rank_lo, rank_hi)                      */
    uint32_t rank_lo, rank_hi;
    uint32_t n_ranges;               /* RANGES: 1 .. SSB_MAX_FACET_RANGES                                                */
    uint32_t unit;                   /* RANGES on a POINT facet: SSB_UNIT_*                                              */
    const uint64_t* range_starts;    /* RANGES: HOST [n_ranges]                                                          */
} ssb_facet_request;
typedef struct { uint32_t value; uint32_t pad; uint64_t count; } ssb_facet_count;   /* value: id (VALUES) or range index (RANGES) */
int32_t ssb_search_lexical_facets(ssb_index* ix, const ssb_lex_batch* q, const ssb_facet_request* req, uint32_t n_req,
                                  const double* bases, ssb_facet_count* out, uint32_t* n_out);
/* The empty query (Search::search("", enable_empty_query = true, ..): search_iterator_shard iterator.rs:316-358 with add_result.rs:95-338,
 * and search_iterator_index iterator.rs:360-413): a batch of filter-only queries over every document.
 *   Batch: q supplies n_queries and the facet filters (filter_offsets / filters / filter_set_values, exactly as for ssb_search_lexical).
 *     Terms must be absent: term_offsets NULL or all zero (HOST array), else SSB_E_INVALID.  field_masks and query_type are ignored.
 *   Documents: the doc ids of the added lexical levels (level << 16 | 0 .. n_docs - 1) outside the delete set — the reference's
 *     0 .. indexed_doc_count when every level but the last is full, which is how the reference writes its levels.  A doc passes when every
 *     filter of its query accepts it (is_facet_filter); a doc without a facet row fails every filter.
 *   Order: the criteria are those of ssb_search_lexical_sorted_ex (the same validation, 64-bit budget and Point bases).  A LEADING `_score`
 *     orders by the doc id in its own direction, as the index route does (deviation: with a filter the reference's shard route keeps the
 *     first k docs in heap order); a later `_score` compares equal scores and ends the comparison.  Ties on every criterion, and no
 *     criterion at all, go to the doc id DESCENDING (min_heap.rs:535-536, search.rs:3575-3579).  Hits carry score 0.
 *   Counts: count_total is exact for Count / TopkCount (unspecified for Topk); Count ignores the sort.  An unfiltered Count costs no kernel.
 *   k up to SSB_K_LIMIT (paged like ssb_search_lexical).  Not on a handle with a communicator (SSB_E_UNSUPPORTED). */
int32_t ssb_search_empty(ssb_index* ix, const ssb_lex_batch* q, const ssb_sort_criterion* sort, uint32_t n_sort, const double* bases,
                         uint32_t k, uint32_t result_type, ssb_hit* hits, uint32_t* n_hits, uint64_t* count_total);
/* Facet counts of the empty query (get_index_string_facets_shard, index.rs:4441-4569): not counts over matches but the index-wide
 * per-value counters ingest keeps.  One result set for the call: out HOST [sum of caps] (caps as for ssb_search_lexical_facets),
 * n_out HOST [n_req].
 *   VALUES (String16 / String32): the `length` ids with the most facet rows, over EVERY row given to ssb_set_facets (no filter, deleted docs
 *     included, as the reference's counters are never decremented); count descending, then id ascending; has_prefix restricts to a
 *     value-order rank interval as in ssb_search_lexical_facets.  Deviation: a row whose id is 0 because its doc had no value is counted
 *     under id 0.  STRINGSET16 / 32: every row counts under each member occurrence of its combination (index.rs:4531-4550), over rows
 *     rather than the ingest counters as for String facets.
 *   RANGES: validated, n_out = 0 (the reference returns no range facets for the empty query).
 * Not on a handle with a communicator (SSB_E_UNSUPPORTED). */
int32_t ssb_search_empty_facets(ssb_index* ix, const ssb_facet_request* req, uint32_t n_req, ssb_facet_count* out, uint32_t* n_out);
/* queries: [n_queries, dims] f32; Cosine: normalised by the callee (search.rs:1464-1475).  score = dot
 * (Dot/Cosine) or -Σ(q-x)² (Euclidean) exactly as Result.score in vector.rs:1489. */
int32_t ssb_search_vector(ssb_index* ix, const float* queries, uint32_t n_queries, uint32_t k,
                          ssb_hit* hits, uint32_t* n_hits);
/* search_vector_shard with all of its arguments (vector.rs:1105-1115): `similarity_threshold: Option<f32>` (pre-mapped as in
 * TopK::new, vector.rs:388-399: (2t-1)*16129 for Dot/Cosine, -t for Euclidean; hits scoring below it are dropped), queries as
 * f32 or — ScalarQuantizationI8 indexes only — as the int8 codes the reference's server holds after quantize_f32_to_i8
 * (search.rs:1477-1490).  ext: [n_queries * k] or NULL (vb fields: level_id, vector_score post-map vector.rs:1495-1499, source);
 * observed: [n_queries] or NULL (observed_vector_count: every record under AnnMode::All).  Rows that share a doc id (one vector
 * per chunk) are collapsed to the best-scoring one, as TopK::push does (vector.rs:436-470). */
enum { SSB_QFMT_F32 = 0, SSB_QFMT_I8 = 1 };
/* AnnMode (vector_similarity.rs:43-66) — which IVF clusters of each level are searched (vector.rs:1300-1392): per (query, level) the
 * query is scored against every cluster's medoid, the n_probe best clusters (score desc, cluster id asc) whose medoid score is not below
 * the pre-mapped cluster threshold are scanned, the others are skipped.  observed = the vectors in the selected clusters. */
enum { SSB_ANN_ALL = 0, SSB_ANN_NPROBE = 1, SSB_ANN_SIMILARITY_THRESHOLD = 2, SSB_ANN_NPROBE_SIMILARITY_THRESHOLD = 3 };
typedef struct {
    const void* queries;          /* [n_queries, dims] f32 or i8, host or device                              */
    uint32_t n_queries, k;
    uint32_t query_format;        /* SSB_QFMT_*                                                               */
    uint32_t has_threshold;       /* 0 = None                                                                 */
    float    similarity_threshold;
    uint32_t ann_mode;            /* SSB_ANN_* (0 = All: exhaustive)                                          */
    uint32_t n_probe;             /* Nprobe / NprobeSimilaritythreshold                                       */
    float    cluster_threshold;   /* Similaritythreshold / NprobeSimilaritythreshold (pre-mapped like similarity_threshold) */
} ssb_vec_query;
int32_t ssb_search_vector_ex(ssb_index* ix, const ssb_vec_query* q, ssb_hit* hits, uint32_t* n_hits, ssb_hit_ext* ext,
                             uint64_t* observed);
/* ssb_search_vector_ex with a field filter per query (search_vector_shard, vector.rs:1226-1238, 1411-1412).  field_masks: HOST array
 * [n_queries] or NULL; bit f = indexed field f is in the query's filter, 0 = no filter (the bits of ssb_lex_batch.field_masks).  A row
 * whose field is not in a non-zero mask is neither scored nor counted for that query.  A non-zero mask on an index without field ids
 * -> SSB_E_STATE.  On a field-tagged index ext.field_id / chunk_id are the field and chunk of the doc's best row among those passing the
 * mask (the earliest in record order on equal scores), here and in ssb_search_vector_ex; observed of a masked query counts the rows in
 * scope (every row, or the selected clusters' rows) whose field passes. */
int32_t ssb_search_vector_fields(ssb_index* ix, const ssb_vec_query* q, const uint32_t* field_masks, ssb_hit* hits,
                                 uint32_t* n_hits, ssb_hit_ext* ext, uint64_t* observed);
/* SearchMode::Hybrid: both searches with length k, RRF (k=0.6, rank from 0), sort, truncate to k.
 * hits: [n_queries * k].  On an index whose vector rows carry field ids, q->field_masks filters the vector half as well
 * (search.rs:1702-1731); on other indexes it filters the lexical half only. */
int32_t ssb_search_hybrid(ssb_index* ix, const ssb_lex_batch* q, const float* queries, uint32_t k,
                          ssb_hit* hits, uint32_t* n_hits);

/* RRF on two host lists (search.rs:1962-2035): out capacity n_lex+n_vec; sorted score desc, doc id asc. */
int32_t ssb_rrf_fuse(const ssb_hit* lex, uint32_t n_lex, const ssb_hit* vec, uint32_t n_vec,
                     ssb_hit* out, uint32_t* n_out);

/* ---- device-resident variants (multi-GPU merge, benchmarking with inputs already in HBM) ----------- */
/* Packed top-k keys: u64 = (ordered(score) << 32) | (0xFFFFFFFF - doc_id); larger = better.  keys_out is a
 * DEVICE buffer [n_queries * 32]; entry j of query i is its j-th best or 0 if none.  Asynchronous on the
 * index stream; ssb_sync() waits. */
int32_t ssb_search_vector_keys(ssb_index* ix, const float* queries, uint32_t n_queries, uint32_t k,
                               uint64_t* keys_out_dev);
int32_t ssb_search_lexical_keys(ssb_index* ix, const ssb_lex_batch* q, uint32_t k, uint32_t result_type,
                                uint64_t* keys_out_dev, uint64_t* count_total_dev);
/* merge `n_lists` key lists per query ([n_lists][n_queries][32], device) into hits (host) */
int32_t ssb_merge_keys(ssb_index* ix, const uint64_t* keys_dev, uint32_t n_lists, uint32_t n_queries,
                       uint32_t k, ssb_hit* hits, uint32_t* n_hits);
/* ---- sharded index over several GPUs (SURVEY.md §8e): one process per GPU, each handle holds a contiguous range of levels ---- */
/* The reference fans a query out over its shards and concatenates + sorts their results (search.rs:1637-1743, 1875-1928, 2097-2106).
 * Here every rank calls the same ssb_search_* with the same queries; once a communicator is set the library itself enqueues the
 * exchange on the search stream — ncclAllGather of the packed top-k keys + the G*k -> k merge, ncclAllReduce of the match
 * counts; hybrid: both lists are merged over the shards first and fused (RRF) afterwards — and every rank returns the GLOBAL
 * result.  Searches on a handle with a communicator are serialised (collectives must be issued in the same order everywhere).
 * NCCL is resolved at run time (the copy already loaded in the process, libnccl.so.2, or $SSB_NCCL_LIB). */
#define SSB_COMM_ID_BYTES 128
int32_t ssb_comm_unique_id(uint8_t* id128);                       /* ncclGetUniqueId; rank 0 calls it and ships the bytes to the others */
int32_t ssb_comm_init(ssb_index* ix, const uint8_t* id128, uint32_t rank, uint32_t world);   /* collective: ncclCommInitRank      */
int32_t ssb_comm_attach(ssb_index* ix, void* nccl_comm, uint32_t rank, uint32_t world);      /* borrow the caller's ncclComm_t      */
int32_t ssb_comm_destroy(ssb_index* ix);
/* collective: install the index-wide document frequencies (idf uses the df of the whole index, search.rs:3225-3230; the commit
 * already received the global N and length sum).  After it, scores equal those of an unsharded index bit for bit. */
int32_t ssb_lexical_sync_df(ssb_index* ix);

int32_t ssb_sync(ssb_index* ix);
/* the CUDA stream the index launches on (cudaStream_t as void*), for event timing */
void*   ssb_stream(ssb_index* ix);
/* run all further work of this index on a caller-owned stream (e.g. the stream NCCL collectives are enqueued
 * on, so the per-GPU top-k -> all-gather -> merge chain needs no host synchronisation).  The value is used
 * as a cudaStream_t as is (NULL = the CUDA legacy default stream); SSB_OWN_STREAM restores the index's own
 * stream. */
#define SSB_OWN_STREAM ((void*)(intptr_t)-1)
int32_t ssb_set_stream(ssb_index* ix, void* cuda_stream);

/* ---- statistics of the last search_* call (for roofline accounting) -------------------------------- */
typedef struct {
    uint64_t kernel_launches;     /* kernels launched by the last call                                   */
    uint64_t algorithmic_bytes;   /* SURVEY.md §8(d) bytes the call's kernels had to move                 */
    uint64_t h2d_bytes, d2h_bytes;
    uint64_t postings_visited;    /* lexical: driver postings enumerated after pruning                    */
    uint64_t probes;              /* lexical: membership probes into other lists                          */
    uint64_t items_processed;     /* lexical: (query, block) work items executed                          */
    uint64_t items_skipped;       /* lexical: work items pruned by block-max                              */
    uint64_t dominant_kernel_ns;  /* CUDA-event duration of the call's dominant kernel (scan / scoring)   */
    uint64_t scan_bytes_read;     /* vector: bytes the scan (+ refine) kernels stream from HBM by construction */
    uint64_t filter_fallbacks;    /* vector, host-facing calls: queries of the filter scan that took the exact fallback scan */
    uint64_t reserved[1];
} ssb_stats;
int32_t ssb_last_stats(const ssb_index* ix, ssb_stats* out);

#ifdef __cplusplus
}
#endif
#endif
