// bm25.h — lexical (BM25) index in HBM + batched query execution.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>

#include "common.cuh"
#include "facets.h"

namespace ssb {

// growable device buffer (grow = new allocation + D2D copy of the used prefix)
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t cap = 0;   // elements
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    int32_t reserve(size_t n, size_t used, cudaStream_t st, bool exact = false) {
        if (n <= cap) return SSB_OK;
        size_t nc = cap ? cap : 1024;
        while (nc < n) nc += nc / 2 + 1024;
        if (exact) nc = n;
        T* q = nullptr;
        cudaError_t e = cudaMalloc(&q, nc * sizeof(T));
        if (e != cudaSuccess) {
            cudaGetLastError();
            nc = n;   // fall back to the exact size
            e = cudaMalloc(&q, nc * sizeof(T));
            if (e != cudaSuccess) { cudaGetLastError(); set_error("cudaMalloc(%zu bytes) failed: %s", nc * sizeof(T), cudaGetErrorString(e)); return SSB_E_NOMEM; }
        }
        if (used && p) {
            e = cudaMemcpyAsync(q, p, used * sizeof(T), cudaMemcpyDeviceToDevice, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
            if (e != cudaSuccess) { cudaFree(q); set_error("DevBuf grow copy failed: %s", cudaGetErrorString(e)); return SSB_E_CUDA; }
        }
        if (p) { cudaStreamSynchronize(st); cudaFree(p); }
        p = q; cap = nc;
        return SSB_OK;
    }
};

inline bool is_device_ptr(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// scoped device temporary (freed on every exit path, including SSB_CUDA_TRY early returns)
template <typename T>
struct DevTmp {
    T* p = nullptr;
    DevTmp() = default;
    DevTmp(const DevTmp&) = delete;
    DevTmp& operator=(const DevTmp&) = delete;
    ~DevTmp() { if (p) cudaFree(p); }
    cudaError_t alloc(size_t n) { return cudaMalloc(&p, (n ? n : 1) * sizeof(T)); }
    T* release() { T* q = p; p = nullptr; return q; }
};

struct LexLevel {
    uint32_t level_id, n_docs, n_terms;
    uint64_t post_base;            // offset of this level's postings in the arenas
    uint32_t n_post;
    uint64_t* d_term_keys;         // [n_terms]
    uint32_t* d_posting_offsets;   // [n_terms+1]
};

// One 32-byte DRAM sector of a dense list's probe structure: the membership words of 128 consecutive doc ids, and per word the
// number of postings before it (rank, low 16 bits of meta) and the largest fp16 bound among its postings (high 16 bits): a probe
// learns presence, the posting's index and a tight score bound from ONE sector.
struct BmSec { uint64_t w[2]; uint32_t meta[2]; uint32_t pad[2]; };
static_assert(sizeof(BmSec) == 32, "BmSec must be one 32-byte sector");

// device view handed to the kernels (all pointers device)
struct LexView {
    const uint64_t* dict_keys; uint32_t n_terms;
    const uint32_t* term_first;   // [n_terms+1] entry ranges
    const float* term_idf;        // [n_terms]
    const uint32_t* term_df;      // [n_terms] (global df)
    const uint32_t* e_level;      // [n_entries] local level index, ascending within a term
    const uint64_t* e_off;        // posting offset in the arenas
    const uint32_t* e_count;
    const float* e_maxcomp;       // block-max basis: max tf*(K+1)/(tf+cache[len]) over the list
    const uint32_t* e_bitmap;     // index into bm_* or 0xFFFFFFFF
    const uint32_t* post;         // stream arena: id16 | bound16<<16 (fp16 bits of the posting's score component, rounded UP)
    const uint32_t* pay;          // payload arena, same index: tf16 | doclen_byte<<16 (read for exact scores only)
    const float* comp;            // component arena, same index: tf*(K+1)/(tf+cache[len]) as f32 (the exact score is idf * comp)
    const uint64_t* bm_words;     // [n_bitmaps][1024] plain membership words (count algebra, NOT lists)
    const BmSec* bm;              // [n_bitmaps][512] sector-packed membership + rank + per-word bound (scoring probes)
    const uint8_t* bm_q8;         // [n_bitmaps][1024] coarse bound per 64-doc word: ceil(word maximum / q8_step), 0 = no posting
    float q8_step;
    const uint32_t* level_ids;    // [n_levels]
    uint32_t n_levels;
    const float* cache;           // [256] bm25_component_cache
    float k1p;                    // K + 1
    // several indexed fields (get_bm25f_multiterm_multifield, add_result.rs:1226-1262): per posting n_fields payloads / exact components;
    // comp[] / the fp16 bounds then hold an UPPER BOUND of sum_f boost[f] * comp_f and every query takes the generic path (fast_t = 0)
    const uint32_t* payf;         // [n_postings][n_fields] tf16 | doclen_byte << 16 of field f (tf 0 = term not in that field)
    const float* compf;           // [n_postings][n_fields] exact component of field f (0 = absent)
    uint32_t n_fields;            // 1 = single field (payf / compf unused)
    uint32_t fast_t;              // queries with <= fast_t live terms take the record path (FAST_T, or 0 with several fields)
    float boost[4];               // indexed_schema_vec[f].boost
    // delete set (shard.delete_hashset, add_result.rs:3435): null = no deleted docs
    const uint32_t* del_slot;     // [65536] level_id -> bitmap slot or 0xFFFFFFFF
    const uint64_t* del_words;    // [n_slots][1024]
    const uint32_t* del_docs;     // [n_del] deleted doc ids, ascending
    uint32_t n_del;
    // facet columns (ssb_set_facets): order-preserving 64-bit keys, [n_facets][facet_rows]; row = doc id - facet_first_doc
    const uint64_t* facet_keys;
    uint64_t facet_rows;
    uint32_t facet_first_doc;
    uint32_t n_facets;
    // term positions (phrase queries): positions[lvl_pos_base[lv] + pos_off[posting] .. + tf), ascending; null = the index holds none
    const uint16_t* positions;
    const uint32_t* pos_off;      // [n_postings] offset of the posting's positions relative to its level's base
    const uint64_t* lvl_pos_base; // [n_levels]
    // per batch (filled by search_keys): the queries' facet filters, QueryPlan.filt_first / n_filt index into them
    const FiltDev* filt;
    const uint64_t* filt_sets;
};

// device-resident delete set shared by the lexical and the vector path
// h_docs: the deleted doc ids, ascending, on the host (the live-doc count of the empty query)
struct DeleteSet {
    uint32_t* d_slot = nullptr; uint64_t* d_words = nullptr; uint32_t* d_docs = nullptr; uint32_t n = 0;
    std::vector<uint32_t> h_docs;
    void release() { cudaFree(d_slot); cudaFree(d_words); cudaFree(d_docs); d_slot = nullptr; d_words = nullptr; d_docs = nullptr; n = 0; h_docs.clear(); }
};

struct QTerm { uint32_t first, n; float idf; uint32_t df; };
// fast: the query takes the record path (lex_score / lex_count): <= fast_t live terms and no facet filter; otherwise lex_generic
struct QueryPlan { QTerm t[SSB_MAX_QUERY_TERMS]; QTerm tn[SSB_MAX_NOT_TERMS]; uint32_t n_live, n_items, n_recs, n_not; uint32_t filt_first, n_filt, fast, field_mask /* field_filter: bit f = indexed field f, 0 = none */;
                   // phrase query: token i of the phrase is unique term phr[i] (index into t[]) and sits at start + phr_off[i] (i, plus 1 per
                   // earlier bigram and 2 per earlier trigram key on an index with n-gram lists); n_phr = 0: not a phrase
                   uint8_t phr[SSB_MAX_QUERY_TERMS]; uint8_t phr_off[SSB_MAX_QUERY_TERMS]; uint32_t n_phr, pad[3]; };

// One (query, level) record, built by lex_plan for queries with <= 4 live terms; 128 bytes = one cache line.
// Slots are in QUERY order (scores are summed in query order, add_result.rs:1450-1452); cnt == 0 marks a term
// that has no postings in this level.
struct LvSlot { uint32_t off_lo; uint32_t offhi_cnt /* (off >> 32) << 20 | cnt */; uint32_t bmi; float ub; };
struct LvRec {
    uint32_t docbase;   // level_id << 16
    uint32_t meta;      // see REC_* below
    float bound;        // in-query-order sum of the present terms' block-max contributions
    uint32_t lv;        // local level index (generic path: directory lookups)
    LvSlot t[4];
    float S[4];         // OR: S[p] = in-order sum of ub over slots with MAXSCORE rank >= p.      AND: S[0] = bound
    float R[4];         // OR: R[p] = in-order sum of ub over slots with MAXSCORE rank >  p.      AND: R[0] = sum over slots != driver
    float idf[4];
};
static_assert(sizeof(LvRec) == 128, "LvRec must be one 128-byte line");
// meta bit fields
//   [0:3)   n_pres   number of present slots
//   [3:11)  perm     MAXSCORE order: 2 bits per rank p -> slot        (ub desc, slot asc; present slots only)
//   [11:19) rank     2 bits per slot -> MAXSCORE rank
//   [19:21) and_drv  AND: slot of the shortest list
//   [21:29) cperm    count order: 2 bits per count-rank -> slot      (cnt desc, slot asc; present slots only)
//   [29:32) n_live   live terms of the query (== n_pres for AND records)

struct LexStats { uint64_t postings_visited, probes, items_processed, items_skipped, recs_processed, dense_words; };
// the statistics of an empty-query call (ssb_last_stats): launches, the bytes the scan staged, (query, tile) pairs evaluated / skipped,
// the CUDA-event time of the scan (or histogram) kernels
struct EmptyStats { uint64_t launches, alg_bytes, items_processed, items_skipped, kernel_ns; };

// Per-call scratch of one search context (api.cu keeps a pool of them: concurrent searches on one index do not share any).
struct LexWorkspace {
    DevBuf<QueryPlan> plans; DevBuf<LvRec> recs; DevBuf<uint16_t> item_start;
    DevBuf<uint64_t> theta;   // [n][2]: the 64-bit θ of an unsorted batch in the first n words, the 128-bit θ {hi, lo} of a sorted one
    DevBuf<int> lock; DevBuf<uint64_t> count;
    DevBuf<uint32_t> ctr;     // [0] score / [2] count / [3] generic work counters, [1] max_items, [4] any query with > 4 live terms
    DevBuf<uint32_t> qoff; DevBuf<uint64_t> qkeys; DevBuf<uint8_t> qflags; DevBuf<LexStats> stats;
    DevBuf<uint32_t> foff, fmask; DevBuf<FiltDev> filt; DevBuf<uint64_t> fsets;   // facet filters and field masks of the batch
    DevBuf<double> bases;     // sorted batches with a POINT criterion: [n_queries][2] bases, staged before search_keys
    // facet count calls (facet_counts): the value / range histograms of one query chunk (FACET_HIST_BYTES), the call's requests, range
    // starts and Point bases, the selected counts of the chunk, the plan's scratch list and the call's work counters {postings, dense
    // words, counted docs}
    DevBuf<uint32_t> fhist; DevBuf<FacetReqDev> freq; DevBuf<uint64_t> fstarts, fstats;
    DevBuf<uint64_t> fcsr;    // [2 * n_req]: per request the StringSet facet's CSR (set offsets, member ids) as addresses, 0 = none
    DevBuf<double> fbases; DevBuf<ssb_facet_count> fout; DevBuf<uint32_t> fnout; DevBuf<uint64_t> fglist;
    // empty-query calls (empty_query.cu): the call's tiles in scan order and its work counters (EQ_STAT_*)
    DevBuf<uint2> etiles; DevBuf<unsigned long long> estats;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;   // recorded around lex_score when set
};

class LexIndex {
public:
    explicit LexIndex(cudaStream_t st, int n_sms, uint32_t max_batch) : st_(st), n_sms_(n_sms), max_batch_(max_batch) {}
    ~LexIndex();
    int32_t add_level(const ssb_level_desc* d);
    int32_t set_fields(uint32_t n_fields, const float* boosts);   // before the first level
    int32_t set_ngram_config(uint32_t similarity, uint32_t df_rule);   // before the first level
    // add_level + the level's n-gram data (ssb_lexical_add_level_ngrams): component tfs of the n-gram postings and the df bytes of the
    // n-gram keys, kept until commit computes their components
    int32_t add_level_ngrams(const ssb_level_desc* d, const ssb_level_ngrams* ng);
    bool has_ngrams() const { return !ng_segs_.empty(); }
    // ssb_lexical_add_level: add_level, refusing keys with low bits set once the index holds n-gram lists (they would be scored with the
    // n-gram keys' dictionary idf 1.0)
    int32_t add_level_plain(const ssb_level_desc* d);
    int32_t commit(uint64_t n_docs, uint64_t len_sum);
    int32_t dict_size(uint64_t* n) const { *n = n_terms_; return SSB_OK; }
    int32_t dict_export(uint64_t* keys, uint32_t* dfs, uint64_t cap) const;
    int32_t set_global_df(const uint64_t* keys, const uint32_t* dfs, uint64_t n);
    // keys_out_dev: [n_queries][32]; count_dev: [n_queries] or null.  Asynchronous on `st`; thread-safe for concurrent
    // calls with distinct workspaces (the committed index is immutable).
    // ceil_dev: optional [n_queries] exclusive key ceilings (paging: only hits ranked after that key; 0 = none left)
    // sort: a sorted batch (prepare_sort); keys_out_dev then holds [n_queries][32] 128-bit keys {hi, lo} (not masked: entries >= k may
    // hold further candidates, callers read the first k) and ceil_dev [n_queries][2]
    int32_t search_keys(LexWorkspace& ws, cudaStream_t st, const ssb_lex_batch* q, uint32_t k, uint32_t result_type,
                        uint64_t* keys_out_dev, uint64_t* count_dev, uint64_t* launches, const uint64_t* ceil_dev = nullptr,
                        const SortDev* sort = nullptr) const;
    // sort_of_criteria against the index's facets, then the check that the facet rows cover every level
    int32_t prepare_sort(const ssb_sort_criterion* crit, uint32_t n, bool has_bases, SortDev* out, bool* sorted) const;
    // a sort with a POINT criterion: copy the host bases [nq][2] into the workspace and point sort->bases at them
    static int32_t stage_sort_bases(LexWorkspace& ws, cudaStream_t st, const double* bases, uint32_t nq, SortDev* sort);
    // ssb_search_lexical_facets: the batch's facet counts into the host arrays out / n_out (synchronous).  *kernel_ns: the CUDA-event time
    // of lex_facets summed over the query chunks; *alg_bytes: list bytes + 8 B of column key per counted doc and request
    int32_t facet_counts(LexWorkspace& ws, cudaStream_t st, const ssb_lex_batch* q, const ssb_facet_request* req, uint32_t n_req,
                         const double* bases, ssb_facet_count* out, uint32_t* n_out, uint64_t* launches, uint64_t* kernel_ns,
                         uint64_t* alg_bytes) const;
    // ssb_search_empty (empty_query.cu): the filter-only batch q over every live doc of the levels, in the order of `sort` — prepared by
    // prepare_sort, at least one criterion (the caller puts `_id` descending in place of none).  keys_out_dev: [n_queries][32] 128-bit keys
    // {hi, lo}, lo = pack_key(0, 0xFFFFFFFF - doc): ties by doc id descending (unmasked: callers read the first k); count_dev: [n_queries]
    // or null, exact unless Topk; ceil_dev: [n_queries][2] exclusive key ceilings of a further page, or null.  Asynchronous on st except
    // for the host checks; the scan's time is recorded between ws.ev0 and ws.ev1.
    int32_t search_empty(LexWorkspace& ws, cudaStream_t st, const ssb_lex_batch* q, uint32_t k, uint32_t result_type, const SortDev& sort,
                         uint64_t* keys_out_dev, uint64_t* count_dev, const uint64_t* ceil_dev, EmptyStats* stats) const;
    // ssb_search_empty_facets (synchronous): the top values of String facets over every facet row; RANGES requests give n_out 0
    int32_t empty_facets(LexWorkspace& ws, cudaStream_t st, const ssb_facet_request* req, uint32_t n_req, ssb_facet_count* out,
                         uint32_t* n_out, EmptyStats* stats) const;
    // the docs of the levels outside the delete set: the count of an unfiltered empty query (kept by commit and refresh_live_docs)
    uint64_t live_docs() const { return live_docs_; }
    void refresh_live_docs();                    // after the delete set changed
    bool committed() const { return committed_; }
    void set_stream(cudaStream_t st) { st_ = st; }   // load-time stream (add_level / commit)
    void set_deleted(const DeleteSet* d) { del_ = d; }
    void set_facets(const FacetSet* f) { facets_ = f; }
    static LexStats read_stats(const LexWorkspace& ws, cudaStream_t st);
    uint64_t n_postings() const { return n_post_; }
    const std::vector<uint64_t>& host_keys() const { return h_dict_keys_; }
    const std::vector<uint32_t>& host_local_df() const { return h_local_df_; }   // df of THIS shard's levels (set_global_df does not touch it)
    uint32_t n_levels() const { return (uint32_t)levels_.size(); }

private:
    struct Batch { LexView v; uint32_t nq, phrase, qt_eff; bool filtered, geo; };
    // the start of search_keys and facet_counts: the batch checks, stage_batch and the one lex_plan launch (lex_plan<true> when `sort` is
    // set), which zeroes glist ([n_queries][32] keys, [n_queries][32][2] when sorted).  topk_only: a Topk batch, whose queries plan
    // without counts unless the batch has a POINT filter or sort criterion (b->geo).  b->nq = 0: an empty batch, nothing staged or launched
    int32_t plan_batch(LexWorkspace& ws, cudaStream_t st, const ssb_lex_batch* q, bool topk_only, const SortDev* sort, uint64_t* glist,
                       Batch* b, uint64_t* launches) const;
    int32_t ensure_workspace(LexWorkspace& ws, cudaStream_t st, uint32_t nq, uint32_t total_terms) const;
    int32_t stage_filters(LexWorkspace& ws, cudaStream_t st, const ssb_lex_batch* q, LexView& v, bool* any, bool* geo_any) const;
    // what every lexical batch starts with: the per-query term checks, the workspace, the terms, the facet filters (*filtered, *geo: a
    // POINT filter) and the field masks (*fmask_dev, null = none) on the device; v: the view with the batch's filters
    int32_t stage_batch(LexWorkspace& ws, cudaStream_t st, const ssb_lex_batch* q, LexView& v, bool* filtered, bool* geo,
                        const uint32_t** fmask_dev) const;
    cudaStream_t st_;
    int n_sms_;
    uint32_t max_batch_;
    bool committed_ = false;
    std::vector<LexLevel> levels_;
    DevBuf<uint32_t> post_, pay_;
    DevBuf<float> comp_;
    // positions of every posting (phrase queries): one arena in posting order + per posting the offset inside its level
    DevBuf<uint16_t> positions_; DevBuf<uint32_t> pos_off_; uint64_t n_positions_ = 0; int has_positions_ = -1 /* -1 unknown, 0 none, 1 all levels */;
    std::vector<uint64_t> h_lvl_pos_base_; uint64_t* d_lvl_pos_base_ = nullptr;
    uint32_t n_fields_ = 1; float boosts_[4] = {1.f, 1.f, 1.f, 1.f};
    DevBuf<uint32_t> payf_; DevBuf<float> compf_;   // several indexed fields: [n_post][n_fields]
    // n-gram lists (add_level_ngrams): one segment per (n-gram key, level) with its postings' range in the arenas and its component tfs
    // in h_ng_tf_ ([n][3], host memory: only commit needs them); the df bytes of every level, resolved at commit by ng_rule_
    struct NgSeg { uint64_t key; uint64_t post_off; uint64_t tf_off; uint32_t cnt; uint8_t dfb[3]; };
    std::vector<NgSeg> ng_segs_; std::vector<uint16_t> h_ng_tf_; uint64_t n_ng_tf_ = 0;
    bool plain_lowbit_ = false;                     // a level added without n-gram data carried keys with low bits set
    uint32_t lex_sim_ = SSB_LEXSIM_BM25F_PROXIMITY, ng_rule_ = SSB_NGRAM_DF_FIRST_LEVEL;
    std::vector<uint64_t> h_ng_keys_;               // sorted unique n-gram keys (their dictionary idf stays 1.0)
    float q8_step_ = 0.f;                           // coarse bound step set by commit: Q8_STEP, larger when n-gram components exceed K + 1
    uint64_t n_post_ = 0;
    // committed structures
    uint64_t n_docs_ = 0, len_sum_ = 0;
    uint32_t n_terms_ = 0, n_entries_ = 0, n_bitmaps_ = 0;
    uint64_t* d_dict_keys_ = nullptr; uint32_t* d_term_first_ = nullptr; float* d_term_idf_ = nullptr; uint32_t* d_term_df_ = nullptr;
    uint32_t* d_e_level_ = nullptr; uint64_t* d_e_off_ = nullptr; uint32_t* d_e_count_ = nullptr; float* d_e_maxcomp_ = nullptr; uint32_t* d_e_bitmap_ = nullptr;
    uint64_t* d_bm_words_ = nullptr; BmSec* d_bm_ = nullptr; uint8_t* d_bm_q8_ = nullptr;
    uint32_t* d_level_ids_ = nullptr; float* d_cache_ = nullptr;
    std::vector<uint64_t> h_dict_keys_; std::vector<uint32_t> h_term_df_, h_local_df_;
    const DeleteSet* del_ = nullptr;
    const FacetSet* facets_ = nullptr;
    uint64_t live_docs_ = 0;
    void free_committed();
    int32_t commit_ngrams(uint64_t n_docs);
    void ngram_idf_one(std::vector<float>& idf) const;
    LexView view() const;
};

// bm25.cu: facet_select over the value / range histograms of nq queries (hist [nq][hist_words]) -> out [nq][out_stride], n_out [nq][n_req]
int32_t launch_facet_select(const FacetSet& fs, const FacetReqDev* req, uint32_t n_req, const uint32_t* hist, uint32_t hist_words, uint32_t nq,
                            ssb_facet_count* out, uint32_t out_stride, uint32_t* n_out, cudaStream_t st);

// loader.cu: the reference's on-disk files -> index
struct VectorLevel { uint32_t level_id; std::vector<uint16_t> ids; std::vector<float> rows; std::vector<uint32_t> cluster_counts;
                     std::vector<uint8_t> fields; std::vector<uint32_t> chunks; /* keep_fields only */ };
int32_t load_index_bin(LexIndex* lex, const uint8_t* bytes, uint64_t len, const ssb_index_bin_params* prm, uint64_t* n_docs_out, bool ngrams = false);
int32_t inspect_index_bin(const uint8_t* bytes, uint64_t len, const ssb_index_bin_params* prm, uint64_t out[8]);
int32_t inspect_index_bin_ngrams(const uint8_t* bytes, uint64_t len, const ssb_index_bin_params* prm, uint64_t out[8]);
int32_t parse_vector_bin(const uint8_t* bytes, uint64_t len, uint32_t dims, std::vector<VectorLevel>& out, bool keep_fields = false);

}  // namespace ssb
