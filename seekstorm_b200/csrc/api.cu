// api.cu — the extern "C" ABI of libseekstorm_b200.so (include/seekstorm_b200.h): handle, search-context pool, search entry
// points with their paging, hybrid RRF, shard merge.  No torch types; CUDA runtime only.
#include <stdarg.h>
#include <string.h>
#include <algorithm>
#include <condition_variable>
#include <exception>
#include <memory>
#include <mutex>
#include <new>
#include <shared_mutex>
#include <vector>

#include "bm25.h"
#include "comm.h"
#include "common.cuh"
#include "vec_index.h"

namespace ssb {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap; va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int32_t encode_tmap_2d_f32(CUtensorMap* out, const void* base, uint64_t inner_elems, uint64_t rows,
                           uint64_t row_pitch_bytes, uint32_t box_inner, uint32_t box_rows, int swizzle128) {
    return encode_tmap_2d(out, base, 4, inner_elems, rows, row_pitch_bytes, box_inner, box_rows, swizzle128 ? 128 : 0);
}

int32_t encode_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes, uint64_t inner_elems, uint64_t rows,
                       uint64_t row_pitch_bytes, uint32_t box_inner, uint32_t box_rows, int swizzle_bytes) {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr; cudaDriverEntryPointQueryResult qr;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr);
        if (e != cudaSuccess || !p || qr != cudaDriverEntryPointSuccess) { set_error("cuTensorMapEncodeTiled unavailable"); return SSB_E_CUDA; }
        fn = (EncodeTiledFn)p;
    }
    cuuint64_t gdim[2] = {inner_elems, rows};
    cuuint64_t gstr[1] = {row_pitch_bytes};
    cuuint32_t box[2] = {box_inner, box_rows};
    cuuint32_t estr[2] = {1, 1};
    const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE;
    CUresult r = fn(out, elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim, gstr, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed: %d", (int)r); return SSB_E_CUDA; }
    return SSB_OK;
}

}  // namespace ssb

using namespace ssb;

// One search context = one CUDA stream + every per-call workspace.  Concurrent ssb_search_* calls on one handle each take a
// context from the pool (SURVEY.md §8b: "handles are thread-safe for concurrent search_* calls — a stream/workspace pool");
// the committed index data is immutable and shared.
struct SearchCtx {
    cudaStream_t st = nullptr;       // stream this context launches on (its own, or the caller's after ssb_set_stream)
    cudaStream_t own_st = nullptr;
    LexWorkspace lex;
    VecWorkspace vec;
    DevBuf<uint64_t> ceil, keys_a, keys_b, counts, gather;   // paging ceilings, result pages, counts, shard all-gather
    std::vector<uint64_t> h_ceil, h_keys_a, h_keys_b, h_counts;
    ssb_stats stats{};
    cudaEvent_t ev0 = nullptr, ev1 = nullptr; bool ev_used = false, last_lex = false;
    ~SearchCtx() {
        if (own_st) cudaStreamSynchronize(own_st);
        if (ev0) cudaEventDestroy(ev0);
        if (ev1) cudaEventDestroy(ev1);
        if (own_st) cudaStreamDestroy(own_st);
    }
};

constexpr size_t SSB_MAX_CTX = 16;

struct ssb_index {
    int device = 0;
    int n_sms = 0;
    cudaStream_t load_st = nullptr;   // load-time stream (add_level / commit)
    // searches hold `rw` shared, index mutation exclusive (mirrors the reference's RwLock around the shard, commit.rs:142)
    std::shared_mutex rw;
    std::mutex pool_mu; std::condition_variable pool_cv;
    std::vector<std::unique_ptr<SearchCtx>> pool; std::vector<SearchCtx*> free_ctx;
    bool ext_stream_set = false; cudaStream_t ext_stream = nullptr;   // ssb_set_stream: every search runs on the caller's stream (one context)
    std::mutex stats_mu; SearchCtx* last_ctx = nullptr; ssb_stats last_stats{};
    LexIndex* lex = nullptr;
    VecIndex vec;
    DeleteSet del;                    // shard.delete_hashset mirrored on the device (ssb_set_deleted)
    FacetSet facets;                  // the shard's facet file as one key column per facet (ssb_set_facets)
    ShardComm comm;                   // set: this handle is one shard of a `world`-way sharded index (one process per GPU)
};

namespace {

// RAII lease of a search context
struct CtxLease {
    ssb_index* ix; SearchCtx* c = nullptr;
    explicit CtxLease(ssb_index* i) : ix(i) {}
    // block = false: give up (c stays null, SSB_OK) instead of waiting when every context is busy
    int32_t acquire(bool block = true) {
        std::unique_lock<std::mutex> g(ix->pool_mu);
        // one context when the caller owns the stream, and when searches contain collectives (every rank must issue them in the
        // same order: concurrent searches on one communicator would interleave them)
        const size_t cap = (ix->ext_stream_set || ix->comm.active()) ? 1 : SSB_MAX_CTX;
        for (;;) {
            if (!ix->free_ctx.empty()) { c = ix->free_ctx.back(); ix->free_ctx.pop_back(); break; }
            if (ix->pool.size() < cap) {
                std::unique_ptr<SearchCtx> n(new (std::nothrow) SearchCtx());
                if (!n) { set_error("out of host memory"); return SSB_E_NOMEM; }
                if (cudaStreamCreateWithFlags(&n->own_st, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); set_error("stream create failed"); return SSB_E_CUDA; }
                cudaEventCreate(&n->ev0); cudaEventCreate(&n->ev1);
                n->lex.ev0 = n->vec.ev0 = n->ev0; n->lex.ev1 = n->vec.ev1 = n->ev1;
                c = n.get(); ix->pool.push_back(std::move(n));
                break;
            }
            if (!block) return SSB_OK;
            ix->pool_cv.wait(g);
        }
        c->st = ix->ext_stream_set ? ix->ext_stream : c->own_st;
        c->stats = ssb_stats{}; c->ev_used = false; c->last_lex = false; c->vec.fb_state = nullptr;
        return SSB_OK;
    }
    ~CtxLease() {
        if (!c) return;
        { std::lock_guard<std::mutex> g(ix->stats_mu); ix->last_ctx = c; ix->last_stats = c->stats; }
        { std::lock_guard<std::mutex> g(ix->pool_mu); ix->free_ctx.push_back(c); }
        ix->pool_cv.notify_one();
    }
};

// every extern "C" body runs inside this guard: no exception (thrust::system_error, std::bad_alloc, ...) crosses the C boundary
#define SSB_API_BEGIN try {
#define SSB_API_END                                                                                              \
    } catch (const std::bad_alloc&) { cudaGetLastError(); set_error("out of memory (host or device)"); return SSB_E_NOMEM; \
    } catch (const std::exception& e) { cudaGetLastError(); set_error("internal error: %s", e.what()); return SSB_E_CUDA;   \
    } catch (...) { cudaGetLastError(); set_error("internal error: unknown exception"); return SSB_E_CUDA; }

// Sharded index: all-gather every rank's [nq][32] key lists and merge them (G*k -> k with the canonical tie rule; the reference
// concatenates the shard results and sorts, search.rs:1875-1928, 2097-2106).  In place; identical result on every rank.
int32_t shard_merge(ssb_index* ix, SearchCtx& c, uint64_t* keys_dev, uint32_t nq) {
    if (!ix->comm.active() || nq == 0) return SSB_OK;
    const size_t n = (size_t)nq * LIST;
    SSB_TRY(c.gather.reserve(n * ix->comm.world, 0, c.st));
    SSB_TRY(comm_all_gather_u64(ix->comm, keys_dev, c.gather.p, n, c.st));
    SSB_TRY(vec::launch_merge_lists(c.gather.p, ix->comm.world, nq, keys_dev, c.st));
    c.stats.kernel_launches += 2;
    return SSB_OK;
}
int32_t shard_sum_counts(ssb_index* ix, SearchCtx& c, uint64_t* counts_dev, uint32_t nq) {
    if (!ix->comm.active() || nq == 0 || !counts_dev) return SSB_OK;
    SSB_TRY(comm_all_reduce_sum_u64(ix->comm, counts_dev, nq, c.st));   // result_count_total = sum over shards (search.rs:1875-1940)
    c.stats.kernel_launches += 1;
    return SSB_OK;
}

// Paging state of the host-facing search calls (k > SSB_K_MAX, or de-duplication of multi-chunk documents).  W = words per key:
// 1 = the 64-bit (score, doc) keys, 2 = the 128-bit keys {hi, lo} of a sorted lexical search, lo = pack_key(score, doc) with its score
// half inverted when score_inv (`_score` ascending).  doc_desc: lo = pack_key(0, 0xFFFFFFFF - doc) of an empty-query search (ties by doc
// id descending).
template <int W>
struct PageState {
    SearchCtx& c; uint32_t nq, k; ssb_hit* hits; uint32_t* n_hits; std::vector<uint32_t> cnt; std::vector<uint8_t> open; bool dedup, score_inv, doc_desc;
    PageState(SearchCtx& c_, uint32_t nq_, uint32_t k_, ssb_hit* h, uint32_t* n, bool dedup_ = false, bool score_inv_ = false, bool doc_desc_ = false)
        : c(c_), nq(nq_), k(k_), hits(h), n_hits(n), cnt(nq_, 0), open(nq_, 1), dedup(dedup_), score_inv(score_inv_), doc_desc(doc_desc_) {
        c.h_ceil.assign(((size_t)nq_ + 256) * W, 0);
    }
    // consume one [nq][32] page that was fetched with `kk` results per query; returns true if any query wants another page
    bool append(const uint64_t* keys, uint32_t kk) {
        bool more = false;
        for (uint32_t q = 0; q < nq; q++) {
            uint64_t* ceil = &c.h_ceil[(size_t)q * W];
            if (!open[q]) { for (int w = 0; w < W; w++) ceil[w] = 0; continue; }   // exhausted or complete on an earlier page
            uint32_t seen = 0; const uint64_t* last = nullptr;
            for (uint32_t j = 0; j < kk && cnt[q] < k; j++) {
                const uint64_t* key = keys + ((size_t)q * LIST + j) * W;
                bool empty = true;
                for (int w = 0; w < W; w++) empty = empty && key[w] == 0;
                if (empty) break;
                seen++; last = key;
                const uint64_t lo = key[W - 1];
                const uint64_t doc = doc_desc ? (uint32_t)lo : key_doc(lo);
                if (dedup) {
                    bool dup = false;
                    for (uint32_t i = 0; i < cnt[q]; i++) dup = dup || hits[(size_t)q * k + i].doc_id == doc;
                    if (dup) continue;
                }
                ssb_hit& h = hits[(size_t)q * k + cnt[q]];
                h.doc_id = doc; h.score = key_score(score_inv ? lo ^ 0xFFFFFFFF00000000ull : lo); h.pad = 0;
                cnt[q]++;
            }
            // another page only if this one was full (else the list is exhausted) and the query still lacks results
            open[q] = seen == kk && cnt[q] < k;
            for (int w = 0; w < W; w++) ceil[w] = open[q] ? last[w] : 0;        // 0 = nothing left below
            more = more || open[q];
        }
        return more;
    }
    uint32_t next_page_k() const {   // results to fetch per query on the next page
        if (dedup) return SSB_K_MAX;
        uint32_t need = 0;
        for (uint32_t q = 0; q < nq; q++) if (open[q]) need = std::max(need, k - cnt[q]);
        return need < SSB_K_MAX ? need : SSB_K_MAX;
    }
    int32_t upload_ceilings() {
        SSB_TRY(c.ceil.reserve(((size_t)nq + 256) * W, 0, c.st));
        SSB_CUDA_TRY(cudaMemcpyAsync(c.ceil.p, c.h_ceil.data(), ((size_t)nq + 256) * W * 8, cudaMemcpyHostToDevice, c.st));
        c.stats.h2d_bytes += (uint64_t)nq * W * 8;
        return SSB_OK;
    }
    void finish() {
        for (uint32_t q = 0; q < nq; q++) {
            for (uint32_t j = cnt[q]; j < k; j++) { ssb_hit& h = hits[(size_t)q * k + j]; h.doc_id = 0; h.score = 0.f; h.pad = 0; }
            if (n_hits) n_hits[q] = cnt[q];
        }
    }
};

// Field-tagged vector rows and a sharded handle exclude each other (the field filter and the best-row step are not built across
// shards): refused when such rows are added to a sharded handle (what = "rows") and when a handle holding them is sharded ("vector rows")
int32_t refuse_tagged_sharded(const char* who, const char* what, bool tagged, bool sharded) {
    if (!tagged || !sharded) return SSB_OK;
    set_error("%s: field-tagged %s on a sharded index are not supported", who, what);
    return SSB_E_UNSUPPORTED;
}

inline bool hit_better(const ssb_hit& a, const ssb_hit& b) { return a.score > b.score || (a.score == b.score && a.doc_id < b.doc_id); }

void finish_stats(ssb_index* ix, SearchCtx& c) {
    if (c.ev_used) {
        float ms = 0.f;
        if (cudaEventSynchronize(c.ev1) == cudaSuccess && cudaEventElapsedTime(&ms, c.ev0, c.ev1) == cudaSuccess)
            c.stats.dominant_kernel_ns = (uint64_t)((double)ms * 1e6);
        else cudaGetLastError();
    }
}

// read back the page the last fetch left in c.keys_a ([nq][32] keys of W words); with it, after a vector filter scan, the count of
// queries that took the exact fallback
template <int W>
int32_t read_page(SearchCtx& c, uint32_t nq) {
    SSB_CUDA_TRY(cudaMemcpyAsync(c.h_keys_a.data(), c.keys_a.p, (size_t)nq * LIST * W * 8, cudaMemcpyDeviceToHost, c.st));
    uint32_t n_fb = 0;
    if (c.vec.fb_state) SSB_CUDA_TRY(cudaMemcpyAsync(&n_fb, c.vec.fb_state, 4, cudaMemcpyDeviceToHost, c.st));
    SSB_CUDA_TRY(cudaStreamSynchronize(c.st));
    c.stats.filter_fallbacks += n_fb;
    c.stats.d2h_bytes += (uint64_t)nq * LIST * W * 8;
    return SSB_OK;
}

// The pages after the first one of a host-facing search (k > SSB_K_MAX, or de-duplication): the first page, read back with k1 results
// per query, is appended; then, while a query wants more, fetch(kk) enqueues into c.keys_a the next kk keys per query strictly below
// the ceilings in c.ceil (the last key of the previous page: keys are a total order).  At most 4096 pages in all.
template <int W, class Fetch>
int32_t page_rest(SearchCtx& c, PageState<W>& ps, uint32_t k1, Fetch fetch) {
    bool more = ps.append(c.h_keys_a.data(), k1);
    for (uint32_t page = 1; more && page < 4096; page++) {
        const uint32_t kk = ps.next_page_k();
        SSB_TRY(ps.upload_ceilings());
        SSB_TRY(fetch(kk));
        SSB_TRY(read_page<W>(c, ps.nq));
        more = ps.append(c.h_keys_a.data(), kk);
    }
    ps.finish();
    return SSB_OK;
}

// host-facing vector search: paging beyond 32 results, de-duplication, optional threshold
int32_t search_vector_host(ssb_index* ix, SearchCtx& c, const void* queries, bool queries_i8, uint32_t nq, uint32_t k, ssb_hit* hits, uint32_t* n_hits,
                           const IvfQuery* ivf = nullptr, const uint32_t* fmask_host = nullptr) {
    SSB_TRY(c.keys_a.reserve((size_t)nq * LIST, 0, c.st));
    c.h_keys_a.resize((size_t)nq * LIST);
    const bool dedup = ix->vec.dup_docs();
    PageState<1> ps(c, nq, k, hits, n_hits, dedup);
    const auto fetch = [&](uint32_t kk, const uint64_t* ceil) -> int32_t {
        SSB_TRY(ix->vec.search_keys(c.vec, c.st, c.stats, &c.ev_used, queries, queries_i8, nq, kk, c.keys_a.p, ceil, ivf, fmask_host));
        return shard_merge(ix, c, c.keys_a.p, nq);
    };
    const uint32_t k1 = dedup ? SSB_K_MAX : (k < SSB_K_MAX ? k : SSB_K_MAX);
    SSB_TRY(fetch(k1, nullptr));
    if (ivf) {   // observed_vector_count = the vectors of the selected clusters (summed over the shards)
        SSB_TRY(shard_sum_counts(ix, c, c.vec.ivf_obs.p, nq));
        c.vec.h_obs.resize(nq);
        SSB_CUDA_TRY(cudaMemcpyAsync(c.vec.h_obs.data(), c.vec.ivf_obs.p, (size_t)nq * 8, cudaMemcpyDeviceToHost, c.st));
    }
    SSB_TRY(read_page<1>(c, nq));
    return page_rest(c, ps, k1, [&](uint32_t kk) { return fetch(kk, c.ceil.p); });
}

// host-facing lexical search: the first page of <= SSB_K_MAX hits with the counts, then Topk pages below the previous page's last key.
// W = 2: a sorted batch (sort), 128-bit keys.
template <int W>
int32_t search_lexical_host(ssb_index* ix, SearchCtx& c, const ssb_lex_batch* q, uint32_t k, uint32_t result_type, ssb_hit* hits, uint32_t* n_hits,
                            uint64_t* count_total, const SortDev* sort) {
    const uint32_t nq = q->n_queries;
    SSB_TRY(c.keys_a.reserve((size_t)nq * LIST * W, 0, c.st));
    SSB_TRY(c.counts.reserve(nq, 0, c.st));
    c.h_keys_a.resize((size_t)nq * LIST * W); c.h_counts.resize(nq);
    const bool want_hits = hits && k && result_type != SSB_RESULT_COUNT;
    const uint32_t k1 = k < SSB_K_MAX ? k : SSB_K_MAX;
    SSB_TRY(ix->lex->search_keys(c.lex, c.st, q, k1, result_type, c.keys_a.p, c.counts.p, &c.stats.kernel_launches, nullptr, sort));
    if (W == 1) SSB_TRY(shard_merge(ix, c, c.keys_a.p, nq));         // (sorted searches refuse a communicator)
    SSB_TRY(shard_sum_counts(ix, c, c.counts.p, nq));
    SSB_CUDA_TRY(cudaMemcpyAsync(c.h_counts.data(), c.counts.p, (size_t)nq * 8, cudaMemcpyDeviceToHost, c.st));
    c.stats.d2h_bytes += (uint64_t)nq * 8;
    SSB_TRY(read_page<W>(c, nq));
    c.ev_used = true;
    finish_stats(ix, c);                                        // the first page's scoring kernel is the one reported
    const LexStats ls = LexIndex::read_stats(c.lex, c.st);
    if (want_hits) {
        PageState<W> ps(c, nq, k, hits, n_hits, false, sort && sort->score_asc);
        // pages beyond the first 32 results: Topk search restricted to keys below the previous page's last key
        SSB_TRY(page_rest(c, ps, k1, [&](uint32_t kk) -> int32_t {
            SSB_TRY(ix->lex->search_keys(c.lex, c.st, q, kk, SSB_RESULT_TOPK, c.keys_a.p, nullptr, &c.stats.kernel_launches, c.ceil.p, sort));
            return W == 1 ? shard_merge(ix, c, c.keys_a.p, nq) : SSB_OK;
        }));
    } else if (n_hits) for (uint32_t i = 0; i < nq; i++) n_hits[i] = 0;
    if (count_total) for (uint32_t i = 0; i < nq; i++) count_total[i] = c.h_counts[i];
    c.stats.postings_visited = ls.postings_visited;
    // SURVEY.md §8(d) accounting with this layout's sizes: 4 B per streamed posting word, 16 B per probe (8 B bitmap word + 4 B
    // rank / word bound + 4 B component), 128 B per (query, level) record read, 8 B per bitmap word of the word-wise count paths;
    // the 1-byte coarse-table lookups of the stream filter are not counted
    c.stats.algorithmic_bytes = ls.postings_visited * 4 + ls.probes * 16 + ls.recs_processed * 128 + ls.dense_words * 8;
    c.stats.probes = ls.probes; c.stats.items_processed = ls.items_processed; c.stats.items_skipped = ls.items_skipped;
    return SSB_OK;
}

// host-facing empty-query search: the first page of <= SSB_K_MAX hits with the counts, then pages below the previous page's last key
int32_t search_empty_host(ssb_index* ix, SearchCtx& c, const ssb_lex_batch* q, uint32_t k, uint32_t result_type, ssb_hit* hits, uint32_t* n_hits,
                          uint64_t* count_total, const SortDev& sort) {
    const uint32_t nq = q->n_queries;
    SSB_TRY(c.keys_a.reserve((size_t)nq * LIST * 2, 0, c.st));
    SSB_TRY(c.counts.reserve(nq, 0, c.st));
    c.h_keys_a.resize((size_t)nq * LIST * 2); c.h_counts.resize(nq);
    const bool want_hits = hits && k && result_type != SSB_RESULT_COUNT;
    const uint32_t k1 = want_hits ? (k < SSB_K_MAX ? k : SSB_K_MAX) : 0;
    EmptyStats es{};
    SSB_TRY(ix->lex->search_empty(c.lex, c.st, q, k1, result_type, sort, c.keys_a.p, c.counts.p, nullptr, &es));
    SSB_CUDA_TRY(cudaMemcpyAsync(c.h_counts.data(), c.counts.p, (size_t)nq * 8, cudaMemcpyDeviceToHost, c.st));
    c.stats.d2h_bytes += (uint64_t)nq * 8;
    SSB_TRY(read_page<2>(c, nq));
    c.ev_used = true;
    finish_stats(ix, c);                                        // the first page's scan is the one reported
    if (want_hits) {
        PageState<2> ps(c, nq, k, hits, n_hits, false, false, true);
        SSB_TRY(page_rest(c, ps, k1, [&](uint32_t kk) {
            return ix->lex->search_empty(c.lex, c.st, q, kk, SSB_RESULT_TOPK, sort, c.keys_a.p, nullptr, c.ceil.p, &es);
        }));
    } else if (n_hits) for (uint32_t i = 0; i < nq; i++) n_hits[i] = 0;
    if (count_total) for (uint32_t i = 0; i < nq; i++) count_total[i] = c.h_counts[i];
    c.stats.kernel_launches += es.launches; c.stats.algorithmic_bytes = es.alg_bytes;
    c.stats.items_processed = es.items_processed; c.stats.items_skipped = es.items_skipped;
    return SSB_OK;
}

}  // namespace

extern "C" {

uint32_t ssb_abi_version(void) { return SSB_ABI_VERSION; }
const char* ssb_last_error(void) { return g_err; }

int32_t ssb_create(const ssb_config* cfg, ssb_index** out) {
    SSB_API_BEGIN
    if (!cfg || !out) { set_error("ssb_create: null argument"); return SSB_E_INVALID; }
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); set_error("no CUDA device visible: libseekstorm_b200 has no CPU fallback"); return SSB_E_NO_DEVICE; }
    if (cfg->device < 0 || cfg->device >= ndev) { set_error("device %d out of range (%d visible)", cfg->device, ndev); return SSB_E_INVALID; }
    if (cfg->vector_similarity > SSB_SIM_EUCLIDEAN) { set_error("bad vector_similarity"); return SSB_E_INVALID; }
    if (cfg->vector_kernel > SSB_VEC_KERNEL_TCGEN05_FILTER_N256_PAIR) { set_error("bad vector kernel"); return SSB_E_INVALID; }
    if (cfg->vector_quantization > SSB_QUANT_TURBO_I8) { set_error("bad vector_quantization"); return SSB_E_INVALID; }
    if (cfg->vector_quantization == SSB_QUANT_TURBO_I8 && cfg->vector_dims > 16384) { set_error("TurboQuantI8: vector_dims above 16384 unsupported"); return SSB_E_UNSUPPORTED; }
    SSB_CUDA_TRY(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    SSB_CUDA_TRY(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0) { set_error("device %d is sm_%d%d; this library is built for sm_90a (H100) only", cfg->device, prop.major, prop.minor); return SSB_E_UNSUPPORTED; }
    std::unique_ptr<ssb_index> ix(new (std::nothrow) ssb_index());
    if (!ix) { set_error("out of host memory"); return SSB_E_NOMEM; }
    ix->device = cfg->device;
    ix->n_sms = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&ix->load_st, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); set_error("stream create failed"); return SSB_E_CUDA; }
    ix->lex = new (std::nothrow) LexIndex(ix->load_st, ix->n_sms, cfg->max_batch ? cfg->max_batch : 4096);
    if (!ix->lex) { cudaStreamDestroy(ix->load_st); set_error("out of host memory"); return SSB_E_NOMEM; }
    ix->lex->set_deleted(&ix->del);
    ix->lex->set_facets(&ix->facets);
    ix->vec.init(*cfg, ix->n_sms, ix->load_st);
    ix->vec.set_deleted(&ix->del);
    *out = ix.release();
    return SSB_OK;
    SSB_API_END
}

int32_t ssb_destroy(ssb_index* ix) {
    SSB_API_BEGIN
    if (!ix) return SSB_OK;
    cudaSetDevice(ix->device);
    {
        std::unique_lock<std::shared_mutex> g(ix->rw);    // waits for searches in flight
        cudaStreamSynchronize(ix->load_st);
        ix->pool.clear();                                  // ~SearchCtx synchronises its stream
        delete ix->lex; ix->lex = nullptr;
        comm_destroy(ix->comm);
        ix->del.release();
        ix->facets.release();
        cudaStreamDestroy(ix->load_st);
    }
    delete ix;
    return SSB_OK;
    SSB_API_END
}

int32_t ssb_lexical_add_level(ssb_index* ix, const ssb_level_desc* level) {
    SSB_API_BEGIN
    if (!ix) { set_error("null index"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    if (level && (is_device_ptr(level->doc_ids) || is_device_ptr(level->term_keys))) SSB_CUDA_TRY(cudaDeviceSynchronize());   // inputs produced on another stream
    return ix->lex->add_level_plain(level);
    SSB_API_END
}

int32_t ssb_lexical_set_field_boosts(ssb_index* ix, uint32_t n_fields, const float* boosts) {
    SSB_API_BEGIN
    if (!ix) { set_error("null index"); return SSB_E_INVALID; }
    if (boosts && is_device_ptr(boosts)) { set_error("boosts must be host memory"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    return ix->lex->set_fields(n_fields, boosts);
    SSB_API_END
}

int32_t ssb_lexical_set_ngram_config(ssb_index* ix, uint32_t lexical_similarity, uint32_t df_level_rule) {
    SSB_API_BEGIN
    if (!ix) { set_error("null index"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    return ix->lex->set_ngram_config(lexical_similarity, df_level_rule);
    SSB_API_END
}

int32_t ssb_lexical_add_level_ngrams(ssb_index* ix, const ssb_level_desc* level, const ssb_level_ngrams* ngrams) {
    SSB_API_BEGIN
    if (!ix) { set_error("null index"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    if (ngrams && ix->comm.active()) { set_error("ssb_lexical_add_level_ngrams: n-gram lists on a sharded index are not supported"); return SSB_E_UNSUPPORTED; }
    if (level && (is_device_ptr(level->doc_ids) || is_device_ptr(level->term_keys))) SSB_CUDA_TRY(cudaDeviceSynchronize());   // inputs produced on another stream
    return ix->lex->add_level_ngrams(level, ngrams);
    SSB_API_END
}

int32_t ssb_lexical_commit(ssb_index* ix, uint64_t n_docs, uint64_t len_sum) {
    SSB_API_BEGIN
    if (!ix) { set_error("null index"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    return ix->lex->commit(n_docs, len_sum);
    SSB_API_END
}

int32_t ssb_lexical_dict_size(const ssb_index* ix, uint64_t* n) { if (!ix || !n) return SSB_E_INVALID; return ix->lex->dict_size(n); }
int32_t ssb_lexical_dict_export(const ssb_index* ix, uint64_t* keys, uint32_t* dfs, uint64_t cap) { if (!ix) return SSB_E_INVALID; return ix->lex->dict_export(keys, dfs, cap); }
int32_t ssb_lexical_set_global_df(ssb_index* ix, const uint64_t* keys, const uint32_t* dfs, uint64_t n) {
    SSB_API_BEGIN
    if (!ix || (n && (!keys || !dfs))) return SSB_E_INVALID;
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    return ix->lex->set_global_df(keys, dfs, n);
    SSB_API_END
}

// capacity hint: allocate the vector arenas for n_rows rows once instead of growing them level by level (growth = new
// allocation + device copy of everything loaded so far)
int32_t ssb_vector_reserve(ssb_index* ix, uint64_t n_rows) {
    SSB_API_BEGIN
    if (!ix) { set_error("null index"); return SSB_E_INVALID; }
    if (ix->vec.dims() == 0) { set_error("no vector index configured (vector_dims = 0)"); return SSB_E_STATE; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    return ix->vec.reserve(n_rows);
    SSB_API_END
}

}  // extern "C"

// one level (= one add call) of the vector index; cluster_counts = the level's IVF cluster table or null (one cluster).  n is only
// bounded by the loader (a level may hold one record per chunk, i.e. more than 64K).
static int32_t vector_add_level_impl(ssb_index* ix, uint32_t level_id, const float* rows, uint64_t row_stride, const uint16_t* local_ids,
                                     uint32_t n, uint32_t dims, const uint32_t* cluster_counts, uint32_t n_clusters,
                                     const uint8_t* field_ids = nullptr, const uint32_t* chunk_ids = nullptr) {
    SSB_API_BEGIN
    if (!ix || (n && !rows)) { set_error("ssb_vector_add_level: null argument"); return SSB_E_INVALID; }
    if (ix->vec.dims() == 0 || dims != ix->vec.dims()) { set_error("dims %u != configured vector_dims %u", dims, ix->vec.dims()); return SSB_E_INVALID; }
    if (cluster_counts) {
        if (is_device_ptr(cluster_counts)) { set_error("cluster_counts must be host memory"); return SSB_E_INVALID; }
        uint64_t sum = 0;
        for (uint32_t c = 0; c < n_clusters; c++) { if (cluster_counts[c] == 0) { set_error("empty cluster %u", c); return SSB_E_INVALID; } sum += cluster_counts[c]; }
        if (sum != n || (n && n_clusters == 0)) { set_error("cluster table covers %llu of %u rows", (unsigned long long)sum, n); return SSB_E_INVALID; }
        if (ix->vec.quant_i8() && n_clusters > 1) { set_error("IVF cluster tables need an f32 vector index"); return SSB_E_UNSUPPORTED; }
    }
    if (level_id >= 65536) { set_error("level_id must be < 65536 (doc id = level_id << 16 | local)"); return SSB_E_INVALID; }
    if (row_stride == 0) row_stride = dims;
    if (row_stride < dims) { set_error("row stride < dims"); return SSB_E_INVALID; }
    if ((field_ids == nullptr) != (chunk_ids == nullptr)) { set_error("ssb_vector_add_level_fields: field_ids and chunk_ids go together"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    return ix->vec.add_level(level_id, rows, row_stride, local_ids, n, cluster_counts, n_clusters, field_ids, chunk_ids);
    SSB_API_END
}

extern "C" {

int32_t ssb_vector_add_level(ssb_index* ix, uint32_t level_id, const float* rows, uint64_t row_stride, const uint16_t* local_ids,
                             uint32_t n, uint32_t dims) {
    if (n > 65536) { set_error("a level holds at most 65536 vectors"); return SSB_E_INVALID; }
    return vector_add_level_impl(ix, level_id, rows, row_stride, local_ids, n, dims, nullptr, 0);
}

int32_t ssb_vector_add_level_clustered(ssb_index* ix, uint32_t level_id, const float* rows, uint64_t row_stride, const uint16_t* local_ids,
                                       uint32_t n, uint32_t dims, const uint32_t* cluster_counts, uint32_t n_clusters) {
    if (n > 65536) { set_error("a level holds at most 65536 vectors"); return SSB_E_INVALID; }
    if (n && !cluster_counts) { set_error("ssb_vector_add_level_clustered: null cluster table"); return SSB_E_INVALID; }
    return vector_add_level_impl(ix, level_id, rows, row_stride, local_ids, n, dims, n ? cluster_counts : nullptr, n_clusters);
}

int32_t ssb_vector_add_level_fields(ssb_index* ix, uint32_t level_id, const float* rows, uint64_t row_stride, const uint16_t* local_ids,
                                    uint32_t n, uint32_t dims, const uint32_t* cluster_counts, uint32_t n_clusters,
                                    const uint8_t* field_ids, const uint32_t* chunk_ids) {
    if (n > 65536) { set_error("a level holds at most 65536 vectors"); return SSB_E_INVALID; }
    if (n && (!field_ids || !chunk_ids)) { set_error("ssb_vector_add_level_fields: null field_ids / chunk_ids"); return SSB_E_INVALID; }
    if (ix) SSB_TRY(refuse_tagged_sharded("ssb_vector_add_level_fields", "rows", true, ix->comm.active()));
    return vector_add_level_impl(ix, level_id, rows, row_stride, local_ids, n, dims, n ? cluster_counts : nullptr, n_clusters,
                                 n ? field_ids : nullptr, n ? chunk_ids : nullptr);
}

int32_t ssb_load_index_bin(ssb_index* ix, const void* bytes, uint64_t len, const ssb_index_bin_params* params, uint64_t* n_docs_out) {
    SSB_API_BEGIN
    if (!ix || !bytes || !params) { set_error("ssb_load_index_bin: null argument"); return SSB_E_INVALID; }
    if (is_device_ptr(bytes)) { set_error("ssb_load_index_bin: bytes must be host memory"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    return load_index_bin(ix->lex, (const uint8_t*)bytes, len, params, n_docs_out);
    SSB_API_END
}

int32_t ssb_index_bin_inspect(const void* bytes, uint64_t len, const ssb_index_bin_params* params, uint64_t out[8]) {
    SSB_API_BEGIN
    if (!bytes || !params || !out) { set_error("ssb_index_bin_inspect: null argument"); return SSB_E_INVALID; }
    return inspect_index_bin((const uint8_t*)bytes, len, params, out);
    SSB_API_END
}

int32_t ssb_load_index_bin_ngrams(ssb_index* ix, const void* bytes, uint64_t len, const ssb_index_bin_params* params, uint64_t* n_docs_out) {
    SSB_API_BEGIN
    if (!ix || !bytes || !params) { set_error("ssb_load_index_bin_ngrams: null argument"); return SSB_E_INVALID; }
    if (is_device_ptr(bytes)) { set_error("ssb_load_index_bin_ngrams: bytes must be host memory"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    if (ix->comm.active()) { set_error("ssb_load_index_bin_ngrams: n-gram lists on a sharded index are not supported"); return SSB_E_UNSUPPORTED; }
    return load_index_bin(ix->lex, (const uint8_t*)bytes, len, params, n_docs_out, true);
    SSB_API_END
}

int32_t ssb_index_bin_inspect_ngrams(const void* bytes, uint64_t len, const ssb_index_bin_params* params, uint64_t out[8]) {
    SSB_API_BEGIN
    if (!bytes || !params || !out) { set_error("ssb_index_bin_inspect_ngrams: null argument"); return SSB_E_INVALID; }
    return inspect_index_bin_ngrams((const uint8_t*)bytes, len, params, out);
    SSB_API_END
}

}  // extern "C"

// keep_fields: VectorHeader.field_id / chunk_id go through the field-tagged add (ssb_load_vector_bin_fields)
static int32_t load_vector_bin_impl(ssb_index* ix, const void* bytes, uint64_t len, uint64_t* n_vectors_out, bool keep_fields) {
    SSB_API_BEGIN
    if (!ix || !bytes) { set_error("ssb_load_vector_bin: null argument"); return SSB_E_INVALID; }
    if (is_device_ptr(bytes)) { set_error("ssb_load_vector_bin: bytes must be host memory"); return SSB_E_INVALID; }
    const uint32_t dims = ix->vec.dims();
    if (dims == 0) { set_error("ssb_load_vector_bin: the index has no vector_dims"); return SSB_E_STATE; }
    SSB_TRY(refuse_tagged_sharded("ssb_load_vector_bin_fields", "rows", keep_fields, ix->comm.active()));
    std::vector<VectorLevel> levels;
    SSB_TRY(parse_vector_bin((const uint8_t*)bytes, len, dims, levels, keep_fields));
    uint64_t total = 0;
    for (auto& vl : levels) {
        // a level may hold more than 64K records (one per chunk); its cluster table (IVF, vector.rs:1066-1094) rides along.  Empty clusters
        // cannot be probed (their medoid would be another cluster's record): such a table is dropped, the level becomes one cluster.
        bool ok = !vl.cluster_counts.empty() && !ix->vec.quant_i8();
        for (uint32_t c : vl.cluster_counts) ok = ok && c != 0;
        SSB_TRY(vector_add_level_impl(ix, vl.level_id, vl.rows.data(), dims, vl.ids.data(), (uint32_t)vl.ids.size(), dims,
                                      ok ? vl.cluster_counts.data() : nullptr, ok ? (uint32_t)vl.cluster_counts.size() : 0,
                                      keep_fields && !vl.ids.empty() ? vl.fields.data() : nullptr, keep_fields && !vl.ids.empty() ? vl.chunks.data() : nullptr));
        total += vl.ids.size();
    }
    if (n_vectors_out) *n_vectors_out = total;
    return SSB_OK;
    SSB_API_END
}

extern "C" {

int32_t ssb_load_vector_bin(ssb_index* ix, const void* bytes, uint64_t len, uint64_t* n_vectors_out) {
    return load_vector_bin_impl(ix, bytes, len, n_vectors_out, false);
}

int32_t ssb_load_vector_bin_fields(ssb_index* ix, const void* bytes, uint64_t len, uint64_t* n_vectors_out) {
    return load_vector_bin_impl(ix, bytes, len, n_vectors_out, true);
}

// shard.delete_hashset (index.rs:1594, filled by delete_document index.rs:5110): deleted docs are neither scored nor counted
// (add_result.rs:3435, vector.rs:1450-1451, union_count union.rs:975-1000).  Replaces the current set; n = 0 clears it.
int32_t ssb_set_deleted(ssb_index* ix, const uint64_t* doc_ids, uint64_t n) {
    SSB_API_BEGIN
    if (!ix || (n && !doc_ids)) { set_error("ssb_set_deleted: null argument"); return SSB_E_INVALID; }
    if (n >= (1ull << 31)) { set_error("ssb_set_deleted: too many doc ids"); return SSB_E_UNSUPPORTED; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    std::vector<uint32_t> docs(n);
    for (uint64_t i = 0; i < n; i++) {
        if (doc_ids[i] >> 32) { set_error("ssb_set_deleted: doc id %llu out of range", (unsigned long long)doc_ids[i]); return SSB_E_INVALID; }
        docs[i] = (uint32_t)doc_ids[i];
    }
    std::sort(docs.begin(), docs.end());
    docs.erase(std::unique(docs.begin(), docs.end()), docs.end());
    for (auto& c : ix->pool) cudaStreamSynchronize(c->own_st);
    ix->del.release();
    if (docs.empty()) { ix->lex->refresh_live_docs(); return SSB_OK; }
    std::vector<uint32_t> slot(65536, 0xFFFFFFFFu);
    uint32_t n_slots = 0;
    for (uint32_t d : docs) if (slot[d >> 16] == 0xFFFFFFFFu) slot[d >> 16] = n_slots++;
    std::vector<uint64_t> words((size_t)n_slots * 1024, 0ull);
    for (uint32_t d : docs) words[(size_t)slot[d >> 16] * 1024 + ((d & 0xFFFFu) >> 6)] |= 1ull << (d & 63u);
    SSB_CUDA_TRY(cudaMalloc(&ix->del.d_slot, 65536 * 4));
    SSB_CUDA_TRY(cudaMalloc(&ix->del.d_words, words.size() * 8));
    SSB_CUDA_TRY(cudaMalloc(&ix->del.d_docs, docs.size() * 4));
    SSB_CUDA_TRY(cudaMemcpy(ix->del.d_slot, slot.data(), 65536 * 4, cudaMemcpyHostToDevice));
    SSB_CUDA_TRY(cudaMemcpy(ix->del.d_words, words.data(), words.size() * 8, cudaMemcpyHostToDevice));
    SSB_CUDA_TRY(cudaMemcpy(ix->del.d_docs, docs.data(), docs.size() * 4, cudaMemcpyHostToDevice));
    ix->del.n = (uint32_t)docs.size();
    ix->del.h_docs = std::move(docs);
    ix->lex->refresh_live_docs();
    return SSB_OK;
    SSB_API_END
}

int32_t ssb_set_facets(ssb_index* ix, const void* rows, uint64_t first_doc_id, uint64_t n_docs, uint32_t row_bytes,
                       const ssb_facet_field* fields, uint32_t n_fields) {
    SSB_API_BEGIN
    if (!ix) { set_error("ssb_set_facets: null index"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    SSB_CUDA_TRY(cudaDeviceSynchronize());        // searches may run on a caller-owned stream (ssb_set_stream): nothing may still read the old columns
    return ix->facets.set_columns(rows, first_doc_id, n_docs, row_bytes, fields, n_fields, ix->load_st);
    SSB_API_END
}

int32_t ssb_set_facet_value_order(ssb_index* ix, uint32_t facet, const uint32_t* rank_of_id, uint32_t n_ids) {
    SSB_API_BEGIN
    if (!ix || (n_ids && !rank_of_id)) { set_error("ssb_set_facet_value_order: null argument"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    FacetSet& fs = ix->facets;
    if (!fs.n_facets) { set_error("ssb_set_facet_value_order: no facets (ssb_set_facets)"); return SSB_E_STATE; }
    if (facet >= fs.n_facets) { set_error("ssb_set_facet_value_order: facet %u of %u", facet, fs.n_facets); return SSB_E_INVALID; }
    const uint32_t type = fs.types[facet];
    if (!facet_is_string(type)) { set_error("ssb_set_facet_value_order: facet %u is not a String16 / String32 facet", facet); return SSB_E_INVALID; }
    const uint64_t lim = type == SSB_FACET_STRING16 ? 65536ull : (1ull << 32);
    if (n_ids == 0 || n_ids > lim) { set_error("ssb_set_facet_value_order: n_ids must be in 1..%llu", (unsigned long long)lim); return SSB_E_INVALID; }
    for (uint32_t i = 0; i < n_ids; i++) if (rank_of_id[i] >= n_ids) { set_error("ssb_set_facet_value_order: rank %u of id %u is not below n_ids", rank_of_id[i], i); return SSB_E_INVALID; }
    SSB_CUDA_TRY(cudaDeviceSynchronize());        // searches on a caller-owned stream may still read the old order
    return fs.set_value_order(facet, rank_of_id, n_ids, ix->load_st);
    SSB_API_END
}

int32_t ssb_set_facet_string_sets(ssb_index* ix, uint32_t facet, const uint64_t* set_offsets, const uint32_t* members, uint32_t n_sets,
                                  uint32_t n_values) {
    SSB_API_BEGIN
    if (!ix || !set_offsets) { set_error("ssb_set_facet_string_sets: null argument"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    FacetSet& fs = ix->facets;
    if (!fs.n_facets) { set_error("ssb_set_facet_string_sets: no facets (ssb_set_facets)"); return SSB_E_STATE; }
    if (facet >= fs.n_facets) { set_error("ssb_set_facet_string_sets: facet %u of %u", facet, fs.n_facets); return SSB_E_INVALID; }
    if (!facet_is_stringset(fs.types[facet])) { set_error("ssb_set_facet_string_sets: facet %u is not a StringSet16 / StringSet32 facet", facet); return SSB_E_INVALID; }
    // the reference's ingest writes at most 65,535 combinations to a StringSet16 facet; the first-member ranks take 16 bits there
    const uint32_t lim = fs.types[facet] == SSB_FACET_STRINGSET16 ? 65535u : 0xFFFFFFFFu;
    if (n_sets > lim) { set_error("ssb_set_facet_string_sets: %u sets, at most %u on a StringSet16 facet", n_sets, lim); return SSB_E_INVALID; }
    if (n_sets == 0 || fs.max_key[facet] >= n_sets) { set_error("ssb_set_facet_string_sets: the column holds id %llu, n_sets is %u", (unsigned long long)fs.max_key[facet], n_sets); return SSB_E_INVALID; }
    if (set_offsets[0] != 0) { set_error("ssb_set_facet_string_sets: set_offsets[0] must be 0"); return SSB_E_INVALID; }
    for (uint32_t c = 0; c < n_sets; c++)
        if (set_offsets[c + 1] < set_offsets[c]) { set_error("ssb_set_facet_string_sets: set_offsets must ascend (set %u)", c); return SSB_E_INVALID; }
    if (set_offsets[n_sets] && !members) { set_error("ssb_set_facet_string_sets: null members"); return SSB_E_INVALID; }
    for (uint64_t j = 0; j < set_offsets[n_sets]; j++)
        if (members[j] >= n_values) { set_error("ssb_set_facet_string_sets: member id %u at %llu is not below n_values %u", members[j], (unsigned long long)j, n_values); return SSB_E_INVALID; }
    SSB_CUDA_TRY(cudaDeviceSynchronize());        // searches on a caller-owned stream may still read the old sets
    return fs.set_string_sets(facet, set_offsets, members, n_sets, n_values, ix->load_st);
    SSB_API_END
}

int32_t ssb_vector_set_turboquant_mask(ssb_index* ix, const float* seed_mask, uint32_t dim) {
    SSB_API_BEGIN
    if (!ix || !seed_mask) { set_error("ssb_vector_set_turboquant_mask: null argument"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    return ix->vec.set_turboquant_mask(seed_mask, dim);
    SSB_API_END
}

int32_t ssb_set_vector_kernel(ssb_index* ix, uint32_t kernel) {
    SSB_API_BEGIN
    if (!ix || kernel > SSB_VEC_KERNEL_TCGEN05_FILTER_N256_PAIR) { set_error("bad vector kernel"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    ix->vec.set_kernel(kernel);
    return SSB_OK;
    SSB_API_END
}

int32_t ssb_vector_count(const ssb_index* ix, uint64_t* n) { if (!ix || !n) return SSB_E_INVALID; *n = ix->vec.n_rows(); return SSB_OK; }

int32_t ssb_search_vector_keys(ssb_index* ix, const float* queries, uint32_t nq, uint32_t k, uint64_t* keys_out_dev) {
    SSB_API_BEGIN
    if (!ix || (nq && (!queries || !keys_out_dev))) { set_error("ssb_search_vector_keys: null argument"); return SSB_E_INVALID; }
    std::shared_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    CtxLease l(ix); SSB_TRY(l.acquire());
    SSB_TRY(ix->vec.search_keys(l.c->vec, l.c->st, l.c->stats, &l.c->ev_used, queries, false, nq, k, keys_out_dev));
    return shard_merge(ix, *l.c, keys_out_dev, nq);
    SSB_API_END
}

int32_t ssb_search_vector(ssb_index* ix, const float* queries, uint32_t nq, uint32_t k, ssb_hit* hits, uint32_t* n_hits) {
    SSB_API_BEGIN
    if (!ix || (nq && (!queries || !hits))) { set_error("ssb_search_vector: null argument"); return SSB_E_INVALID; }
    std::shared_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    if (nq == 0) return SSB_OK;
    if (k == 0 || k > SSB_K_LIMIT) { set_error("k must be in 1..%u", SSB_K_LIMIT); return SSB_E_UNSUPPORTED; }
    CtxLease l(ix); SSB_TRY(l.acquire());
    SSB_TRY(search_vector_host(ix, *l.c, queries, false, nq, k, hits, n_hits));
    finish_stats(ix, *l.c);
    return SSB_OK;
    SSB_API_END
}

}  // extern "C"

static int32_t search_vector_ex_impl(ssb_index* ix, const ssb_vec_query* vq, const uint32_t* field_masks, ssb_hit* hits, uint32_t* n_hits,
                                     ssb_hit_ext* ext, uint64_t* observed) {
    SSB_API_BEGIN
    if (!ix || !vq || (vq->n_queries && (!vq->queries || !hits))) { set_error("ssb_search_vector_ex: null argument"); return SSB_E_INVALID; }
    if (vq->query_format > SSB_QFMT_I8) { set_error("bad query_format"); return SSB_E_INVALID; }
    std::shared_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    const uint32_t nq = vq->n_queries, k = vq->k;
    if (nq == 0) return SSB_OK;
    const uint32_t* fm = nullptr;
    SSB_TRY(ix->vec.field_masks(field_masks, nq, "ssb_search_vector_fields", &fm));
    if (k == 0 || k > SSB_K_LIMIT) { set_error("k must be in 1..%u", SSB_K_LIMIT); return SSB_E_UNSUPPORTED; }
    CtxLease l(ix); SSB_TRY(l.acquire());
    std::vector<uint32_t> nh(nq, 0);
    const bool euclid = ix->vec.euclid();
    if (vq->ann_mode > SSB_ANN_NPROBE_SIMILARITY_THRESHOLD) { set_error("bad ann_mode"); return SSB_E_INVALID; }
    IvfQuery ivf{vq->ann_mode, vq->n_probe, 0.f};
    {   // the cluster threshold goes through the same pre-map as the result threshold (TopK::new, vector.rs:388-399)
        volatile float c2 = vq->cluster_threshold * 2.0f; volatile float c21 = c2 - 1.0f;
        ivf.thr = euclid ? -vq->cluster_threshold : c21 / (1.0f / 16129.0f);
    }
    const bool use_ivf = vq->ann_mode != SSB_ANN_ALL;
    SSB_TRY(search_vector_host(ix, *l.c, vq->queries, vq->query_format == SSB_QFMT_I8, nq, k, hits, nh.data(), use_ivf ? &ivf : nullptr, fm));
    finish_stats(ix, *l.c);
    // TopK::new (vector.rs:388-399): threshold pre-map (2t-1)*16129 for Dot/Cosine, -t for Euclidean; TopK::push (:421) rejects
    // score < threshold.  The hits are sorted by score, so dropping the tail is the same filter.
    volatile float t2 = vq->similarity_threshold * 2.0f; volatile float t21 = t2 - 1.0f;
    const float cut = euclid ? -vq->similarity_threshold : t21 / (1.0f / 16129.0f);
    for (uint32_t q = 0; q < nq; q++) {
        uint32_t n = nh[q];
        if (vq->has_threshold) {
            uint32_t m = 0;
            while (m < n && !(hits[(size_t)q * k + m].score < cut)) m++;
            for (uint32_t j = m; j < n; j++) hits[(size_t)q * k + j] = ssb_hit{0, 0.f, 0};
            n = m;
        }
        nh[q] = n;
        if (n_hits) n_hits[q] = n;
        if (observed) observed[q] = use_ivf ? l.c->vec.h_obs[q] : ix->vec.n_rows();   // AnnMode::All scores every record (observed_vector_count, vector.rs:420); else: the selected clusters' vectors
        if (ext) for (uint32_t j = 0; j < k; j++) {
            ssb_hit_ext& e = ext[(size_t)q * k + j];
            memset(&e, 0, sizeof(e));
            if (j >= n) continue;
            const ssb_hit& h = hits[(size_t)q * k + j];
            e.level_id = (uint32_t)(h.doc_id >> 16);           // vector.rs:1448 doc id = level << 16 | local
            volatile float sn = h.score * (1.0f / 16129.0f); volatile float s1 = sn + 1.0f;
            e.vector_score = euclid ? -h.score : s1 * 0.5f;     // vector.rs:1495-1499 (SIMILARITY_NORMALIZATION_64_I8 regardless of precision)
            e.cluster_score = euclid ? 0.f : 0.5f;              // no clustering (AnnMode::All, Clustering::None): cluster_score = 0 -> post-map 0.5 / -0
            e.source = SSB_SOURCE_VECTOR;
        }
    }
    if (fm && observed) SSB_TRY(ix->vec.masked_observed(l.c->vec, l.c->st, nq, fm, use_ivf, observed));
    // field-tagged rows: which field and chunk of each doc won (after the threshold: only the hits returned)
    if (ext && ix->vec.tagged()) SSB_TRY(ix->vec.best_rows(l.c->vec, l.c->st, l.c->stats, vq->queries, nq, k, hits, nh.data(), fm, ext));
    return SSB_OK;
    SSB_API_END
}

extern "C" {

int32_t ssb_search_vector_ex(ssb_index* ix, const ssb_vec_query* vq, ssb_hit* hits, uint32_t* n_hits, ssb_hit_ext* ext, uint64_t* observed) {
    return search_vector_ex_impl(ix, vq, nullptr, hits, n_hits, ext, observed);
}

int32_t ssb_search_vector_fields(ssb_index* ix, const ssb_vec_query* vq, const uint32_t* field_masks, ssb_hit* hits, uint32_t* n_hits,
                                 ssb_hit_ext* ext, uint64_t* observed) {
    return search_vector_ex_impl(ix, vq, field_masks, hits, n_hits, ext, observed);
}

int32_t ssb_search_lexical_keys(ssb_index* ix, const ssb_lex_batch* q, uint32_t k, uint32_t result_type, uint64_t* keys_out_dev,
                                uint64_t* count_dev) {
    SSB_API_BEGIN
    if (!ix || !q) { set_error("ssb_search_lexical_keys: null argument"); return SSB_E_INVALID; }
    std::shared_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    CtxLease l(ix); SSB_TRY(l.acquire());
    l.c->ev_used = true; l.c->last_lex = true;
    SSB_TRY(ix->lex->search_keys(l.c->lex, l.c->st, q, k, result_type, keys_out_dev, count_dev, &l.c->stats.kernel_launches));
    SSB_TRY(shard_merge(ix, *l.c, keys_out_dev, q->n_queries));
    return shard_sum_counts(ix, *l.c, count_dev, q->n_queries);
    SSB_API_END
}

int32_t ssb_search_lexical(ssb_index* ix, const ssb_lex_batch* q, uint32_t k, uint32_t result_type, ssb_hit* hits, uint32_t* n_hits,
                           uint64_t* count_total) {
    SSB_API_BEGIN
    if (!ix || !q || (q->n_queries && k && result_type != SSB_RESULT_COUNT && !hits)) { set_error("ssb_search_lexical: null argument"); return SSB_E_INVALID; }
    std::shared_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    if (q->n_queries == 0) return SSB_OK;
    if (k > SSB_K_LIMIT) { set_error("k=%u exceeds SSB_K_LIMIT=%u", k, SSB_K_LIMIT); return SSB_E_UNSUPPORTED; }
    CtxLease l(ix); SSB_TRY(l.acquire());
    return search_lexical_host<1>(ix, *l.c, q, k, result_type, hits, n_hits, count_total, nullptr);
    SSB_API_END
}

int32_t ssb_search_lexical_sorted(ssb_index* ix, const ssb_lex_batch* q, const ssb_sort_criterion* sort, uint32_t n_sort, uint32_t k, uint32_t result_type,
                                  ssb_hit* hits, uint32_t* n_hits, uint64_t* count_total) {
    return ssb_search_lexical_sorted_ex(ix, q, sort, n_sort, nullptr, k, result_type, hits, n_hits, count_total);
}

// bases: per-query (lat, lon) of a Point criterion (ResultSort.base = FacetValue::Point); NULL drops that criterion
int32_t ssb_search_lexical_sorted_ex(ssb_index* ix, const ssb_lex_batch* q, const ssb_sort_criterion* sort, uint32_t n_sort, const double* bases,
                                     uint32_t k, uint32_t result_type, ssb_hit* hits, uint32_t* n_hits, uint64_t* count_total) {
    SSB_API_BEGIN
    // ResultType::Count ignores the sort (search.rs:2498); k = 0 is Count (search.rs:2472-2478)
    if (result_type == SSB_RESULT_COUNT || k == 0) return ssb_search_lexical(ix, q, k, result_type, hits, n_hits, count_total);
    if (!ix || !q || (q->n_queries && !hits)) { set_error("ssb_search_lexical_sorted: null argument"); return SSB_E_INVALID; }
    std::shared_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    SortDev sd{}; bool sorted = false;
    SSB_TRY(ix->lex->prepare_sort(sort, n_sort, bases != nullptr, &sd, &sorted));
    if (sorted && ix->comm.active()) { set_error("ssb_search_lexical_sorted: sorted search across shards is not built"); return SSB_E_UNSUPPORTED; }
    if (q->n_queries == 0) return SSB_OK;
    if (k > SSB_K_LIMIT) { set_error("k=%u exceeds SSB_K_LIMIT=%u", k, SSB_K_LIMIT); return SSB_E_UNSUPPORTED; }
    CtxLease l(ix); SSB_TRY(l.acquire());
    if (!sorted) return search_lexical_host<1>(ix, *l.c, q, k, result_type, hits, n_hits, count_total, nullptr);   // "_score desc" = the default order
    SSB_TRY(LexIndex::stage_sort_bases(l.c->lex, l.c->st, bases, q->n_queries, &sd));
    return search_lexical_host<2>(ix, *l.c, q, k, result_type, hits, n_hits, count_total, &sd);
    SSB_API_END
}

// query_facets of Search::search (facet_count, add_result.rs:487-640): the facet counts of a lexical batch, next to its search
int32_t ssb_search_lexical_facets(ssb_index* ix, const ssb_lex_batch* q, const ssb_facet_request* req, uint32_t n_req,
                                  const double* bases, ssb_facet_count* out, uint32_t* n_out) {
    SSB_API_BEGIN
    if (!ix || !q) { set_error("ssb_search_lexical_facets: null argument"); return SSB_E_INVALID; }
    std::shared_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    if (ix->comm.active()) { set_error("ssb_search_lexical_facets: facet counts across shards are not built"); return SSB_E_UNSUPPORTED; }
    CtxLease l(ix); SSB_TRY(l.acquire());
    SearchCtx& c = *l.c;
    return ix->lex->facet_counts(c.lex, c.st, q, req, n_req, bases, out, n_out, &c.stats.kernel_launches, &c.stats.dominant_kernel_ns,
                                 &c.stats.algorithmic_bytes);
    SSB_API_END
}

// Search::search("", enable_empty_query = true, ..) on committed data: a batch of filter-only queries over every live doc of the levels
int32_t ssb_search_empty(ssb_index* ix, const ssb_lex_batch* q, const ssb_sort_criterion* sort, uint32_t n_sort, const double* bases, uint32_t k,
                         uint32_t result_type, ssb_hit* hits, uint32_t* n_hits, uint64_t* count_total) {
    SSB_API_BEGIN
    if (!ix || !q || (n_sort && !sort) || (q->n_queries && k && result_type != SSB_RESULT_COUNT && !hits)) { set_error("ssb_search_empty: null argument"); return SSB_E_INVALID; }
    if (result_type > SSB_RESULT_TOPKCOUNT) { set_error("ssb_search_empty: bad result_type"); return SSB_E_INVALID; }
    std::shared_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    if (ix->comm.active()) { set_error("ssb_search_empty: the empty query across shards is not built"); return SSB_E_UNSUPPORTED; }
    if (k > SSB_K_LIMIT) { set_error("k=%u exceeds SSB_K_LIMIT=%u", k, SSB_K_LIMIT); return SSB_E_UNSUPPORTED; }
    if (n_sort > SSB_MAX_SORT_CRITERIA) { set_error("ssb_search_empty: more than %u criteria", SSB_MAX_SORT_CRITERIA); return SSB_E_UNSUPPORTED; }
    // a leading `_score` orders by doc id in its own direction (the index route, iterator.rs:360-413); a later one compares the all-zero
    // scores and ends the comparison, ties then go to the larger doc id (min_heap.rs:535-536)
    ssb_sort_criterion crit[SSB_MAX_SORT_CRITERIA];
    for (uint32_t i = 0; i < n_sort; i++) crit[i] = sort[i];
    if (n_sort && crit[0].source == SSB_SORT_SCORE) crit[0].source = SSB_SORT_ID;
    SortDev sd{}; bool sorted = false;
    SSB_TRY(ix->lex->prepare_sort(crit, n_sort, bases != nullptr, &sd, &sorted));
    if (sd.n == 0) {                                            // no criterion: doc id descending
        const ssb_sort_criterion id_desc{SSB_SORT_ID, 0, SSB_SORT_DESCENDING, 0};
        SSB_TRY(ix->lex->prepare_sort(&id_desc, 1, false, &sd, &sorted));
    }
    if (q->n_queries == 0) return SSB_OK;
    CtxLease l(ix); SSB_TRY(l.acquire());
    if ((result_type == SSB_RESULT_COUNT || k == 0) && !(q->filter_offsets && q->filter_offsets[q->n_queries])) {
        if (!ix->lex->committed()) { set_error("search before ssb_lexical_commit"); return SSB_E_STATE; }
        for (uint32_t i = 0; i < q->n_queries; i++) {           // unfiltered counts: the live docs, no kernel
            if (count_total) count_total[i] = ix->lex->live_docs();
            if (n_hits) n_hits[i] = 0;
        }
        return SSB_OK;
    }
    SSB_TRY(LexIndex::stage_sort_bases(l.c->lex, l.c->st, bases, q->n_queries, &sd));
    return search_empty_host(ix, *l.c, q, k, result_type, hits, n_hits, count_total, sd);
    SSB_API_END
}

int32_t ssb_search_empty_facets(ssb_index* ix, const ssb_facet_request* req, uint32_t n_req, ssb_facet_count* out, uint32_t* n_out) {
    SSB_API_BEGIN
    if (!ix) { set_error("ssb_search_empty_facets: null argument"); return SSB_E_INVALID; }
    std::shared_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    if (ix->comm.active()) { set_error("ssb_search_empty_facets: facet counts across shards are not built"); return SSB_E_UNSUPPORTED; }
    CtxLease l(ix); SSB_TRY(l.acquire());
    SearchCtx& c = *l.c;
    EmptyStats es{};
    SSB_TRY(ix->lex->empty_facets(c.lex, c.st, req, n_req, out, n_out, &es));
    c.stats.kernel_launches = es.launches; c.stats.algorithmic_bytes = es.alg_bytes; c.stats.dominant_kernel_ns = es.kernel_ns;
    return SSB_OK;
    SSB_API_END
}

int32_t ssb_rrf_fuse(const ssb_hit* lex, uint32_t n_lex, const ssb_hit* vec, uint32_t n_vec, ssb_hit* out, uint32_t* n_out) {
    SSB_API_BEGIN
    // search.rs:1962-2035: k = 0.6, rank from 0 over each list sorted by score desc; then :2097-2106 sort desc.
    if ((n_lex && !lex) || (n_vec && !vec) || !out) { set_error("ssb_rrf_fuse: null argument"); return SSB_E_INVALID; }
    const float kf = 0.6f;
    uint32_t n = 0;
    for (uint32_t i = 0; i < n_lex; i++) {
        volatile float denom = kf + (float)i; float s = 1.0f / denom;
        uint32_t j = 0; for (; j < n; j++) if (out[j].doc_id == lex[i].doc_id) break;
        if (j == n) { out[n].doc_id = lex[i].doc_id; out[n].score = s; out[n].pad = 0; n++; } else out[j].score = s;
    }
    for (uint32_t i = 0; i < n_vec; i++) {
        volatile float denom = kf + (float)i; float s = 1.0f / denom;
        uint32_t j = 0; for (; j < n; j++) if (out[j].doc_id == vec[i].doc_id) break;
        if (j == n) { out[n].doc_id = vec[i].doc_id; out[n].score = s; out[n].pad = 0; n++; }
        else { volatile float sum = out[j].score + s; out[j].score = sum; }
    }
    std::stable_sort(out, out + n, hit_better);
    if (n_out) *n_out = n;
    return SSB_OK;
    SSB_API_END
}

int32_t ssb_search_hybrid(ssb_index* ix, const ssb_lex_batch* q, const float* queries, uint32_t k, ssb_hit* hits, uint32_t* n_hits) {
    SSB_API_BEGIN
    if (!ix || !q || !queries || !hits) { set_error("ssb_search_hybrid: null argument"); return SSB_E_INVALID; }
    if (k == 0 || k > SSB_K_MAX) { set_error("k must be in 1..%u", SSB_K_MAX); return SSB_E_UNSUPPORTED; }
    std::shared_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    const uint32_t nq = q->n_queries;
    if (nq == 0) return SSB_OK;
    // the lexical field filter applies to the vector half as well (search.rs:1702-1731), on an index whose rows carry field ids
    const uint32_t* fm = nullptr;
    if (ix->vec.tagged()) SSB_TRY(ix->vec.field_masks(q->field_masks, nq, "ssb_search_hybrid", &fm));
    // the two per-shard searches are independent until the fusion: the lexical one runs on this context's stream, the vector one
    // on a second context's stream, so lex_score and the scan share the GPU instead of running back to back
    CtxLease l(ix); SSB_TRY(l.acquire());
    SearchCtx& c = *l.c;
    CtxLease l2(ix);
    SearchCtx* cv = &c;
    if (!ix->ext_stream_set) { SSB_TRY(l2.acquire(false)); if (l2.c) cv = l2.c; }   // never wait for a second context (no hold-and-wait)
    SSB_TRY(c.keys_a.reserve((size_t)nq * LIST, 0, c.st));
    SSB_TRY(cv->keys_b.reserve((size_t)nq * LIST, 0, cv->st));
    c.h_keys_a.resize((size_t)nq * LIST); cv->h_keys_b.resize((size_t)nq * LIST);
    SSB_TRY(ix->lex->search_keys(c.lex, c.st, q, k, SSB_RESULT_TOPK, c.keys_a.p, nullptr, &c.stats.kernel_launches));
    // sharded: both lists are merged over the shards FIRST and fused afterwards — RRF ranks are positions in the merged lists
    // (search.rs:1962-2035 runs after the shard results were concatenated and sorted)
    SSB_TRY(shard_merge(ix, c, c.keys_a.p, nq));
    SSB_CUDA_TRY(cudaMemcpyAsync(c.h_keys_a.data(), c.keys_a.p, (size_t)nq * LIST * 8, cudaMemcpyDeviceToHost, c.st));
    // multi-chunk documents: fetch the full 32-list so that k distinct docs survive the per-doc de-duplication
    SSB_TRY(ix->vec.search_keys(cv->vec, cv->st, cv->stats, &cv->ev_used, queries, false, nq, ix->vec.dup_docs() ? SSB_K_MAX : k, cv->keys_b.p,
                                nullptr, nullptr, fm));
    SSB_TRY(shard_merge(ix, *cv, cv->keys_b.p, nq));
    SSB_CUDA_TRY(cudaMemcpyAsync(cv->h_keys_b.data(), cv->keys_b.p, (size_t)nq * LIST * 8, cudaMemcpyDeviceToHost, cv->st));
    SSB_CUDA_TRY(cudaStreamSynchronize(c.st));
    if (cv != &c) SSB_CUDA_TRY(cudaStreamSynchronize(cv->st));
    c.stats.kernel_launches += cv != &c ? cv->stats.kernel_launches : 0;
    c.stats.h2d_bytes += cv != &c ? cv->stats.h2d_bytes : 0;
    c.stats.d2h_bytes += (uint64_t)nq * LIST * 16;
    std::vector<ssb_hit> a((size_t)nq * k), b((size_t)nq * k), f(2 * (size_t)k);
    PageState<1> pa(c, nq, k, a.data(), nullptr), pb(c, nq, k, b.data(), nullptr, ix->vec.dup_docs());
    pa.append(c.h_keys_a.data(), LIST); pb.append(cv->h_keys_b.data(), LIST);
    for (uint32_t i = 0; i < nq; i++) {
        uint32_t nf = 0;
        ssb_rrf_fuse(a.data() + (size_t)i * k, pa.cnt[i], b.data() + (size_t)i * k, pb.cnt[i], f.data(), &nf);
        uint32_t n = nf < k ? nf : k;     // search.rs:2117-2119 truncate(length)
        for (uint32_t j = 0; j < k; j++) hits[(size_t)i * k + j] = j < n ? f[j] : ssb_hit{0, 0.f, 0};
        if (n_hits) n_hits[i] = n;
    }
    return SSB_OK;
    SSB_API_END
}

int32_t ssb_merge_keys(ssb_index* ix, const uint64_t* keys_dev, uint32_t n_lists, uint32_t nq, uint32_t k, ssb_hit* hits, uint32_t* n_hits) {
    SSB_API_BEGIN
    if (!ix || !keys_dev || !hits) { set_error("ssb_merge_keys: null argument"); return SSB_E_INVALID; }
    if (k == 0 || k > SSB_K_MAX) { set_error("k must be in 1..%u", SSB_K_MAX); return SSB_E_UNSUPPORTED; }
    std::shared_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    if (nq == 0) return SSB_OK;
    CtxLease l(ix); SSB_TRY(l.acquire());
    SearchCtx& c = *l.c;
    SSB_TRY(c.keys_b.reserve((size_t)nq * LIST, 0, c.st));
    SSB_TRY(vec::launch_merge_lists(keys_dev, n_lists, nq, c.keys_b.p, c.st));
    c.stats.kernel_launches += 1;
    c.h_keys_b.resize((size_t)nq * LIST);
    SSB_CUDA_TRY(cudaMemcpyAsync(c.h_keys_b.data(), c.keys_b.p, (size_t)nq * LIST * 8, cudaMemcpyDeviceToHost, c.st));
    SSB_CUDA_TRY(cudaStreamSynchronize(c.st));
    PageState<1> ps(c, nq, k, hits, n_hits, ix->vec.dup_docs());
    ps.append(c.h_keys_b.data(), LIST);
    ps.finish();
    return SSB_OK;
    SSB_API_END
}

// ---- sharded index: one process per GPU, NCCL communicator owned by (or lent to) the handle -------------------------------
int32_t ssb_comm_unique_id(uint8_t* id128) {
    SSB_API_BEGIN
    if (!id128) { set_error("ssb_comm_unique_id: null argument"); return SSB_E_INVALID; }
    return comm_unique_id(id128);
    SSB_API_END
}

int32_t ssb_comm_init(ssb_index* ix, const uint8_t* id128, uint32_t rank, uint32_t world) {
    SSB_API_BEGIN
    if (!ix || !id128) { set_error("ssb_comm_init: null argument"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    if (ix->comm.comm) { set_error("ssb_comm_init: the index already has a communicator"); return SSB_E_STATE; }
    if (ix->lex->has_ngrams() && world > 1) { set_error("ssb_comm_init: n-gram lists on a sharded index are not supported"); return SSB_E_UNSUPPORTED; }
    SSB_TRY(refuse_tagged_sharded("ssb_comm_init", "vector rows", ix->vec.tagged(), world > 1));
    SSB_TRY(comm_init(ix->comm, id128, rank, world));
    std::lock_guard<std::mutex> g2(ix->pool_mu);
    if (ix->pool.size() > 1) { ix->pool.resize(1); ix->free_ctx.clear(); ix->free_ctx.push_back(ix->pool[0].get()); ix->last_ctx = nullptr; }
    return SSB_OK;
    SSB_API_END
}

int32_t ssb_comm_attach(ssb_index* ix, void* nccl_comm, uint32_t rank, uint32_t world) {
    SSB_API_BEGIN
    if (!ix || !nccl_comm || world == 0 || rank >= world) { set_error("ssb_comm_attach: bad argument"); return SSB_E_INVALID; }
    std::unique_lock<std::shared_mutex> g(ix->rw);
    if (ix->comm.comm) { set_error("ssb_comm_attach: the index already has a communicator"); return SSB_E_STATE; }
    if (ix->lex->has_ngrams() && world > 1) { set_error("ssb_comm_attach: n-gram lists on a sharded index are not supported"); return SSB_E_UNSUPPORTED; }
    SSB_TRY(refuse_tagged_sharded("ssb_comm_attach", "vector rows", ix->vec.tagged(), world > 1));
    ix->comm.comm = nccl_comm; ix->comm.rank = rank; ix->comm.world = world; ix->comm.owned = false;
    std::lock_guard<std::mutex> g2(ix->pool_mu);
    if (ix->pool.size() > 1) { ix->pool.resize(1); ix->free_ctx.clear(); ix->free_ctx.push_back(ix->pool[0].get()); ix->last_ctx = nullptr; }
    return SSB_OK;
    SSB_API_END
}

int32_t ssb_comm_destroy(ssb_index* ix) {
    SSB_API_BEGIN
    if (!ix) return SSB_E_INVALID;
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    comm_destroy(ix->comm);
    return SSB_OK;
    SSB_API_END
}

// Global document frequencies of a sharded index (idf must use the df of the WHOLE index, search.rs:3225-3230): every rank
// contributes its dictionary (sorted keys + local df), the sum per key is installed on every rank.  Collective.
int32_t ssb_lexical_sync_df(ssb_index* ix) {
    SSB_API_BEGIN
    if (!ix) return SSB_E_INVALID;
    std::unique_lock<std::shared_mutex> g(ix->rw);
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    if (!ix->comm.active()) return SSB_OK;
    if (ix->lex->has_ngrams()) { set_error("ssb_lexical_sync_df: n-gram lists on a sharded index are not supported"); return SSB_E_UNSUPPORTED; }
    if (!ix->lex->committed()) { set_error("ssb_lexical_sync_df before ssb_lexical_commit"); return SSB_E_STATE; }
    cudaStream_t st = ix->load_st;
    const std::vector<uint64_t>& keys = ix->lex->host_keys();
    const std::vector<uint32_t>& dfs = ix->lex->host_local_df();
    const uint32_t world = ix->comm.world;
    DevTmp<uint64_t> d_n; SSB_CUDA_TRY(d_n.alloc(1));
    uint64_t n_max = keys.size();
    SSB_CUDA_TRY(cudaMemcpyAsync(d_n.p, &n_max, 8, cudaMemcpyHostToDevice, st));
    SSB_TRY(comm_all_reduce_max_u64(ix->comm, d_n.p, 1, st));
    SSB_CUDA_TRY(cudaMemcpyAsync(&n_max, d_n.p, 8, cudaMemcpyDeviceToHost, st));
    SSB_CUDA_TRY(cudaStreamSynchronize(st));
    if (n_max == 0) return SSB_OK;
    // send [n_max] keys (padded with ~0, which sorts last and matches nothing) and [n_max] dfs
    std::vector<uint64_t> sk(n_max, ~0ull), sd(n_max, 0);
    for (size_t i = 0; i < keys.size(); i++) { sk[i] = keys[i]; sd[i] = dfs[i]; }
    DevTmp<uint64_t> d_sk, d_sd, d_rk, d_rd;
    SSB_CUDA_TRY(d_sk.alloc(n_max)); SSB_CUDA_TRY(d_sd.alloc(n_max)); SSB_CUDA_TRY(d_rk.alloc(n_max * world)); SSB_CUDA_TRY(d_rd.alloc(n_max * world));
    SSB_CUDA_TRY(cudaMemcpyAsync(d_sk.p, sk.data(), n_max * 8, cudaMemcpyHostToDevice, st));
    SSB_CUDA_TRY(cudaMemcpyAsync(d_sd.p, sd.data(), n_max * 8, cudaMemcpyHostToDevice, st));
    SSB_TRY(comm_all_gather_u64(ix->comm, d_sk.p, d_rk.p, n_max, st));
    SSB_TRY(comm_all_gather_u64(ix->comm, d_sd.p, d_rd.p, n_max, st));
    std::vector<uint64_t> rk(n_max * world), rd(n_max * world);
    SSB_CUDA_TRY(cudaMemcpyAsync(rk.data(), d_rk.p, n_max * world * 8, cudaMemcpyDeviceToHost, st));
    SSB_CUDA_TRY(cudaMemcpyAsync(rd.data(), d_rd.p, n_max * world * 8, cudaMemcpyDeviceToHost, st));
    SSB_CUDA_TRY(cudaStreamSynchronize(st));
    std::vector<uint32_t> total(keys.size(), 0);
    for (uint32_t r = 0; r < world; r++) {          // merge-join of two sorted key arrays
        const uint64_t* k2 = rk.data() + (size_t)r * n_max; const uint64_t* d2 = rd.data() + (size_t)r * n_max;
        size_t j = 0;
        for (size_t i = 0; i < keys.size(); i++) {
            while (j < n_max && k2[j] < keys[i]) j++;
            if (j < n_max && k2[j] == keys[i]) total[i] += (uint32_t)d2[j];
        }
    }
    return ix->lex->set_global_df(keys.data(), total.data(), keys.size());
    SSB_API_END
}

int32_t ssb_sync(ssb_index* ix) {
    SSB_API_BEGIN
    if (!ix) return SSB_E_INVALID;
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    std::vector<cudaStream_t> sts;
    {
        std::lock_guard<std::mutex> g(ix->pool_mu);
        for (auto& c : ix->pool) sts.push_back(ix->ext_stream_set ? ix->ext_stream : c->own_st);
    }
    for (cudaStream_t s : sts) SSB_CUDA_TRY(cudaStreamSynchronize(s));
    return SSB_OK;
    SSB_API_END
}

void* ssb_stream(ssb_index* ix) {
    if (!ix) return nullptr;
    if (ix->ext_stream_set) return (void*)ix->ext_stream;
    std::lock_guard<std::mutex> g(ix->pool_mu);
    return ix->pool.empty() ? (void*)ix->load_st : (void*)ix->pool[0]->own_st;
}

int32_t ssb_set_stream(ssb_index* ix, void* stream) {
    SSB_API_BEGIN
    if (!ix) return SSB_E_INVALID;
    std::unique_lock<std::shared_mutex> g(ix->rw);       // no search in flight
    SSB_CUDA_TRY(cudaSetDevice(ix->device));
    {
        std::lock_guard<std::mutex> g2(ix->pool_mu);
        for (auto& c : ix->pool) SSB_CUDA_TRY(cudaStreamSynchronize(ix->ext_stream_set ? ix->ext_stream : c->own_st));
        if (stream == SSB_OWN_STREAM) { ix->ext_stream_set = false; ix->ext_stream = nullptr; }
        else { ix->ext_stream_set = true; ix->ext_stream = (cudaStream_t)stream; }
        // with a caller-owned stream every search runs on that one stream: keep a single context
        if (ix->ext_stream_set && ix->pool.size() > 1) {
            ix->pool.resize(1); ix->free_ctx.clear(); ix->free_ctx.push_back(ix->pool[0].get()); ix->last_ctx = nullptr;
        }
    }
    return SSB_OK;
    SSB_API_END
}

int32_t ssb_last_stats(const ssb_index* cix, ssb_stats* out) {
    SSB_API_BEGIN
    if (!cix || !out) return SSB_E_INVALID;
    ssb_index* ix = const_cast<ssb_index*>(cix);
    SearchCtx* c = nullptr;
    { std::lock_guard<std::mutex> g(ix->stats_mu); *out = ix->last_stats; c = ix->last_ctx; }
    if (c && c->ev_used && out->dominant_kernel_ns == 0) {   // asynchronous *_keys call: wait for its kernel's events now
        cudaSetDevice(ix->device);
        float ms = 0.f;
        if (cudaEventSynchronize(c->ev1) == cudaSuccess && cudaEventElapsedTime(&ms, c->ev0, c->ev1) == cudaSuccess)
            out->dominant_kernel_ns = (uint64_t)((double)ms * 1e6);
        else cudaGetLastError();
        if (c->last_lex && out->postings_visited == 0 && c->lex.stats.p) {
            const LexStats ls = LexIndex::read_stats(c->lex, ix->ext_stream_set ? ix->ext_stream : c->own_st);
            out->postings_visited = ls.postings_visited; out->probes = ls.probes; out->items_processed = ls.items_processed; out->items_skipped = ls.items_skipped;
            if (ls.postings_visited) out->algorithmic_bytes = ls.postings_visited * 4 + ls.probes * 16 + ls.recs_processed * 128 + ls.dense_words * 8;
        }
    }
    return SSB_OK;
    SSB_API_END
}

}  // extern "C"
