// empty_query.cu — the empty query (Search::search("", enable_empty_query = true, ..), sm_90a): every live doc of the lexical levels
// through a batch's facet filters into its sorted top-k lists and counts, and the index-wide value counts of String facets.
//
// Replaces (all paths seekstorm/src/ of the reference): search_iterator_shard (iterator.rs:316-358) — docs 0..indexed_doc_count through
// add_result_singleterm_multifield with the delete set and is_facet_filter (add_result.rs:95-338, 340-478), the top-k by the sort criteria
// with ties to the larger doc id (min_heap.rs:535-536, 1043-1044); search_iterator_index (iterator.rs:360-413) as the one-criterion
// `_id` / `_score` order; get_index_string_facets_shard (index.rs:4441-4569).
//
// empty_scan: the doc ids of the levels are cut into tiles of `tile` docs inside one level, taken by persistent CTAs from an atomic
// counter in descending doc-id order (the default order, doc id descending, then fills every query's list from the first tiles and its θ
// prunes the rest).  Per tile the CTA decides for every query of the batch from the level zones (FacetSet::d_zones) and θ alone whether
// it needs the tile's rows; only then it stages the columns of the facets the batch touches (filters and sort criteria) into shared
// memory, next to the tile's delete words.  One warp per (tile, query) then tests 32 docs per round from shared memory and inserts the
// passing docs into a 128-bit top-k list (sort_list.cuh), merged into the query's global list once per tile.
#include "bm25.h"
#include "facets.cuh"
#include "sort_list.cuh"

#include <algorithm>

namespace ssb {

constexpr uint32_t EQ_WARPS = 8;
// CTAs per SM: the staging of one CTA overlaps the tests of the others.  A batch with a POINT filter or criterion runs 2: its out-of-line
// distance test needs the registers of the third (ptxas spills at 3)
template <bool GEO> constexpr uint32_t eq_minb() { return GEO ? 2u : 3u; }
constexpr size_t EQ_STAGE_BYTES = 64 * 1024;       // staged columns per CTA
enum { EQ_STAT_PROCESSED = 0, EQ_STAT_SKIPPED = 1, EQ_STAT_ROWS = 2, EQ_STAT_TILES = 3, EQ_STAT_WORDS = 4 };

struct EmptyArgs {
    const uint2* tiles; uint32_t n_tiles, tile;                       // tiles: {first doc id, docs}, descending
    const uint64_t* keys; uint64_t rows; uint32_t first_doc;          // the facet columns (FacetSet)
    uint32_t nt; uint32_t col[SSB_MAX_FACETS]; uint32_t slot[SSB_MAX_FACETS];   // staged slot s holds facet col[s]; slot[facet] = its slot
    const uint64_t* zones; uint32_t zone_block0, n_zone_blocks;
    const uint32_t* del_slot; const uint64_t* del_words;
    const uint32_t* foff; const FiltDev* filt; const uint64_t* sets;   // foff null: no query is filtered
    uint32_t nq, k, result_type;
    uint32_t* ctr; uint64_t* theta; int* lock; unsigned long long* count; uint64_t* glist; const uint64_t* ceil;
    unsigned long long* stats;                                         // EQ_STAT_*
};

// What query q needs of a tile (docs doc0 .. doc0 + n - 1 of level `level`; the facet rows cover its docs [rl, rh)).  The zones decide
// its RANGE and POINT filters for the whole level: a filter no row of the level passes skips the tile, a RANGE filter every row passes is
// dropped from `mask` (the filters still tested per doc).  `insert`: the tile can hold a doc of q's top-k (its bound is not below θ.hi;
// θ only rises, so a tile found prunable stays so).  `rows`: the per-doc test runs (filters left, docs without a facet row, or inserts).
struct EqPlan { bool skip, insert, rows, check_rows; uint32_t mask; };
__device__ __forceinline__ EqPlan eq_plan(const EmptyArgs& a, uint32_t q, uint32_t level, uint32_t rl, uint32_t rh, uint32_t n, uint64_t bound_hi) {
    EqPlan p{false, false, false, false, 0u};
    const uint32_t f0 = a.foff ? __ldg(&a.foff[q]) : 0u, nf = a.foff ? __ldg(&a.foff[q + 1]) - f0 : 0u;
    if (nf) {
        if (rh <= rl) { p.skip = true; return p; }                     // no doc of the tile has a facet row: every filter rejects it
        const uint32_t b = level - a.zone_block0;
        for (uint32_t i = 0; i < nf; i++) {
            const FiltDev f = a.filt[f0 + i];
            if (f.kind == FILT_NEVER) { p.skip = true; return p; }
            if (f.kind == FILT_RANGE || f.kind == FILT_POINT) {
                const uint64_t* z = a.zones + ((size_t)f.facet * a.n_zone_blocks + b) * 2;
                const uint64_t zmin = __ldg(&z[0]), zmax = __ldg(&z[1]);
                if (zmax < f.lo || zmin >= f.hi) { p.skip = true; return p; }
                if (f.kind == FILT_RANGE && zmin >= f.lo && zmax < f.hi) continue;
            }
            p.mask |= 1u << i;
        }
        p.check_rows = rl != 0 || rh != n;
    }
    p.insert = a.result_type != SSB_RESULT_COUNT && !(bound_hi < __ldcg(&a.theta[2 * q]));
    if (!p.insert && a.result_type == SSB_RESULT_TOPK) { p.skip = true; return p; }
    p.rows = p.insert || p.mask || p.check_rows;
    return p;
}

template <bool GEO>
__global__ void __launch_bounds__(EQ_WARPS * 32, eq_minb<GEO>()) empty_scan(EmptyArgs a, SortDev s) {
    extern __shared__ __align__(16) unsigned char eq_smem[];
    const uint32_t T = a.tile;
    uint64_t* stage = reinterpret_cast<uint64_t*>(eq_smem);                     // [nt][T]
    uint64_t* sdel = stage + (size_t)a.nt * T;                                   // [T / 64]
    FiltDev* wfilt = reinterpret_cast<FiltDev*>(sdel + T / 64);                  // [EQ_WARPS][16]
    __shared__ uint32_t s_item;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    FiltDev* myf = wfilt + warp * SSB_MAX_FILTERS_PER_QUERY;
    uint64_t st_proc = 0, st_skip = 0;
    for (;;) {
        if (threadIdx.x == 0) s_item = atomicAdd(a.ctr, 1u);
        __syncthreads();
        const uint32_t item = s_item;
        if (item >= a.n_tiles) break;
        const uint2 t = __ldg(&a.tiles[item]);
        const uint32_t doc0 = t.x, n = t.y, level = doc0 >> 16;
        const uint64_t rows_lo = a.first_doc, rows_hi = (uint64_t)a.first_doc + a.rows;
        const uint32_t rl = (uint32_t)(rows_lo > doc0 ? min(rows_lo - doc0, (uint64_t)n) : 0ull);
        const uint32_t rh = (uint32_t)(rows_hi > doc0 ? min(rows_hi - doc0, (uint64_t)n) : 0ull);
        const uint64_t bound_hi = level_sort_bound(s, level, doc0 & 0xFFFFu, (doc0 & 0xFFFFu) + n - 1);
        // does any query need the tile's rows?
        bool need = false;
        for (uint32_t q = threadIdx.x; q < a.nq && !need; q += blockDim.x) need = eq_plan(a, q, level, rl, rh, n, bound_hi).rows;
        need = __syncthreads_or(need) != 0;
        if (need) {
            for (uint32_t i = threadIdx.x; i < a.nt * T; i += blockDim.x) {
                const uint32_t sl = i / T, r = i - sl * T;
                stage[i] = r >= rl && r < rh ? __ldg(&a.keys[(size_t)a.col[sl] * a.rows + (doc0 + r - a.first_doc)]) : 0ull;
            }
        }
        for (uint32_t w = threadIdx.x; w < T / 64; w += blockDim.x) {
            uint64_t x = 0;
            if (a.del_slot && w * 64 < n) {
                const uint32_t sl = __ldg(&a.del_slot[level]);
                if (sl != 0xFFFFFFFFu) x = __ldg(&a.del_words[(size_t)sl * 1024 + (((doc0 & 0xFFFFu) >> 6) + w)]);
            }
            if (w * 64 + 64 > n) x &= w * 64 < n ? (1ull << (n - w * 64)) - 1ull : 0ull;   // docs past the level's end
            sdel[w] = x;
        }
        if (threadIdx.x == 0) {
            atomicAdd(&a.stats[EQ_STAT_TILES], 1ull);
            if (need) atomicAdd(&a.stats[EQ_STAT_ROWS], (unsigned long long)n);
            if (a.del_slot) atomicAdd(&a.stats[EQ_STAT_WORDS], (unsigned long long)((n + 63) / 64));
        }
        __syncthreads();
        uint32_t n_del = 0;
        for (uint32_t w = lane; w < (n + 63) / 64; w += 32) n_del += __popcll(sdel[w]);
        n_del = __reduce_add_sync(FULL, n_del);
        for (uint32_t q = warp; q < a.nq; q += EQ_WARPS) {
            const EqPlan p = eq_plan(a, q, level, rl, rh, n, bound_hi);
            if (p.skip) { st_skip++; continue; }
            st_proc++;
            uint32_t cnt = 0;
            if (!p.rows) cnt = n - n_del;                                // every live doc of the tile passes
            else {
                const uint32_t f0 = a.foff ? __ldg(&a.foff[q]) : 0u;
                __syncwarp();
                if (lane < 32 - __clz(p.mask)) myf[lane] = a.filt[f0 + lane];
                __syncwarp();
                SortTop top{0ull, 0ull, __ldcg(&a.theta[2 * q])};
                bool dirty = false;
                const uint64_t ch = a.ceil ? __ldg(&a.ceil[2 * q]) : ~0ull, cl = a.ceil ? __ldg(&a.ceil[2 * q + 1]) : ~0ull;
                for (int base = (int)((n - 1) & ~31u); base >= 0; base -= 32) {   // from the tile's top: doc id descending
                    const uint32_t r = (uint32_t)base + lane, doc = doc0 + r;
                    bool ok = r < n && !((sdel[r >> 6] >> (r & 63)) & 1ull);
                    if (p.check_rows) ok = ok && r >= rl && r < rh;
                    for (uint32_t m = p.mask; ok && m; m &= m - 1) {
                        const FiltDev& f = myf[__ffs(m) - 1];
                        ok = !filter_rejects_key<GEO>(f, stage[(size_t)a.slot[f.facet] * T + r], a.sets);
                    }
                    cnt += __popc(__ballot_sync(FULL, ok));
                    if (p.insert) {
                        uint64_t hi = 0;
                        if (ok) hi = sort_hi_of<GEO>(s, doc, q, [&](uint32_t i) { return stage[(size_t)a.slot[s.facet[i]] * T + r]; });
                        insert_sorted(top, ok && hi >= top.thr, hi, 0.f, 0xFFFFFFFFu - doc, false, a.k, lane, dirty, ch, cl);
                    }
                }
                if (dirty) publish_sorted(top, q, a.k, lane, a.theta, a.lock, a.glist);
            }
            if (a.result_type != SSB_RESULT_TOPK && lane == 0 && cnt) atomicAdd(&a.count[q], (unsigned long long)cnt);
        }
        __syncthreads();
    }
    if (lane == 0) {
        atomicAdd(&a.stats[EQ_STAT_PROCESSED], (unsigned long long)st_proc);
        atomicAdd(&a.stats[EQ_STAT_SKIPPED], (unsigned long long)st_skip);
    }
}

// value counts of one String facet over every facet row (index-wide, as the counters ingest keeps): hist[key]++, per-CTA shared
// histogram when it fits.  A StringSet facet (set_off / set_mem: its CSR, else null) scatters each row to the member ids of its
// combination, once per occurrence (index.rs:4531-4550).
constexpr uint32_t EQ_HIST_LOCAL = 12288;          // bins of a per-CTA shared histogram
__global__ void __launch_bounds__(256) empty_value_hist(const uint64_t* __restrict__ col, uint64_t rows, uint32_t n_bins, const uint64_t* __restrict__ set_off,
                                                        const uint32_t* __restrict__ set_mem, uint32_t* __restrict__ hist) {
    extern __shared__ uint32_t eh[];
    const bool local = n_bins <= EQ_HIST_LOCAL;
    if (local) { for (uint32_t i = threadIdx.x; i < n_bins; i += blockDim.x) eh[i] = 0; __syncthreads(); }
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t v = (uint32_t)__ldg(&col[r]);
        if (!set_off) { if (local) atomicAdd(&eh[v], 1u); else atomicAdd(&hist[v], 1u); continue; }
        const uint64_t e = __ldg(&set_off[v + 1]);
        for (uint64_t j = __ldg(&set_off[v]); j < e; j++) {
            const uint32_t m = __ldg(&set_mem[j]);
            if (local) atomicAdd(&eh[m], 1u); else atomicAdd(&hist[m], 1u);
        }
    }
    if (local) {
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < n_bins; i += blockDim.x) if (eh[i]) atomicAdd(&hist[i], eh[i]);
    }
}

// ================================================================= host side
void LexIndex::refresh_live_docs() {
    std::vector<uint32_t> n_of(65536, 0);
    uint64_t live = 0;
    for (const LexLevel& l : levels_) { n_of[l.level_id & 0xFFFFu] = l.n_docs; live += l.n_docs; }
    if (del_) for (uint32_t d : del_->h_docs) if ((d & 0xFFFFu) < n_of[d >> 16]) live--;
    live_docs_ = live;
}

int32_t LexIndex::search_empty(LexWorkspace& ws, cudaStream_t st, const ssb_lex_batch* q, uint32_t k, uint32_t result_type, const SortDev& sort,
                               uint64_t* keys_out_dev, uint64_t* count_dev, const uint64_t* ceil_dev, EmptyStats* stats) const {
    if (!committed_) { set_error("search before ssb_lexical_commit"); return SSB_E_STATE; }
    if (k > SSB_K_MAX) { set_error("k=%u exceeds SSB_K_MAX=%u", k, SSB_K_MAX); return SSB_E_UNSUPPORTED; }
    if (result_type > SSB_RESULT_TOPKCOUNT) { set_error("bad result_type"); return SSB_E_INVALID; }
    if (result_type != SSB_RESULT_COUNT && k == 0) result_type = SSB_RESULT_COUNT;   // search.rs:2472-2478
    const uint32_t nq = q->n_queries;
    if (nq == 0) return SSB_OK;
    if (q->term_offsets) {                                             // a filter-only batch: no terms
        if (is_device_ptr(q->term_offsets)) { set_error("search_empty: term_offsets must be a host array or NULL"); return SSB_E_INVALID; }
        for (uint32_t i = 0; i <= nq; i++) if (q->term_offsets[i]) { set_error("search_empty: query %u has terms", i ? i - 1 : 0); return SSB_E_INVALID; }
    }
    SSB_TRY(ensure_workspace(ws, st, nq, 0));
    LexView v = view();
    bool filtered = false, geo = false;
    if (q->filter_offsets) SSB_TRY(stage_filters(ws, st, q, v, &filtered, &geo));
    geo = geo || sort_has_point(sort);
    // the facets the batch touches, each staged once per tile
    EmptyArgs a{};
    bool touched[SSB_MAX_FACETS] = {};
    if (filtered) for (uint32_t i = 0; i < q->filter_offsets[nq]; i++) touched[q->filters[i].facet] = true;
    for (uint32_t j = 0; j < sort.n; j++) if (sort.src[j] == SORT_SRC_FACET) touched[sort.facet[j]] = true;
    for (uint32_t f = 0; f < SSB_MAX_FACETS; f++) if (touched[f]) { a.slot[f] = a.nt; a.col[a.nt++] = f; }
    // the tile: as many docs as keep the staged columns within EQ_STAGE_BYTES, 512 .. 4096, a multiple of 64
    uint32_t T = 4096;
    while (T > 512 && (size_t)a.nt * T * 8 > EQ_STAGE_BYTES) T >>= 1;
    std::vector<const LexLevel*> lv;
    for (const LexLevel& l : levels_) if (l.n_docs) lv.push_back(&l);
    std::sort(lv.begin(), lv.end(), [](const LexLevel* x, const LexLevel* y) { return x->level_id > y->level_id; });
    std::vector<uint2> tiles;
    for (const LexLevel* l : lv)
        for (int64_t s0 = (int64_t)((l->n_docs - 1) / T) * T; s0 >= 0; s0 -= T)
            tiles.push_back(make_uint2(l->level_id << 16 | (uint32_t)s0, std::min<uint32_t>(T, l->n_docs - (uint32_t)s0)));
    SSB_TRY(ws.etiles.reserve(tiles.size() + 1, 0, st, true));
    SSB_TRY(ws.estats.reserve(8, 0, st, true));
    if (!tiles.empty()) SSB_CUDA_TRY(cudaMemcpyAsync(ws.etiles.p, tiles.data(), tiles.size() * sizeof(uint2), cudaMemcpyHostToDevice, st));
    SSB_CUDA_TRY(cudaMemsetAsync(ws.ctr.p, 0, 32, st));
    SSB_CUDA_TRY(cudaMemsetAsync(ws.theta.p, 0, (size_t)nq * 16, st));
    SSB_CUDA_TRY(cudaMemsetAsync(ws.lock.p, 0, (size_t)nq * sizeof(int), st));
    SSB_CUDA_TRY(cudaMemsetAsync(ws.count.p, 0, (size_t)nq * 8, st));
    SSB_CUDA_TRY(cudaMemsetAsync(keys_out_dev, 0, (size_t)nq * LIST * 16, st));
    SSB_CUDA_TRY(cudaMemsetAsync(ws.estats.p, 0, 8 * 8, st));
    a.tiles = ws.etiles.p; a.n_tiles = (uint32_t)tiles.size(); a.tile = T;
    a.keys = v.facet_keys; a.rows = v.facet_rows; a.first_doc = v.facet_first_doc;
    if (facets_) { a.zones = facets_->d_zones; a.zone_block0 = facets_->zone_block0; a.n_zone_blocks = facets_->n_zone_blocks; }
    a.del_slot = v.del_slot; a.del_words = v.del_words;
    if (filtered) { a.foff = ws.foff.p; a.filt = v.filt; a.sets = v.filt_sets; }
    a.nq = nq; a.k = k ? k : 1; a.result_type = result_type;
    a.ctr = ws.ctr.p; a.theta = ws.theta.p; a.lock = ws.lock.p; a.count = reinterpret_cast<unsigned long long*>(ws.count.p);
    a.glist = keys_out_dev; a.ceil = ceil_dev; a.stats = ws.estats.p;
    auto kern = geo ? empty_scan<true> : empty_scan<false>;
    const size_t smem = (size_t)a.nt * T * 8 + (T / 64) * 8 + EQ_WARPS * SSB_MAX_FILTERS_PER_QUERY * sizeof(FiltDev);
    SSB_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const uint32_t grid = std::max<uint32_t>(1u, std::min<uint32_t>((uint32_t)n_sms_ * (geo ? eq_minb<true>() : eq_minb<false>()), a.n_tiles));
    if (ws.ev0) cudaEventRecord(ws.ev0, st);
    kern<<<grid, EQ_WARPS * 32, smem, st>>>(a, sort);
    SSB_CUDA_TRY(cudaGetLastError());
    if (ws.ev1) cudaEventRecord(ws.ev1, st);
    if (count_dev) SSB_CUDA_TRY(cudaMemcpyAsync(count_dev, ws.count.p, (size_t)nq * 8, cudaMemcpyDeviceToDevice, st));
    if (stats) {
        unsigned long long c[8];
        SSB_CUDA_TRY(cudaMemcpyAsync(c, ws.estats.p, sizeof(c), cudaMemcpyDeviceToHost, st));
        SSB_CUDA_TRY(cudaStreamSynchronize(st));
        stats->launches += 1;
        stats->items_processed += c[EQ_STAT_PROCESSED]; stats->items_skipped += c[EQ_STAT_SKIPPED];
        stats->alg_bytes += c[EQ_STAT_ROWS] * a.nt * 8 + c[EQ_STAT_WORDS] * 8;
    }
    return SSB_OK;
}

int32_t LexIndex::empty_facets(LexWorkspace& ws, cudaStream_t st, const ssb_facet_request* req, uint32_t n_req, ssb_facet_count* out,
                               uint32_t* n_out, EmptyStats* stats) const {
    if (n_req && (!req || !out || !n_out)) { set_error("search_empty_facets: null argument"); return SSB_E_INVALID; }
    if (n_req > SSB_MAX_FACET_REQUESTS) { set_error("search_empty_facets: %u requests, at most %u", n_req, SSB_MAX_FACET_REQUESTS); return SSB_E_UNSUPPORTED; }
    if (n_req == 0) return SSB_OK;
    if (!facets_ || !facets_->n_facets) { set_error("search_empty_facets: facet counts need ssb_set_facets"); return SSB_E_STATE; }
    const FacetSet& fs = *facets_;
    std::vector<FacetReqDev> rd(n_req);
    std::vector<uint64_t> starts;
    uint64_t hist_words = 0, out_stride = 0;
    for (uint32_t i = 0; i < n_req; i++) {
        const uint32_t f = req[i].facet;
        if (f >= fs.n_facets) { set_error("facet request %u: facet %u of %u", i, f, fs.n_facets); return SSB_E_INVALID; }
        const bool set = facet_is_stringset(fs.types[f]);
        const bool has_order = set ? fs.n_sets[f] != 0 : fs.d_rank[f] && fs.max_key[f] < fs.n_rank[f];
        SSB_TRY(encode_facet_request(req[i], i, fs.types[f], has_order, set ? (uint64_t)fs.n_values[f] - 1 : fs.max_key[f], true, &rd[i], starts));
        rd[i].out_off = (uint32_t)out_stride;
        if (rd[i].kind == FREQ_VALUES) {
            out_stride += rd[i].length;
            if (rd[i].length) { rd[i].hist_off = (uint32_t)hist_words; hist_words += rd[i].n_bins; }
        } else { out_stride += rd[i].n_bins; rd[i].length = 0; rd[i].kind = FREQ_VALUES; }   // range facets of the empty query: none
    }
    if (hist_words * 4 > (256ull << 20)) { set_error("search_empty_facets: the value histograms take %llu bytes, above 256 MiB", (unsigned long long)hist_words * 4); return SSB_E_UNSUPPORTED; }
    SSB_TRY(ws.fhist.reserve(hist_words + 1, 0, st, true));
    SSB_TRY(ws.freq.reserve(SSB_MAX_FACET_REQUESTS, 0, st, true));
    SSB_TRY(ws.fout.reserve(out_stride + 1, 0, st, true));
    SSB_TRY(ws.fnout.reserve(n_req, 0, st, true));
    SSB_CUDA_TRY(cudaMemcpyAsync(ws.freq.p, rd.data(), n_req * sizeof(FacetReqDev), cudaMemcpyHostToDevice, st));
    SSB_CUDA_TRY(cudaMemsetAsync(ws.fhist.p, 0, (hist_words + 1) * 4, st));
    if (ws.ev0) cudaEventRecord(ws.ev0, st);
    for (uint32_t i = 0; i < n_req; i++) {
        if (rd[i].kind != FREQ_VALUES || !rd[i].length) continue;
        const size_t smem = rd[i].n_bins <= EQ_HIST_LOCAL ? (size_t)rd[i].n_bins * 4 : 0;
        const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((fs.n_rows + 255) / 256, (uint64_t)n_sms_ * 4));
        const uint32_t f = rd[i].facet;
        const bool set = facet_is_stringset(fs.types[f]);
        empty_value_hist<<<grid, 256, smem, st>>>(fs.d_keys + (size_t)f * fs.n_rows, fs.n_rows, rd[i].n_bins, set ? fs.d_set_off[f] : nullptr,
                                                  set ? fs.d_set_mem[f] : nullptr, ws.fhist.p + rd[i].hist_off);
        SSB_CUDA_TRY(cudaGetLastError());
        // the column, and for a StringSet facet the two offsets of every row and its member ids
        if (stats) { stats->launches += 1; stats->alg_bytes += fs.n_rows * 8 + (set ? fs.n_rows * 16 + fs.member_rows[f] * 4 : 0); }
    }
    if (ws.ev1) cudaEventRecord(ws.ev1, st);
    SSB_TRY(launch_facet_select(fs, ws.freq.p, n_req, ws.fhist.p, (uint32_t)hist_words, 1, ws.fout.p, (uint32_t)out_stride, ws.fnout.p, st));
    if (stats) stats->launches += 1;
    if (out_stride) SSB_CUDA_TRY(cudaMemcpyAsync(out, ws.fout.p, out_stride * sizeof(ssb_facet_count), cudaMemcpyDeviceToHost, st));
    SSB_CUDA_TRY(cudaMemcpyAsync(n_out, ws.fnout.p, n_req * 4, cudaMemcpyDeviceToHost, st));
    SSB_CUDA_TRY(cudaStreamSynchronize(st));
    float ms = 0.f;
    if (stats && ws.ev0 && ws.ev1 && cudaEventElapsedTime(&ms, ws.ev0, ws.ev1) == cudaSuccess) stats->kernel_ns = (uint64_t)((double)ms * 1e6);
    else cudaGetLastError();
    return SSB_OK;
}

}  // namespace ssb
