// bm25.cu — BM25 AND/OR top-k over block-partitioned posting lists (sm_90a).
//
// Replaces, for committed data (all paths /root/reference/seekstorm/src/; the per-candidate chain — delete set, NOT lists, facet filters,
// field filter, phrase check: add_result.rs:3435-3500, 3124-3137, 3586-3684, multi-field phrase 3247-3389 — runs as predicates of the scoring
// kernels, see lex_generic):
//   intersection_blockid / intersection_docid   intersection.rs:2023-2301 / 112-2013   (AND)
//   intersection_bitmap_2                       intersection.rs:33-108                 (dense x dense: bitmap-word AND + popcount)
//   union_docid_2 / union_docid_3 / single_blockid  union.rs:1168-1479, single.rs:292-417 (OR + block-max)
//   union_count                                 union.rs:807-1164                      (exact |union|: bitmap-word OR + popcount)
//   add_result_multiterm_singlefield + get_bm25f_multiterm_singlefield  add_result.rs:3418-3706, 1429-1482
//   MinHeap::add_topk  min_heap.rs:1193-1259
//
// HBM layout (built once at load; the reference's per-level byte arrays are decoded by the caller / loader):
//   post[] u32 = id16 | bound16<<16 — the STREAM arena, one word per posting, all levels concatenated (level-major,
//          term-major inside a level).  bound16 = fp16 bits of the posting's query-independent score component
//          tf*(K+1)/(tf+cache[len]) rounded UP (filled at commit, when avgdl is known): the per-posting upper bound
//          idf*bound + R is three instructions (cvt, ffma, compare) and needs no table lookup, so a warp filters 128
//          postings per 16-byte-per-lane load.
//   pay[]  u32 = tf16 | doclen_byte<<16 — the PAYLOAD arena (same index): read only for the few postings whose exact
//          score is computed.  The doc-length byte is co-located with the posting, so scoring never gathers from the
//          64 KB per-level length array the way add_result.rs:1437-1442 does.
//   directory: sorted dict_keys -> per-term list of (level, offset, count, block-max, bitmap) entries;
//          lists with >= 256 postings additionally get an 8 KB bitmap + 2 KB rank index for O(1) probes (the
//          reference's Bitmap container starts at 4096, compress_postinglist.rs:256-332).
//
// Execution: one batch = lex_plan (per query: dictionary lookup, per-level bound = Σ idf·block-max in query order,
// levels sorted by bound, one fully resolved 128-byte RECORD per (query, level) with the MAXSCORE order and the
// in-order suffix bounds precomputed by one thread, records grouped into work ITEMS of <= 8 levels) + one persistent
// lex_score launch whose warps pull items wave by wave (every query's best levels first).  Inside an item the warp keeps
// its top-k list and threshold in registers across levels, streams the essential lists, pushes the postings that pass the
// bound filter into a per-warp shared-memory queue and runs the expensive stages (bitmap presence filter, exact in-order
// re-score) on 32 queued survivors at a time — lanes of one batch may belong to different levels and drivers.
// A per-query global threshold θ (k-th best key so far, merged under a per-query lock once per dirty item) gives
// block-max pruning across items.  Scores are bit-exact w.r.t. the CPU oracle: every f32 op individually rounded
// (__fmul_rn/__fdiv_rn/__fadd_rn), summed in query order from 0.0 (add_result.rs:1450-1452), idf and the 256-entry
// cache computed on the host.
#include "bm25.h"
#include "facets.cuh"
#include "sort_list.cuh"

#include <algorithm>
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <thrust/device_ptr.h>
#include <thrust/execution_policy.h>
#include <thrust/reduce.h>
#include <thrust/scan.h>
#include <thrust/sort.h>
#include <thrust/iterator/constant_iterator.h>
#include <thrust/iterator/discard_iterator.h>

namespace ssb {

constexpr uint32_t NONE = 0xFFFFFFFFu;
#ifndef SSB_DENSE_MIN
#define SSB_DENSE_MIN 128
#endif
constexpr uint32_t DENSE_MIN = SSB_DENSE_MIN;     // lists at least this long get a bitmap + rank index (O(1) probes)
constexpr uint32_t MAX_LEVELS = 4096;   // per GPU (268M docs); plan kernel smem bound
constexpr uint32_t FAST_T = 4;          // queries with <= 4 live terms take the record path
constexpr uint32_t ENT_NONE = 0xFFFFu;
constexpr uint32_t GMAX = 8;            // records (levels) per work item
constexpr uint32_t ITEM_W = 4096;       // target size of an item: postings of its top-ranked lists (+64 per record)
constexpr uint32_t QCAP = 192;          // survivor queue slots per warp: < 32 pending + 4 x 32 pushed per iteration
constexpr float Q8_STEP = (2.2f * 1.01f) / 255.0f;   // coarse byte bounds: components are < K + 1 = 2.2 (fp16 round-up included in the 1 %)
constexpr float INFL = 1.000002f;       // bound inflation covering the fp16 round-up + different association of <= 4 additions

// ================================================================= build kernels
__global__ void validate_offsets(const uint32_t* __restrict__ offs, uint32_t n_terms, uint32_t* bad) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0 && offs[0] != 0) atomicAdd(bad, 1u);
    if (i < n_terms && offs[i + 1] < offs[i]) atomicAdd(bad, 1u);
}
__global__ void validate_keys_sorted_unique(const uint64_t* __restrict__ sorted_keys, uint32_t n, uint32_t* bad) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i + 1 < n && sorted_keys[i] == sorted_keys[i + 1]) atomicAdd(bad, 1u);
}
// posting i belongs to the term whose offset range contains it (binary search over posting_offsets)
__global__ void validate_level(const uint16_t* __restrict__ ids, const uint16_t* __restrict__ tfs, const uint32_t* __restrict__ offs,
                               uint32_t n_terms, uint32_t n, uint32_t n_docs, uint32_t* bad, uint32_t nf) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t lo = 0, hi = n_terms;                     // term t with offs[t] <= i < offs[t+1]
    while (lo < hi) { uint32_t m = (lo + hi) >> 1; if (offs[m + 1] <= i) lo = m + 1; else hi = m; }
    uint32_t tfmax = 0;
    for (uint32_t f = 0; f < nf; f++) tfmax = max(tfmax, (uint32_t)tfs[(size_t)i * nf + f]);   // the term occurs in at least one field
    bool ok = lo < n_terms && ids[i] < n_docs && tfmax >= 1;
    if (ok && i > offs[lo] && ids[i] <= ids[i - 1]) ok = false;
    if (!ok) atomicAdd(bad, 1u);
}

// positions of one level: the posting's tf positions must ascend strictly (get_next_position_singlefield decodes ascending deltas).
// Several fields: the posting holds one run per field (field 0's tfs[0] positions, then field 1's, ...), each run ascends strictly and
// restarts from 0 (add_result.rs:3258-3283 reads them field by field).
__global__ void validate_positions(const uint16_t* __restrict__ pos, const uint32_t* __restrict__ off, const uint16_t* __restrict__ tfs, uint32_t n,
                                   uint32_t nf, uint32_t* bad) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t o = off[i];
    for (uint32_t f = 0; f < nf; f++) {
        const uint32_t tf = tfs[(size_t)i * nf + f];
        for (uint32_t j = 1; j < tf; j++) if (pos[o + j] <= pos[o + j - 1]) { atomicAdd(bad, 1u); return; }
        o += tf;
    }
}
// positions of one posting: Σ_f tf_f
__global__ void widen_tf(const uint16_t* __restrict__ tfs, uint32_t* __restrict__ out, uint32_t n, uint32_t nf) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t s = 0;
    for (uint32_t f = 0; f < nf; f++) s += tfs[(size_t)i * nf + f];
    out[i] = s;
}

__global__ void build_postings(const uint16_t* __restrict__ ids, const uint16_t* __restrict__ tfs, const uint8_t* __restrict__ len_bytes,
                               uint32_t* __restrict__ post, uint32_t* __restrict__ pay, uint32_t n,
                               uint32_t nf, uint32_t n_docs, uint32_t* __restrict__ payf /*several fields: [n][nf]*/) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t id = ids[i];
    post[i] = id;                                                 // bound16 is filled by fill_bounds at commit
    pay[i] = (uint32_t)tfs[(size_t)i * nf] | ((uint32_t)len_bytes[id] << 16);  // tf16 | len8<<16 (field 0)
    if (nf > 1)
        for (uint32_t f = 0; f < nf; f++) payf[(size_t)i * nf + f] = (uint32_t)tfs[(size_t)i * nf + f] | ((uint32_t)len_bytes[(size_t)f * n_docs + id] << 16);
}

// query-independent posting score component: tf*(K+1)/(tf+cache[len])   (add_result.rs:1450)
__device__ __forceinline__ float comp_of(const LexView& v, uint32_t payload) {
    const float tf = (float)(payload & 0xFFFFu);
    return __fdiv_rn(__fmul_rn(tf, v.k1p), __fadd_rn(tf, __ldg(&v.cache[(payload >> 16) & 255u])));
}

__global__ void fill_bounds(LexView v, uint32_t* __restrict__ post, float* __restrict__ comp, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float c;
    if (v.n_fields > 1) {
        // several fields: exact per-field components for the scorer; comp[] / the fp16 bound carry an upper bound of the posting's
        // boost-weighted sum.  The exact score adds up to 4 products (boost*idf)*comp_f per term while a bound adds ONE idf*comp per term:
        // the rounding of the two sums is not comparable term by term, 2^-16 of slack covers <= 128 + 32 f32 additions with room.
        float b = 0.f;
        for (uint32_t f = 0; f < v.n_fields; f++) {
            const uint32_t pl = v.payf[i * v.n_fields + f];
            const float cf = (pl & 0xFFFFu) ? comp_of(v, pl) : 0.f;
            const_cast<float*>(v.compf)[i * v.n_fields + f] = cf;
            b = __fadd_ru(b, __fmul_ru(v.boost[f], cf));
        }
        c = __fmul_ru(b, 1.0000153f);
    } else c = comp_of(v, v.pay[i]);
    comp[i] = c;                                                  // the IEEE divide + cache lookup happen once, here
    const __half h = __float2half_ru(c);                          // rounded UP: idf*h >= idf*comp
    post[i] = (post[i] & 0xFFFFu) | ((uint32_t)__half_as_ushort(h) << 16);
}

// n-gram lists (ssb_lexical_add_level_ngrams).  One (n-gram key, level) segment at commit: its postings in the arenas, the first of its
// component tfs in the commit's tf array (segments in tf order), the resolved component idfs (n_comp = 0: BM25F_PROXIMITY, the list adds 0)
struct NgSegDev { uint64_t post_off, tf_off; uint32_t cnt, n_comp; float idf[3]; uint32_t pad; };
__device__ __forceinline__ float ngram_part(const LexView& v, uint32_t tf, float bc) {
    const float t = (float)tf;
    return __fdiv_rn(__fmul_rn(t, v.k1p), __fadd_rn(t, bc));       // tf_c*(K+1)/(tf_c + cache[len]) (+ SIGMA = 0)
}
// BM25F of an n-gram posting (add_result.rs:1448-1478): idf1*part(tf1) + idf2*part(tf2) [+ idf3*part(tf3)], summed left to right.  It
// replaces the posting's component and fp16 bound (the list's dictionary idf is 1.0, so idf * comp is that sum bit for bit); maxbits
// collects the largest component (positive floats order like their bits) for the coarse bound step.  One thread per n-gram posting (the
// segment by binary search over the segments' first tf slots), one atomic per warp.
__global__ void fill_ngram_bounds(LexView v, const NgSegDev* __restrict__ segs, uint32_t n_segs, const uint16_t* __restrict__ tfs, uint64_t n,
                                  uint32_t* __restrict__ post, float* __restrict__ comp, uint32_t* maxbits) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float c = 0.f;
    if (i < n) {
        uint32_t lo = 0, hi = n_segs;                                  // the last segment whose first slot is <= i
        while (hi - lo > 1) { const uint32_t m = (lo + hi) >> 1; if (segs[m].tf_off <= i) lo = m; else hi = m; }
        const NgSegDev sg = segs[lo];
        const uint64_t p = sg.post_off + (i - sg.tf_off);
        const uint16_t* t = tfs + 3 * i;
        const float bc = __ldg(&v.cache[(v.pay[p] >> 16) & 255u]);
        if (sg.n_comp) {
            c = __fadd_rn(__fmul_rn(sg.idf[0], ngram_part(v, t[0], bc)), __fmul_rn(sg.idf[1], ngram_part(v, t[1], bc)));
            if (sg.n_comp == 3) c = __fadd_rn(c, __fmul_rn(sg.idf[2], ngram_part(v, t[2], bc)));
        }
        comp[p] = c;
        post[p] = (post[p] & 0xFFFFu) | ((uint32_t)__half_as_ushort(__float2half_ru(c)) << 16);
    }
    for (int s = 16; s; s >>= 1) c = fmaxf(c, __shfl_xor_sync(FULL, c, s));
    if ((threadIdx.x & 31) == 0) atomicMax(maxbits, __float_as_uint(c));
}

__global__ void gather_dict(const uint64_t* __restrict__ term_keys, uint32_t n_terms, uint32_t level_idx,
                            uint64_t* __restrict__ keys_out, uint64_t* __restrict__ vals_out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_terms) return;
    keys_out[i] = term_keys[i];
    vals_out[i] = ((uint64_t)level_idx << 32) | i;
}

__global__ void build_entries(const uint64_t* __restrict__ vals, uint32_t n, const uint32_t* const* __restrict__ lvl_offsets,
                              const uint64_t* __restrict__ lvl_base, uint32_t* e_level, uint64_t* e_off, uint32_t* e_count) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t lv = (uint32_t)(vals[i] >> 32), t = (uint32_t)vals[i];
    const uint32_t* po = lvl_offsets[lv];
    uint32_t a = po[t], b = po[t + 1];
    e_level[i] = lv; e_off[i] = lvl_base[lv] + a; e_count[i] = b - a;
}

// one warp per entry: block-max basis (get_max_score, index.rs:2938-3049 — here exact over the list)
__global__ void entry_maxcomp(LexView v, uint32_t n_entries, float* __restrict__ out) {
    uint32_t e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (e >= n_entries) return;
    int lane = threadIdx.x & 31;
    uint64_t off = v.e_off[e]; uint32_t cnt = v.e_count[e];
    float m = 0.f;
    for (uint32_t i = lane; i < cnt; i += 32) m = fmaxf(m, v.comp[off + i]);
    for (int s = 16; s; s >>= 1) m = fmaxf(m, __shfl_xor_sync(FULL, m, s));
    if (lane == 0) out[e] = m;
}

__global__ void mark_dense(const uint32_t* __restrict__ e_count, uint32_t n, uint32_t* flags) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flags[i] = e_count[i] >= DENSE_MIN ? 1u : 0u;
}
__global__ void assign_bitmap(const uint32_t* __restrict__ e_count, const uint32_t* __restrict__ scan, uint32_t n, uint32_t* e_bitmap) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) e_bitmap[i] = e_count[i] >= DENSE_MIN ? scan[i] : NONE;
}
// one CTA (256 threads) per dense entry
__global__ void __launch_bounds__(256) build_bitmaps(const uint32_t* __restrict__ e_bitmap, const uint64_t* __restrict__ e_off,
                                                     const uint32_t* __restrict__ e_count, uint32_t n_entries,
                                                     const uint32_t* __restrict__ post, uint64_t* bm_words, BmSec* bm, uint8_t* bm_q8,
                                                     float q8_step, const uint32_t* __restrict__ dense_list) {
    __shared__ unsigned long long w[1024];
    __shared__ uint32_t pc[1024];
    __shared__ uint32_t mx[1024];      // fp16 bits of the word's largest bound (non-negative halves order like integers)
    uint32_t e = dense_list[blockIdx.x];
    uint32_t b = e_bitmap[e];
    for (int i = threadIdx.x; i < 1024; i += 256) { w[i] = 0ull; mx[i] = 0u; }
    __syncthreads();
    uint64_t off = e_off[e]; uint32_t cnt = e_count[e];
    for (uint32_t i = threadIdx.x; i < cnt; i += 256) {
        const uint32_t pw = post[off + i];
        const uint32_t d = pw & 0xFFFFu;
        atomicOr(&w[d >> 6], 1ull << (d & 63));
        atomicMax(&mx[d >> 6], pw >> 16);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 1024; i += 256) pc[i] = __popcll(w[i]);
    __syncthreads();
    // exclusive prefix over 1024 counts: thread t handles words 4t..4t+3 after a block scan of 4-sums
    __shared__ uint32_t part[256];
    uint32_t s4 = pc[4 * threadIdx.x] + pc[4 * threadIdx.x + 1] + pc[4 * threadIdx.x + 2] + pc[4 * threadIdx.x + 3];
    part[threadIdx.x] = s4;
    __syncthreads();
    for (int d = 1; d < 256; d <<= 1) {
        uint32_t v = threadIdx.x >= d ? part[threadIdx.x - d] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    uint32_t run = part[threadIdx.x] - s4;
    for (int j = 0; j < 4; j++) {
        const int wi = 4 * threadIdx.x + j;
        bm_words[(size_t)b * 1024 + wi] = w[wi];
        BmSec* sec = bm + (size_t)b * 512 + (wi >> 1);
        sec->w[wi & 1] = w[wi];
        sec->meta[wi & 1] = (run & 0xFFFFu) | (mx[wi] << 16);
        sec->pad[wi & 1] = 0u;
        // coarse byte bound: the smallest q with q * step >= word maximum (checked in float, the way the kernels evaluate it)
        uint32_t q = 0;
        if (w[wi]) {
            const float h = __half2float(__ushort_as_half((unsigned short)mx[wi]));
            q = (uint32_t)ceilf(h / q8_step);
            while ((float)q * q8_step < h) q++;
            q = q < 1u ? 1u : (q > 255u ? 255u : q);
        }
        bm_q8[(size_t)b * 1024 + wi] = (uint8_t)q;
        run += pc[wi];
    }
}
__global__ void compact_dense(const uint32_t* __restrict__ e_bitmap, uint32_t n, uint32_t* dense_list) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && e_bitmap[i] != NONE) dense_list[e_bitmap[i]] = i;
}

// ================================================================= record helpers (host + device)
__device__ __forceinline__ uint32_t slot_cnt(const LvSlot& s) { return s.offhi_cnt & 0xFFFFFu; }
__device__ __forceinline__ uint64_t slot_off(const LvSlot& s) { return ((uint64_t)(s.offhi_cnt >> 20) << 32) | s.off_lo; }
__device__ __forceinline__ uint32_t meta_npres(uint32_t m) { return m & 7u; }
__device__ __forceinline__ uint32_t meta_perm(uint32_t m, uint32_t p) { return (m >> (3 + 2 * p)) & 3u; }
__device__ __forceinline__ uint32_t meta_rank(uint32_t m, uint32_t s) { return (m >> (11 + 2 * s)) & 3u; }
__device__ __forceinline__ uint32_t meta_anddrv(uint32_t m) { return (m >> 19) & 3u; }
__device__ __forceinline__ uint32_t meta_cperm(uint32_t m, uint32_t c) { return (m >> (21 + 2 * c)) & 3u; }

// ================================================================= plan kernel
// One CTA per query.  Dictionary lookup (replaces decode_posting_list_object / segment.get, search.rs:2292-2423,
// 3194-3217), live-term list in query order, per-level bound and presence count, levels sorted by bound desc
// (intersection.rs:2224-2225, single.rs:372).  Then one THREAD per (query, level) resolves everything the scoring warp
// would otherwise derive per item with warp-uniform code: directory entries of every term, MAXSCORE order (terms by
// block bound), the in-query-order suffix sums S[p] / R[p], the count order, the AND driver — and writes them as one
// 128-byte record.  Thread 0 finally cuts the sorted record list into work items.
// SORTED (ssb_search_lexical_sorted): every query takes lex_generic, theta / glist are the 128-bit θ and lists, and the levels are ordered
// by the upper bound of the sort key instead of the score bound (its top 32 bits: the order only decides how early θ rises; the exact
// bound goes into the record, rec_sort_bound, for the skip test).
__device__ __forceinline__ void rec_set_sort_bound(LvRec& r, uint64_t b) { r.S[0] = __uint_as_float((uint32_t)b); r.S[1] = __uint_as_float((uint32_t)(b >> 32)); }
__device__ __forceinline__ uint64_t rec_sort_bound(const LvRec& r) { return ((uint64_t)__float_as_uint(r.S[1]) << 32) | __float_as_uint(r.S[0]); }
template <bool SORTED>
__global__ void __launch_bounds__(128) lex_plan(LexView v, const uint32_t* __restrict__ q_off, const uint64_t* __restrict__ q_keys,
                                                const uint8_t* __restrict__ q_flags /*or null*/, const uint32_t* __restrict__ f_off /*or null*/, const uint32_t* __restrict__ f_mask /*or null*/, uint32_t flags /* bit 0 phrase batch, bit 1 no counts wanted, bit 2 the index holds n-gram lists */, uint32_t query_type, QueryPlan* plans, LvRec* recs, uint16_t* item_start, uint32_t* ctr,
                                                uint64_t* theta, int* lock, uint64_t* count, uint64_t* glist, uint32_t n_pow2,
                                                uint32_t item_w, uint32_t first_lim, uint32_t gmax, SortDev sort) {
    extern __shared__ __align__(16) uint8_t sm_raw[];
    float* bound = (float*)sm_raw;                                     // [n_levels]
    uint32_t* cnt = (uint32_t*)(bound + v.n_levels);                   // [n_levels]; after the sort: item weights by sorted position
    uint16_t* ent = (uint16_t*)(cnt + v.n_levels);                     // [FAST_T][n_levels] entry index relative to term.first
    uint64_t* skey = (uint64_t*)(((uintptr_t)(ent + FAST_T * v.n_levels) + 7) & ~(uintptr_t)7);  // [n_pow2]
    __shared__ QTerm st[SSB_MAX_QUERY_TERMS + SSB_MAX_NOT_TERMS];
    __shared__ uint8_t sflag[SSB_MAX_QUERY_TERMS + SSB_MAX_NOT_TERMS];
    __shared__ QueryPlan pl;
    __shared__ uint32_t n_valid;

    const uint32_t q = blockIdx.x;
    const uint32_t nlv = v.n_levels;
    const uint32_t t0 = q_off[q], nt_raw = q_off[q + 1] - t0;
    const uint32_t nt = nt_raw > SSB_MAX_QUERY_TERMS + SSB_MAX_NOT_TERMS ? SSB_MAX_QUERY_TERMS + SSB_MAX_NOT_TERMS : nt_raw;
    if constexpr (SORTED) {
        if (threadIdx.x < 2 * LIST) glist[(size_t)q * 2 * LIST + threadIdx.x] = 0;
        if (threadIdx.x == 0) { theta[2 * q] = 0; theta[2 * q + 1] = 0; lock[q] = 0; count[q] = 0; n_valid = 0; }
    } else {
    if (threadIdx.x < 32) glist[(size_t)q * LIST + threadIdx.x] = 0;
    if (threadIdx.x == 0) { theta[q] = 0; lock[q] = 0; count[q] = 0; n_valid = 0; }
    }
    if (threadIdx.x < nt) {
        uint64_t key = q_keys[t0 + threadIdx.x];
        uint32_t lo = 0, hi = v.n_terms;
        while (lo < hi) { uint32_t m = (lo + hi) >> 1; if (v.dict_keys[m] < key) lo = m + 1; else hi = m; }
        QTerm t; t.first = 0; t.n = 0; t.idf = 0.f; t.df = 0;
        if (lo < v.n_terms && v.dict_keys[lo] == key && v.term_df[lo] > 0) {
            t.first = v.term_first[lo]; t.n = v.term_first[lo + 1] - t.first; t.idf = v.term_idf[lo]; t.df = v.term_df[lo];
        }
        st[threadIdx.x] = t;
        sflag[threadIdx.x] = q_flags ? q_flags[t0 + threadIdx.x] : (uint8_t)0;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t nl = 0, nn = 0; bool missing = false;
        uint32_t n_phr = 0, phr_off = 0;
        for (uint32_t t = 0; t < nt; t++) {
            if (sflag[t] & SSB_TERM_NOT) {                  // '-' terms: exclusion lists, never scored (an unknown NOT term excludes nothing)
                bool dup = false;
                for (uint32_t u = 0; u < nn; u++) dup = dup || pl.tn[u].first == st[t].first;
                if (st[t].n && !dup && nn < SSB_MAX_NOT_TERMS) pl.tn[nn++] = st[t];
                continue;
            }
            if (nl >= SSB_MAX_QUERY_TERMS) continue;
            if (!st[t].n) { missing = true; continue; }
            bool dup = false;                       // the reference scores unique_terms (search.rs:3023-3039): drop repeated keys
            uint32_t uidx = nl;
            for (uint32_t u = 0; u < nl; u++) if (pl.t[u].first == st[t].first) { dup = true; uidx = u; }
            if (!dup) pl.t[nl++] = st[t];
            // phrase: token n_phr of the phrase (term_index_nonunique) is unique term uidx (non_unique_query_list, add_result.rs:3594-3607)
            // an n-gram token spans 2 (bigram) or 3 (trigram) positions: the tokens after it sit 1 or 2 further on (preceding_ngram_count,
            // search.rs:3305-3330).  The offsets stay below 32 + 2 * 31.
            if ((flags & 1u) && n_phr < SSB_MAX_QUERY_TERMS) {
                pl.phr[n_phr] = (uint8_t)uidx; pl.phr_off[n_phr] = (uint8_t)phr_off; n_phr++;
                const uint32_t ty = (flags & 4u) ? (uint32_t)(q_keys[t0 + t] & 7u) : 0u;
                phr_off += ty == 0 ? 1u : (ty <= SSB_NGRAM_RF ? 2u : 3u);
            }
        }
        if ((flags & 1u) && (missing || nl == 0)) n_phr = 0;
        pl.n_phr = ((flags & 1u) && n_phr >= 2 && nl) ? n_phr : 0u;      // a one-token phrase is a plain term query
        // search.rs:3290-3296: AND with an unknown term -> empty result; OR drops the term
        if (query_type == SSB_QUERY_INTERSECTION && missing) nl = 0;
        pl.n_live = nl; pl.n_items = 0; pl.n_recs = 0; pl.n_not = nl ? nn : 0;
        // facet filters: such a query is scored and counted by the one-term-per-lane kernel, which enumerates every match
        pl.filt_first = f_off ? f_off[q] : 0u; pl.n_filt = f_off ? f_off[q + 1] - f_off[q] : 0u;
        pl.field_mask = (f_mask && v.n_fields > 1) ? (f_mask[q] & ((1u << v.n_fields) - 1u)) : 0u;   // one indexed field: the filter can never reject
        // facet-filtered queries stay on the record path when nothing has to be counted (flags bit 1): lex_score tests the filter on the
        // exact-score survivors; with counts every match must be tested -> lex_generic
        pl.fast = (nl <= v.fast_t && (pl.n_filt == 0 || (flags & 2u)) && pl.field_mask == 0 && pl.n_phr == 0) ? 1u : 0u;
        if constexpr (SORTED) pl.fast = 0;
    }
    for (uint32_t b = threadIdx.x; b < nlv; b += blockDim.x) {
        bound[b] = 0.f; cnt[b] = 0;
        for (uint32_t t = 0; t < FAST_T; t++) ent[t * nlv + b] = (uint16_t)ENT_NONE;
    }
    __syncthreads();
    const uint32_t nl = pl.n_live;
    const bool fastq = pl.fast != 0;
    for (uint32_t t = 0; t < nl; t++) {   // QUERY ORDER: the bound is summed exactly like a score would be
        const QTerm qt = pl.t[t];
        for (uint32_t e = threadIdx.x; e < qt.n; e += blockDim.x) {
            uint32_t lv = v.e_level[qt.first + e];
            bound[lv] = __fadd_rn(bound[lv], __fmul_rn(qt.idf, v.e_maxcomp[qt.first + e]));
            cnt[lv] += 1;
            if (t < FAST_T) ent[t * nlv + lv] = (uint16_t)e;
        }
        __syncthreads();
    }
    for (uint32_t b = threadIdx.x; b < n_pow2; b += blockDim.x) {
        uint64_t key = 0;
        if (b < nlv) {
            bool ok = query_type == SSB_QUERY_INTERSECTION ? (nl > 0 && cnt[b] == nl) : (cnt[b] > 0);
            if constexpr (SORTED) {
                if (ok) { key = (level_sort_bound(sort, v.level_ids[b]) & 0xFFFFFFFF00000000ull) | (uint64_t)(0xFFFFFFFFu - b); atomicAdd(&n_valid, 1u); }
            } else
            if (ok) { key = ((uint64_t)ord_f32(bound[b]) << 32) | (uint64_t)(0xFFFFFFFFu - b); atomicAdd(&n_valid, 1u); }
        }
        skey[b] = key;
    }
    __syncthreads();
    // bitonic sort, descending
    for (uint32_t size = 2; size <= n_pow2; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t i = threadIdx.x; i < n_pow2 / 2; i += blockDim.x) {
                uint32_t lo = 2 * i - (i & (stride - 1));   // index with bit `stride` cleared
                uint32_t hi = lo + stride;
                bool desc = (lo & size) == 0;
                uint64_t a = skey[lo], b = skey[hi];
                if (desc ? (a < b) : (a > b)) { skey[lo] = b; skey[hi] = a; }
            }
            __syncthreads();
        }
    }
    // ---- one thread per sorted position: the resolved record ----
    const uint32_t nv = n_valid;
    const bool is_and = query_type == SSB_QUERY_INTERSECTION;
    for (uint32_t j = threadIdx.x; j < nv; j += blockDim.x) {
        const uint32_t lv = 0xFFFFFFFFu - (uint32_t)skey[j];
        LvRec r;
        r.docbase = v.level_ids[lv] << 16; r.bound = bound[lv]; r.lv = lv;
        uint32_t c0 = 0, c1 = 0, c2 = 0, c3 = 0; float u0 = 0.f, u1 = 0.f, u2 = 0.f, u3 = 0.f;
        uint32_t weight = item_w;
        uint32_t meta = 0;
#pragma unroll
        for (uint32_t s = 0; s < FAST_T; s++) {
            LvSlot sl; sl.off_lo = 0; sl.offhi_cnt = 0; sl.bmi = NONE; sl.ub = 0.f;
            float idf = 0.f;
            if (s < nl && fastq) {
                const QTerm qt = pl.t[s];
                idf = qt.idf;
                const uint32_t er = ent[s * nlv + lv];
                if (er != ENT_NONE) {
                    const uint32_t e = qt.first + er;
                    const uint64_t off = v.e_off[e]; const uint32_t c = v.e_count[e];
                    sl.off_lo = (uint32_t)off; sl.offhi_cnt = ((uint32_t)(off >> 32) << 20) | c; sl.bmi = v.e_bitmap[e];
                    sl.ub = __fmul_rn(qt.idf, v.e_maxcomp[e]);
                    if (s == 0) { c0 = c; u0 = sl.ub; } else if (s == 1) { c1 = c; u1 = sl.ub; } else if (s == 2) { c2 = c; u2 = sl.ub; } else { c3 = c; u3 = sl.ub; }
                }
            }
            r.t[s] = sl; r.idf[s] = idf;
        }
        if (fastq) {
            const uint32_t cs[4] = {c0, c1, c2, c3}; const float us[4] = {u0, u1, u2, u3};
            uint32_t np = 0, rank[4], crank[4];
#pragma unroll
            for (int s = 0; s < 4; s++) np += cs[s] ? 1u : 0u;
#pragma unroll
            for (int s = 0; s < 4; s++) {
                uint32_t rk = 0, ck = 0;
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    if (u == s || !cs[u]) continue;
                    if (us[u] > us[s] || (us[u] == us[s] && u < s)) rk++;
                    if (cs[u] > cs[s] || (cs[u] == cs[s] && u < s)) ck++;
                }
                rank[s] = cs[s] ? rk : 3u; crank[s] = cs[s] ? ck : 3u;
            }
            uint32_t perm = 0, cperm = 0, rankbits = 0, and_drv = 0;
#pragma unroll
            for (int s = 0; s < 4; s++) {
                if (!cs[s]) continue;
                perm |= (uint32_t)s << (2 * rank[s]); cperm |= (uint32_t)s << (2 * crank[s]); rankbits |= rank[s] << (2 * s);
                if (crank[s] == np - 1) and_drv = s;            // the shortest list drives an intersection (intersection.rs:258-273)
            }
            meta = np | (perm << 3) | (rankbits << 11) | (and_drv << 19) | (cperm << 21) | (nl << 29);
#pragma unroll
            for (int p = 0; p < 4; p++) {
                float S = 0.f, R = 0.f;
#pragma unroll
                for (int s = 0; s < 4; s++) {   // query order
                    if (!cs[s]) continue;
                    if (is_and) { if (p == 0) { S = __fadd_rn(S, us[s]); if ((uint32_t)s != and_drv) R = __fadd_rn(R, us[s]); } }
                    else { if (rank[s] >= (uint32_t)p) S = __fadd_rn(S, us[s]); if (rank[s] > (uint32_t)p) R = __fadd_rn(R, us[s]); }
                }
                r.S[p] = S; r.R[p] = R;
            }
            uint32_t wsl = is_and ? and_drv : (perm & 3u);
            weight = cs[wsl];
        } else {
            meta = (nl < 7u ? nl : 7u) << 29;
#pragma unroll
            for (int p = 0; p < 4; p++) { r.S[p] = 0.f; r.R[p] = 0.f; }
            // lex_generic does not read S[].  A sorted query's items take up to gmax levels whatever their lists' lengths: the warp's own
            // list then bounds the later (lower-bound) levels of its item, which it skips without waiting for θ
            if constexpr (SORTED) { rec_set_sort_bound(r, level_sort_bound(sort, v.level_ids[lv])); weight = 0; }
        }
        r.meta = meta;
        const uint4* src = reinterpret_cast<const uint4*>(&r);
        uint4* dst = reinterpret_cast<uint4*>(recs + (size_t)q * nlv + j);
#pragma unroll
        for (int i = 0; i < 8; i++) dst[i] = src[i];
        cnt[j] = weight;                                        // (cnt[] by level is dead after the key build above)
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        // items: consecutive records of the bound-sorted list, <= GMAX levels and ~ITEM_W postings of their top lists each.
        // The first item stays small so that the query's threshold is published early.
        uint16_t* is = item_start + (size_t)q * (nlv + 1);
        uint32_t ni = 0, acc = 0, nin = 0;
        is[0] = 0;
        for (uint32_t j = 0; j < nv; j++) {
            const uint32_t lim = ni == 0 ? first_lim : gmax;
            const uint32_t w = cnt[j] + 64u;
            if (nin > 0 && (nin >= lim || acc + w > item_w)) { ni++; is[ni] = (uint16_t)j; acc = 0; nin = 0; }
            acc += w; nin++;
        }
        if (nv) { ni++; is[ni] = (uint16_t)nv; }
        pl.n_items = ni; pl.n_recs = nv;
        plans[q] = pl;
        atomicMax(&ctr[1], ni);
        if (!pl.fast) atomicOr(&ctr[4], 1u);
        if (pl.n_not) atomicOr(&ctr[5], 1u);
    }
}

// ================================================================= scoring kernel
struct TermRegs {   // generic path: lane t holds query term t of the current item
    uint32_t cnt; uint64_t off; uint32_t bmi; float idf; float ub;
};

// The term directory and the list arenas, by value for the out-of-line predicates: a LexView reference would force the whole view
// onto the thread stack.  The helpers below take either this or a LexView (V).
struct ListView { const uint32_t* e_level; const uint32_t* e_count; const uint32_t* e_bitmap; const uint32_t* post; const uint64_t* e_off;
                  const BmSec* bm; const uint64_t* bm_words; };
__device__ __forceinline__ ListView list_view(const LexView& v) { return ListView{v.e_level, v.e_count, v.e_bitmap, v.post, v.e_off, v.bm, v.bm_words}; }

// directory entry e of term qt at local level lv (a term's entries ascend by level); false = the term has no list there.  qt by value:
// its fields are loaded once up front, as the callers' copies did.  A bool, not an index-or-NONE, so that callers branch on the search.
template <class V>
__device__ __forceinline__ bool find_entry(const V& v, QTerm qt, uint32_t lv, uint32_t& e) {
    uint32_t a = 0, b = qt.n;
    while (a < b) { const uint32_t m = (a + b) >> 1; if (__ldg(&v.e_level[qt.first + m]) < lv) a = m + 1; else b = m; }
    if (a < qt.n && __ldg(&v.e_level[qt.first + a]) == lv) { e = qt.first + a; return true; }
    return false;
}

// membership + rank probe of doc d in the list described by (cnt, off, bmi)
template <class V>
__device__ __forceinline__ bool probe(const V& v, uint32_t cnt, uint64_t off, uint32_t bmi, uint32_t d, uint32_t& rank) {
    if (bmi != NONE) {
        // word + rank sit in the same 32-byte sector: one DRAM access, two independent loads
        const BmSec* sec = v.bm + (size_t)bmi * 512 + (d >> 7);
        const uint64_t w = __ldg(&sec->w[(d >> 6) & 1u]);
        const uint32_t r0 = __ldg(&sec->meta[(d >> 6) & 1u]) & 0xFFFFu;
        rank = r0 + (uint32_t)__popcll(w & ((1ull << (d & 63)) - 1ull));
        return ((w >> (d & 63)) & 1ull) != 0;
    }
    uint32_t lo = 0, hi = cnt;
    const uint32_t* a = v.post + off;
    while (lo < hi) { uint32_t m = (lo + hi) >> 1; if ((__ldg(&a[m]) & 0xFFFFu) < d) lo = m + 1; else hi = m; }
    rank = lo;
    return lo < cnt && (__ldg(&a[lo]) & 0xFFFFu) == d;
}
// membership only
template <class V>
__device__ __forceinline__ bool present_in(const V& v, uint32_t cnt, uint64_t off, uint32_t bmi, uint32_t d) {
    if (bmi != NONE) return ((__ldg(&v.bm_words[(size_t)bmi * 1024 + (d >> 6)]) >> (d & 63)) & 1ull) != 0;
    uint32_t lo = 0, hi = cnt;
    const uint32_t* a = v.post + off;
    while (lo < hi) { uint32_t m = (lo + hi) >> 1; if ((__ldg(&a[m]) & 0xFFFFu) < d) lo = m + 1; else hi = m; }
    return lo < cnt && (__ldg(&a[lo]) & 0xFFFFu) == d;
}
// is doc d in term qt's list at local level lv?
template <class V>
__device__ __forceinline__ bool term_has(const V& v, QTerm qt, uint32_t lv, uint32_t d) {
    uint32_t e;
    if (!find_entry(v, qt, lv, e)) return false;
    const uint32_t cnt = __ldg(&v.e_count[e]), bmi = __ldg(&v.e_bitmap[e]); const uint64_t off = __ldg(&v.e_off[e]);
    return present_in(v, cnt, off, bmi, d);
}
// the posting of doc d in term qt's list at local level lv: false when the term has no list there or d is not in it
__device__ __forceinline__ bool find_posting(const ListView& v, QTerm qt, uint32_t lv, uint32_t d, uint64_t& pos) {
    uint32_t e;
    if (!find_entry(v, qt, lv, e)) return false;
    const uint32_t cnt = __ldg(&v.e_count[e]), bmi = __ldg(&v.e_bitmap[e]); const uint64_t off = __ldg(&v.e_off[e]);
    uint32_t rank;
    if (!probe(v, cnt, off, bmi, d, rank)) return false;
    pos = off + rank;
    return true;
}

__device__ __forceinline__ float term_score(const LexView& v, float idf, uint64_t pos) {
    // idf * ((tf*(K+1)/(tf+comp)) + SIGMA), SIGMA = 0 (x + 0.0 == x); the bracket is precomputed at commit (fill_bounds)
    return __fmul_rn(idf, __ldg(&v.comp[pos]));
}
// bm25f += the term's contribution, generic path.  One field: bm25f += idf * comp (add_result.rs:1450).  Several fields
// (get_bm25f_multiterm_multifield, add_result.rs:1232-1262): for each field the term occurs in, ascending, bm25f += weight * idf * comp_f,
// evaluated left to right and accumulated straight into the running sum.
__device__ __forceinline__ float acc_term(const LexView& v, float score, float idf, uint64_t pos) {
    if (v.n_fields <= 1) return __fadd_rn(score, term_score(v, idf, pos));
    for (uint32_t f = 0; f < v.n_fields; f++) {
        const float cf = __ldg(&v.compf[pos * v.n_fields + f]);
        if (cf != 0.f) score = __fadd_rn(score, __fmul_rn(__fmul_rn(v.boost[f], idf), cf));
    }
    return score;
}

// shard.delete_hashset.contains(docid) (add_result.rs:3435): one table lookup + one bitmap word, only for exact-score survivors
__device__ __forceinline__ bool is_deleted(const LexView& v, uint32_t doc) {
    if (!v.del_slot) return false;
    const uint32_t slot = __ldg(&v.del_slot[doc >> 16]);
    if (slot == NONE) return false;
    return ((__ldg(&v.del_words[(size_t)slot * 1024 + ((doc & 0xFFFFu) >> 6)]) >> (doc & 63u)) & 1ull) != 0;
}

// not_query_list (add_result.rs:3440-3496): is doc d of local level lv in one of the query's NOT lists?  Out of line and fed by
// value (ListView) — the call sits on the rare survivor path.
__device__ __noinline__ bool in_not_lists_impl(ListView v, const QueryPlan* pl, uint32_t n_not, uint32_t lv, uint32_t d) {
    for (uint32_t i = 0; i < n_not; i++) if (term_has(v, pl->tn[i], lv, d)) return true;
    return false;
}
__device__ __forceinline__ bool in_not_lists(const LexView& v, const QueryPlan* pl, uint32_t n_not, uint32_t lv, uint32_t d) {
    return in_not_lists_impl(list_view(v), pl, n_not, lv, d);
}

// field_filter (`field_filter_set`, add_result.rs:3124-3137, 3558-3571): every query term the doc contains must occur in at least one
// field of the filter — tested only when (fields the term occurs in) + (fields of the filter) <= indexed fields, otherwise they overlap for
// certain.  The score still sums every field.  true = the doc is filtered OUT.  Out of line, on the filtered path of lex_generic only.
__device__ __noinline__ bool field_rejects_impl(ListView v, const uint32_t* payf, uint32_t n_fields, const QueryPlan* pl, uint32_t n_live, uint32_t lv,
                                                uint32_t d, uint32_t field_mask) {
    const uint32_t n_filter = (uint32_t)__popc(field_mask);
    for (uint32_t t = 0; t < n_live; t++) {
        uint64_t pos;
        if (!find_posting(v, pl->t[t], lv, d, pos)) continue;           // the doc does not contain this term (OR)
        uint32_t present = 0;
        for (uint32_t f = 0; f < n_fields; f++) if (__ldg(&payf[pos * n_fields + f]) & 0xFFFFu) present |= 1u << f;
        if ((uint32_t)__popc(present) + n_filter <= n_fields && !(present & field_mask)) return true;
    }
    return false;
}
// Phrase check (add_result.rs:3586-3684): the doc (already known to contain every term) matches iff some start position p has token i of
// the phrase at p + i for every i — the reference finds it by a k-way merge of the tokens' position lists aligned by their index in the
// phrase (term_index_nonunique); the same merge here, one thread per candidate doc (rare path, out of line).  Unique term u's positions
// are positions[ubase[u] .. + utf[u]); true = some start s has token i at s + phr_off[i] for every i (phrasematch_count >= 1); phr_off[i]
// is i unless an earlier token is an n-gram.  OFFS = false (several indexed fields, which hold no n-gram lists): the offsets are i.  The cursors `cur`
// (one per token) are an array of the calling check, on the thread's stack: declared there, after its own arrays, they keep that
// function's frame layout and with it the register allocation of lex_generic<true>.
template <bool OFFS>
__device__ __forceinline__ bool phrase_in_runs(const uint16_t* positions, const QueryPlan* pl, const uint64_t* ubase, const uint32_t* utf, uint32_t* cur) {
    const uint32_t m = pl->n_phr, u0 = pl->phr[0];
    for (uint32_t i = 0; i < m; i++) cur[i] = 0;
    while (cur[0] < utf[u0]) {                                               // anchor = token 0
        const uint32_t s = __ldg(&positions[ubase[u0] + cur[0]]);
        bool all = true; uint32_t next_s = s;
        for (uint32_t i = 1; i < m; i++) {
            const uint32_t u = pl->phr[i];
            const uint32_t o = OFFS ? (uint32_t)pl->phr_off[i] : i;
            while (cur[i] < utf[u] && (uint32_t)__ldg(&positions[ubase[u] + cur[i]]) < s + o) cur[i]++;
            if (cur[i] >= utf[u]) return false;                             // a token's positions are exhausted: no (further) match
            const uint32_t p = __ldg(&positions[ubase[u] + cur[i]]);
            if (p != s + o) { all = false; next_s = p - o; break; }          // p > s + o: the start must move up to at least p - o
        }
        if (all) return true;
        while (cur[0] < utf[u0] && (uint32_t)__ldg(&positions[ubase[u0] + cur[0]]) < next_s) cur[0]++;
    }
    return false;
}
struct PhraseArgs { const uint32_t* pay; const uint16_t* positions; const uint32_t* pos_off; const uint64_t* lvl_pos_base; };
__device__ __noinline__ bool phrase_rejects_impl(ListView v, PhraseArgs a, const QueryPlan* pl, uint32_t n_live, uint32_t lv, uint32_t d) {
    uint64_t ubase[SSB_MAX_QUERY_TERMS]; uint32_t utf[SSB_MAX_QUERY_TERMS];
    const uint64_t lbase = __ldg(&a.lvl_pos_base[lv]);
    for (uint32_t t = 0; t < n_live; t++) {
        uint64_t pos;
        if (!find_posting(v, pl->t[t], lv, d, pos)) return true;
        ubase[t] = lbase + __ldg(&a.pos_off[pos]);
        utf[t] = __ldg(&a.pay[pos]) & 0xFFFFu;
    }
    uint32_t cur[SSB_MAX_QUERY_TERMS];
    return !phrase_in_runs<true>(a.positions, pl, ubase, utf, cur);
}
// Several indexed fields (add_result.rs:3247-3389): a posting's positions are one run per field, field 0 first, each restarting from 0, of
// the posting's per-field tfs (a.pay = payf here).  The same merge as above runs field by field on those runs only — a phrase never spans two
// fields: field f is searched when every unique term occurs in it and, if the query has a field filter (pl->field_mask != 0), when f is in
// the filter (field_filter_set.contains).  The doc matches on the first field that holds the phrase.  Out of line like the single-field
// check and only in lex_generic<true>, so that the single-field kernel keeps its code.
__device__ __noinline__ bool phrase_rejects_fields_impl(ListView v, PhraseArgs a, const QueryPlan* pl, uint32_t n_live, uint32_t lv, uint32_t d,
                                                        uint32_t n_fields) {
    uint64_t ubase[SSB_MAX_QUERY_TERMS], ftf[SSB_MAX_QUERY_TERMS];       // per unique term: its first position in field 0, its tfs (16 bits per field)
    uint32_t utf[SSB_MAX_QUERY_TERMS];
    const uint64_t lbase = __ldg(&a.lvl_pos_base[lv]);
    for (uint32_t t = 0; t < n_live; t++) {
        uint64_t pos;
        if (!find_posting(v, pl->t[t], lv, d, pos)) return true;
        ubase[t] = lbase + __ldg(&a.pos_off[pos]);
        uint64_t tfs = 0;
        for (uint32_t f = 0; f < n_fields; f++) tfs |= (uint64_t)(__ldg(&a.pay[pos * n_fields + f]) & 0xFFFFu) << (16 * f);
        ftf[t] = tfs;
    }
    const uint32_t field_mask = pl->field_mask;
    uint32_t cur[SSB_MAX_QUERY_TERMS];
    for (uint32_t f = 0; f < n_fields; f++) {
        bool in_all = true;
        for (uint32_t t = 0; t < n_live; t++) {
            if (f) ubase[t] += utf[t];                                       // field f's run follows the run of field f - 1
            utf[t] = (uint32_t)(ftf[t] >> (16 * f)) & 0xFFFFu;
            in_all = in_all && utf[t] != 0;
        }
        if (!in_all || (field_mask && !((field_mask >> f) & 1u))) continue;
        if (phrase_in_runs<false>(a.positions, pl, ubase, utf, cur)) return false;
    }
    return true;
}
// facet filters, the field filter and the phrase check of one query on one doc: true = filtered OUT.  FIELD_RUNS: the index has several
// fields and a phrase batch is running (positions in per-field runs) — its own instantiation of lex_generic, so that the single-field kernel
// keeps its code and register allocation
template <bool FIELD_RUNS, bool GEO>
__device__ __forceinline__ bool filters_reject(const LexView& v, const QueryPlan* pl, uint32_t f0, uint32_t nf, uint32_t field_mask, uint32_t n_live, uint32_t lv, uint32_t d, uint32_t doc) {
    if (nf && facet_rejects<GEO>(v, f0, nf, doc)) return true;
    if (field_mask && field_rejects_impl(list_view(v), v.payf, v.n_fields, pl, n_live, lv, d, field_mask)) return true;
    if (!FIELD_RUNS && pl->n_phr && phrase_rejects_impl(list_view(v), PhraseArgs{v.pay, v.positions, v.pos_off, v.lvl_pos_base}, pl, n_live, lv, d)) return true;
    if (FIELD_RUNS && pl->n_phr && phrase_rejects_fields_impl(list_view(v), PhraseArgs{v.payf, v.positions, v.pos_off, v.lvl_pos_base}, pl, n_live, lv, d,
                                                              v.n_fields)) return true;
    return false;
}

__device__ __forceinline__ float bound_of_word(uint32_t w) { return __half2float(__ushort_as_half((unsigned short)(w >> 16))); }

__device__ __forceinline__ void insert_candidates(uint64_t& L, uint32_t& thr, bool cand, float score, uint32_t doc,
                                                  uint32_t k, int lane, bool& dirty, uint64_t ceil) {
    // `ceil`: exclusive upper bound on keys (paging beyond 32 results: everything >= ceil was returned by an earlier page)
    const uint64_t key = pack_key(score, doc);
    unsigned m = __ballot_sync(FULL, cand && key < ceil);
    if (!m) return;
    while (m) {
        int src = __ffs(m) - 1; m &= m - 1;
        wl_insert(L, shfl64(key, src), lane);
    }
    dirty = true;
    uint32_t kth = (uint32_t)(shfl64(L, (int)k - 1) >> 32);
    if (kth > thr) thr = kth;
}

struct ItemCtx {
    uint32_t q, lv, n, k, docbase, bound_ord, n_not, n_filt /* facet filters + (field filter ? 1 : 0): 0 = unfiltered query */, n_facet_filt, filt_first, field_mask;
    uint64_t ceil, ceil_lo /* sorted batches: the ceiling is the 128-bit key (ceil, ceil_lo) */;
    bool scoring, need_count, is_and;
};

struct WarpSm { LvRec recs[GMAX]; uint2 queue[QCAP]; uint4 q2[64]; const QueryPlan* pl; uint32_t n_not; uint32_t nq2; uint32_t it_base; unsigned it_mask; uint32_t n_filt, filt_first /* facet filters of the item's query (HAS_NOT instantiations) */; };   // 1024 + 1536 + 1024 + 32 B per warp

// thresholds derived from the ordered-uint k-th score `thr` (0 = list not full yet): BM25 scores are non-negative, so
// the per-posting tests are plain float compares against thr_lo = thr_f / INFL (rounded down).
struct Thr {
    uint32_t u; float lo;
    __device__ __forceinline__ void set(uint32_t t) { u = t; lo = t ? __fdiv_rd(unord_f32(t), INFL) : -1.0f; }
};

// ---- stage 3 on up to 32 survivors of stage 2 (queue 2, full lanes): exact in-query-order score (add_result.rs:1450-1452).
// Entry: x = pos(17) | record(3) | driver rank(2) | 4 x 2 flag bits (0 absent, 1 present at the stored rank, 3 no bitmap: search),
// y = the driver's posting word, z / w = posting ranks of slots 0..3 inside their lists (u16 each).  Every address is known up front:
// the component loads of all terms are independent (one memory latency), the IEEE divide and the cache lookup happened at commit.
template <bool IS_AND, bool HAS_NOT>
__device__ __forceinline__ void score_queued(const LexView& v, const WarpSm& w, uint4 e, bool active, int lane, uint32_t k, uint64_t ceil,
                                             uint64_t& L, Thr& thr, bool& dirty, uint32_t& st_probes) {
    const uint32_t pos = e.x & 0x1FFFFu, ri = (e.x >> 17) & 7u, p = (e.x >> 20) & 3u;
    const uint32_t d = e.y & 0xFFFFu;
    const LvRec& rec = w.recs[ri];
    const uint32_t meta = rec.meta;
    const uint32_t drv = IS_AND ? meta_anddrv(meta) : meta_perm(meta, p);
    bool alive = active;
    float comp[FAST_T];
#pragma unroll
    for (uint32_t s = 0; s < FAST_T; s++) {
        const uint32_t fl = s == drv ? 1u : ((e.x >> (22 + 2 * s)) & 3u);
        const uint32_t rank = s == drv ? pos : ((s & 2 ? e.w : e.z) >> (16 * (s & 1))) & 0xFFFFu;
        comp[s] = 0.f;
        if (active && fl == 1u) comp[s] = __ldg(&v.comp[slot_off(rec.t[s]) + rank]);
    }
    float score = 0.f;
#pragma unroll
    for (uint32_t s = 0; s < FAST_T; s++) {
        if (!alive) continue;
        const uint32_t fl = s == drv ? 1u : ((e.x >> (22 + 2 * s)) & 3u);
        if (fl == 0u) continue;
        float c = comp[s];
        if (fl == 3u) {                                      // list without a bitmap (< 256 postings): binary search now
            uint32_t rank; st_probes++;
            const uint64_t soff = slot_off(rec.t[s]);
            if (!probe(v, slot_cnt(rec.t[s]), soff, NONE, d, rank)) { if (IS_AND) alive = false; continue; }
            if (!IS_AND && meta_rank(meta, s) < p) { alive = false; continue; }   // already emitted when that term was the driver
            c = __ldg(&v.comp[soff + rank]);
        }
        score = __fadd_rn(score, __fmul_rn(rec.idf[s], c));
    }
    uint32_t t = thr.u;
    alive = alive && ord_f32(score) >= thr.u;
    if (alive && is_deleted(v, rec.docbase | d)) alive = false;
    if (HAS_NOT) {   // per-survivor predicates: their own kernel instantiation, the common one carries no out-of-line call
        if (alive && w.n_not && in_not_lists(v, w.pl, w.n_not, rec.lv, d)) alive = false;                       // '-' terms (not_query_list)
        if (alive && w.n_filt && facet_rejects(v, w.filt_first, w.n_filt, rec.docbase | d)) alive = false;      // facet filters (Topk: record path)
    }
    insert_candidates(L, t, alive, score, rec.docbase | d, k, lane, dirty, ceil);
    if (t != thr.u) thr.set(t);
}

// ---- stage 2 on up to 32 survivors of the stream filter (queue 1; lanes may belong to different records / drivers): replace the
// level-wide bound by what the bitmap sectors say about THIS doc.  One 32-byte sector per bitmap-backed term holds the membership
// word, the posting rank before the word and the largest fp16 bound of the word's 64 docs: (OR) a doc that is in an earlier-ranked
// list was already emitted there, a term the doc is not in contributes nothing, and a term it is in contributes at most
// idf * (word maximum); (AND) a doc missing from any list is dead.  Lists without a bitmap count as "maybe".  Survivors go to
// queue 2 together with the ranks found, so that stage 3 runs on 32 of them at a time. ----
template <bool IS_AND, bool HAS_NOT>
__device__ __forceinline__ void filter_queued(const LexView& v, WarpSm& w, uint2 e, bool active, bool flush2, int lane, uint32_t k, uint64_t ceil,
                                              uint64_t& L, Thr& thr, bool& dirty, uint32_t& st_probes) {
    const uint32_t ri = (e.x >> 17) & 7u, p = (e.x >> 20) & 3u;
    const uint32_t d = e.y & 0xFFFFu;
    const LvRec& rec = w.recs[ri];
    const uint32_t meta = rec.meta;
    const uint32_t drv = IS_AND ? meta_anddrv(meta) : meta_perm(meta, p);
    uint64_t bw[FAST_T]; uint32_t bm[FAST_T];
    uint32_t bmi[FAST_T], cnts[FAST_T];
#pragma unroll
    for (uint32_t s = 0; s < FAST_T; s++) {
        cnts[s] = slot_cnt(rec.t[s]); bmi[s] = rec.t[s].bmi;
        const bool need = active && s != drv && cnts[s] != 0 && bmi[s] != NONE;
        const BmSec* sec = v.bm + (size_t)bmi[s] * 512 + (d >> 7);
        bw[s] = need ? __ldg(&sec->w[(d >> 6) & 1u]) : 0ull;
        bm[s] = need ? __ldg(&sec->meta[(d >> 6) & 1u]) : 0u;          // same sector as the word
        st_probes += need ? 1u : 0u;
    }
    float B = rec.idf[drv] * bound_of_word(e.y);
    bool dead = !active;
    uint32_t flags = 0, r01 = 0, r23 = 0;
#pragma unroll
    for (uint32_t s = 0; s < FAST_T; s++) {
        if (s == drv || cnts[s] == 0) continue;
        const uint32_t rk = meta_rank(meta, s);
        if (bmi[s] != NONE) {
            const bool pres = ((bw[s] >> (d & 63)) & 1ull) != 0;
            if (!pres) { if (IS_AND) dead = true; continue; }
            if (!IS_AND && rk < p) { dead = true; continue; }
            B += rec.idf[s] * bound_of_word(bm[s]);                       // meta = rank16 | (fp16 word maximum) << 16
            const uint32_t rank = (bm[s] & 0xFFFFu) + (uint32_t)__popcll(bw[s] & ((1ull << (d & 63)) - 1ull));
            flags |= 1u << (2 * s);
            if (s & 2) r23 |= rank << (16 * (s & 1)); else r01 |= rank << (16 * (s & 1));
        } else {
            if (IS_AND || rk > p) B += rec.t[s].ub;
            flags |= 3u << (2 * s);
        }
    }
    const bool alive = !dead && B >= thr.lo;
    const unsigned m = __ballot_sync(FULL, alive);
    uint32_t n2 = w.nq2;
    if (alive) w.q2[n2 + __popc(m & ((1u << lane) - 1u))] = make_uint4((e.x & 0x3FFFFFu) | (flags << 22), e.y, r01, r23);
    n2 += __popc(m);
    __syncwarp();
#pragma unroll 1
    while (n2 >= 32u || (flush2 && n2)) {                    // the ONE place exact scores are computed (code size: instruction cache)
        const bool act = (uint32_t)lane < n2;
        const uint4 e4 = act ? w.q2[lane] : make_uint4(0u, 0u, 0u, 0u);
        __syncwarp();
        score_queued<IS_AND, HAS_NOT>(v, w, e4, act, lane, k, ceil, L, thr, dirty, st_probes);
        const uint32_t rem = n2 > 32u ? n2 - 32u : 0u;
        uint4 tmp = make_uint4(0u, 0u, 0u, 0u);
        if ((uint32_t)lane < rem) tmp = w.q2[32 + lane];
        __syncwarp();
        if ((uint32_t)lane < rem) w.q2[lane] = tmp;
        n2 = rem;
        __syncwarp();
    }
    if (lane == 0) w.nq2 = n2;
    __syncwarp();
}

// drain full batches of the survivor queue; keeps < 32 entries at the front.  flush: everything goes, queue 2 included (one
// batch runs even when queue 1 is empty, so that the leftovers of queue 2 get their exact score).
template <bool IS_AND, bool HAS_NOT>
__device__ __forceinline__ void drain_queue(const LexView& v, WarpSm& w, uint32_t& nq_in, bool flush, int lane, uint32_t k, uint64_t ceil,
                                            uint64_t& L, Thr& thr, bool& dirty, uint32_t& st_probes) {
    uint32_t head = 0;
#pragma unroll 1
    for (;;) {
        const bool act = head + (uint32_t)lane < nq_in;
        const bool lastb = flush && head + 32u >= nq_in;
        const uint2 e = act ? w.queue[head + lane] : make_uint2(0u, 0u);
        filter_queued<IS_AND, HAS_NOT>(v, w, e, act, lastb, lane, k, ceil, L, thr, dirty, st_probes);
        head = head + 32u < nq_in ? head + 32u : nq_in;
        if (flush ? head >= nq_in : nq_in - head < 32u) break;
    }
    const uint32_t rem = nq_in - head;
    uint2 tmp = make_uint2(0u, 0u);
    if ((uint32_t)lane < rem) tmp = w.queue[head + lane];
    __syncwarp();
    if ((uint32_t)lane < rem) w.queue[lane] = tmp;
    __syncwarp();
    nq_in = rem;
}

// coarse per-word bounds of the terms a driven posting may still collect from (OR: MAXSCORE rank > p; AND: every other term):
// dense lists contribute cf * q8[d >> 6] (q8 = 0: no posting of that term within the 64 docs around d), the others their list
// maximum, folded into `base`.  Warp-uniform.
struct Coarse { uint32_t off[FAST_T - 1]; float cf[FAST_T - 1]; uint32_t n; float base; };

template <bool IS_AND>
__device__ __forceinline__ Coarse coarse_of(const LexView& v, const LvRec& rec, uint32_t drv, uint32_t p) {
    Coarse c; c.n = 0; c.base = 0.f;
#pragma unroll
    for (uint32_t j = 0; j < FAST_T - 1; j++) { c.off[j] = 0; c.cf[j] = 0.f; }
#pragma unroll
    for (uint32_t s = 0; s < FAST_T; s++) {
        if (s == drv || slot_cnt(rec.t[s]) == 0) continue;
        if (!IS_AND && meta_rank(rec.meta, s) < p) continue;
        if (rec.t[s].bmi != NONE) {
#pragma unroll
            for (uint32_t j = 0; j < FAST_T - 1; j++) if (j == c.n) { c.off[j] = rec.t[s].bmi * 1024u; c.cf[j] = rec.idf[s] * v.q8_step; }
            c.n++;
        } else c.base += rec.t[s].ub;
    }
    return c;
}

// stream one list 128 postings per iteration (one 16-byte load per lane) and queue the postings whose bound reaches θ.
// The bound of a posting is idf * (its own fp16 component bound) + the coarse bounds of the other terms AT ITS DOC ID (a byte
// per 64 docs, L1-resident: 1 KB per dense list) — the sector probes of stage 2 are only paid by postings that pass it.
template <bool IS_AND, bool HAS_NOT>
__device__ __forceinline__ void stream_driver(const LexView& v, WarpSm& w, uint32_t tag /* ri<<17 | p<<20 */, uint64_t doff, uint32_t dcnt,
                                              float didf, float R, const Coarse& co, bool flush, uint32_t& nq_in, int lane, uint32_t k, uint64_t ceil,
                                              uint64_t& L, Thr& thr, bool& dirty, uint32_t& st_probes) {
    // 32-bit indices relative to the 16-byte aligned start: the list occupies [r0, r1) of the words fetched
    // (flush: dcnt = 0 and one empty iteration whose only effect is the final drain — one call site for everything downstream)
    const uint32_t r0 = (uint32_t)doff & 3u, r1 = r0 + dcnt;
    const uint32_t n_it = flush ? 1u : (r1 + 127u) >> 7;
    const uint4* src = reinterpret_cast<const uint4*>(v.post + (doff - r0)) + lane;
    uint32_t rel = 4u * lane;                                   // first word of this lane's vector
    uint4 nxt = rel < r1 ? __ldg(src) : make_uint4(0u, 0u, 0u, 0u);
    for (uint32_t it = 0; it < n_it; it++, rel += 128u) {
        const uint4 cur = nxt;
        // software pipelining: the next 128 postings are requested before these are filtered (two vectors ahead was measured:
        // the extra registers spill and cost more than the deeper prefetch gains)
        // (L1 policy was measured too: ld.global.nc.L1::no_allocate on this stream and L1::evict_last on the coarse bytes change the
        // kernel time by < 1 % — the coarse-byte loads stall on latency, not on evictions by the stream)
        src += 32;
        nxt = rel + 128u < r1 ? __ldg(src) : make_uint4(0u, 0u, 0u, 0u);
        bool a0 = rel      >= r0 && rel      < r1 && fmaf(didf, bound_of_word(cur.x), R) >= thr.lo;
        bool a1 = rel + 1u >= r0 && rel + 1u < r1 && fmaf(didf, bound_of_word(cur.y), R) >= thr.lo;
        bool a2 = rel + 2u >= r0 && rel + 2u < r1 && fmaf(didf, bound_of_word(cur.z), R) >= thr.lo;
        bool a3 = rel + 3u >= r0 && rel + 3u < r1 && fmaf(didf, bound_of_word(cur.w), R) >= thr.lo;
        bool any = __any_sync(FULL, a0 | a1 | a2 | a3);
        if (any && co.n) {
            float b0 = fmaf(didf, bound_of_word(cur.x), co.base), b1 = fmaf(didf, bound_of_word(cur.y), co.base);
            float b2 = fmaf(didf, bound_of_word(cur.z), co.base), b3 = fmaf(didf, bound_of_word(cur.w), co.base);
            // (requesting the bytes of all terms before the first use — one round trip per iteration instead of one per term — was measured:
            // 2 % slower for OR, 7 % for AND; the extra live registers cost more than the overlap gains)
#pragma unroll
            for (uint32_t j = 0; j < FAST_T - 1; j++) {
                if (j >= co.n) break;
                const uint8_t* tb = v.bm_q8 + co.off[j];
                const uint32_t q0 = a0 ? __ldg(tb + ((cur.x & 0xFFFFu) >> 6)) : 0u, q1 = a1 ? __ldg(tb + ((cur.y & 0xFFFFu) >> 6)) : 0u;
                const uint32_t q2 = a2 ? __ldg(tb + ((cur.z & 0xFFFFu) >> 6)) : 0u, q3 = a3 ? __ldg(tb + ((cur.w & 0xFFFFu) >> 6)) : 0u;
                if (IS_AND) { a0 = a0 && q0; a1 = a1 && q1; a2 = a2 && q2; a3 = a3 && q3; }
                b0 = fmaf(co.cf[j], (float)q0, b0); b1 = fmaf(co.cf[j], (float)q1, b1);
                b2 = fmaf(co.cf[j], (float)q2, b2); b3 = fmaf(co.cf[j], (float)q3, b3);
            }
            a0 = a0 && b0 >= thr.lo; a1 = a1 && b1 >= thr.lo; a2 = a2 && b2 >= thr.lo; a3 = a3 && b3 >= thr.lo;
            any = __any_sync(FULL, a0 | a1 | a2 | a3);
        }
        if (any) {
            const uint32_t lt = (1u << lane) - 1u;
            unsigned m;
            m = __ballot_sync(FULL, a0); if (a0) w.queue[nq_in + __popc(m & lt)] = make_uint2((rel      - r0) | tag, cur.x); nq_in += __popc(m);
            m = __ballot_sync(FULL, a1); if (a1) w.queue[nq_in + __popc(m & lt)] = make_uint2((rel + 1u - r0) | tag, cur.y); nq_in += __popc(m);
            m = __ballot_sync(FULL, a2); if (a2) w.queue[nq_in + __popc(m & lt)] = make_uint2((rel + 2u - r0) | tag, cur.z); nq_in += __popc(m);
            m = __ballot_sync(FULL, a3); if (a3) w.queue[nq_in + __popc(m & lt)] = make_uint2((rel + 3u - r0) | tag, cur.w); nq_in += __popc(m);
            __syncwarp();
        }
        if (nq_in >= 32u || flush) drain_queue<IS_AND, HAS_NOT>(v, w, nq_in, flush, lane, k, ceil, L, thr, dirty, st_probes);
    }
}

// enumerate a whole list 128 postings per iteration: f(doc id, valid) is called 4x per lane per iteration (warp-converged)
template <class F>
__device__ __forceinline__ void for_each_posting(const LexView& v, uint64_t doff, uint32_t dcnt, int lane, F f) {
    const uint32_t r0 = (uint32_t)doff & 3u, r1 = r0 + dcnt;
    const uint4* src = reinterpret_cast<const uint4*>(v.post + (doff - r0)) + lane;
    for (uint32_t rel = 4u * lane; rel - 4u * lane < r1; rel += 128u, src += 32) {
        const uint4 cur = rel < r1 ? __ldg(src) : make_uint4(0u, 0u, 0u, 0u);
        f(cur.x & 0xFFFFu, rel      >= r0 && rel      < r1);
        f(cur.y & 0xFFFFu, rel + 1u >= r0 && rel + 1u < r1);
        f(cur.z & 0xFFFFu, rel + 2u >= r0 && rel + 2u < r1);
        f(cur.w & 0xFFFFu, rel + 3u >= r0 && rel + 3u < r1);
    }
}

// enumerate several lists of one record back to back, 128 postings per iteration, with the NEXT vector (of this or of the
// following list) always in flight: f(list position, doc id, valid) 4x per lane per iteration; list_done(position) after a list's
// last vector.  slot_of(position) names the record slot.
template <class SlotOf, class F, class G>
__device__ __forceinline__ void stream_lists(const LexView& v, const LvRec& rec, uint32_t nlists, int lane, SlotOf slot_of, F f, G list_done) {
    if (nlists == 0) return;
    uint32_t li = 0, r0n = 0, r1n = 0, reln = 0;
    const uint4* srcn = nullptr;
    auto open = [&](uint32_t i) {
        const LvSlot& t = rec.t[slot_of(i)];
        const uint64_t off = slot_off(t);
        r0n = (uint32_t)off & 3u; r1n = r0n + slot_cnt(t); reln = 4u * lane;
        srcn = reinterpret_cast<const uint4*>(v.post + (off - r0n)) + lane;
    };
    open(0);
    // two vectors in flight per lane (1 KB per warp): the fetch position runs two steps ahead of the processing position
    const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
    uint4 q0, q1;                                                       // fetched vectors and what they are (a_*)
    uint32_t a_r0[2], a_r1[2], a_rel[2], a_ci[2]; bool a_end[2], a_has[2];
    auto fetch = [&](int k, uint4& dst) {
        a_has[k] = li < nlists;
        a_r0[k] = r0n; a_r1[k] = r1n; a_rel[k] = reln; a_ci[k] = li;
        dst = (a_has[k] && reln < r1n) ? __ldg(srcn) : zero;
        reln += 128u; srcn += 32;
        a_end[k] = a_has[k] && (reln - 4u * lane >= r1n);               // warp-uniform
        if (a_end[k]) { li++; if (li < nlists) open(li); }
    };
    fetch(0, q0); fetch(1, q1);
    for (;;) {
        const uint4 cur = q0;
        const uint32_t r0 = a_r0[0], r1 = a_r1[0], rel = a_rel[0], ci = a_ci[0];
        const bool end = a_end[0];
        if (!a_has[0]) break;
        q0 = q1; a_r0[0] = a_r0[1]; a_r1[0] = a_r1[1]; a_rel[0] = a_rel[1]; a_ci[0] = a_ci[1]; a_end[0] = a_end[1]; a_has[0] = a_has[1];
        fetch(1, q1);
        f(ci, cur.x & 0xFFFFu, rel      >= r0 && rel      < r1);
        f(ci, cur.y & 0xFFFFu, rel + 1u >= r0 && rel + 1u < r1);
        f(ci, cur.z & 0xFFFFu, rel + 2u >= r0 && rel + 2u < r1);
        f(ci, cur.w & 0xFFFFu, rel + 3u >= r0 && rel + 3u < r1);
        if (end) list_done(ci);
    }
}

// counting kernels: a bitmap of the level's 65536 doc ids per warp in shared memory
constexpr uint32_t UNION_WORDS = 2048;   // 8 KB of words vs 4 B per posting
struct CountSm { LvRec recs[GMAX]; uint32_t bm[2048]; uint32_t it_base; unsigned it_mask; uint32_t pad[2]; };

// ---- exact match count of one AND record (TopkCount / Count) ----
// Every list >= UNION_WORDS postings: popcount of the AND of the bitmap words (intersection_bitmap_2, intersection.rs:33-108).
// Otherwise the shortest list A marks its docs in the warp-private shared-memory bitmap and the second shortest list B is streamed
// against it (4 B per posting, no global probes); hits are checked against the remaining lists.  When B is much longer than A,
// A's postings probe the other lists instead (one 32-byte sector per probe).
__device__ __forceinline__ uint32_t count_intersection(const LexView& v, const LvRec& rec, uint32_t* bm, int lane, uint32_t& st_visited,
                                                       uint32_t& st_probes, uint32_t& st_words) {
    const uint32_t meta = rec.meta, np = meta_npres(meta);
    uint32_t acc = 0;
    if (np == 0) return 0;
    const uint32_t sa = meta_cperm(meta, np - 1u);                       // cperm: count descending -> the shortest list
    const uint32_t cnt_a = slot_cnt(rec.t[sa]);
    if (np == 1) return lane == 0 ? cnt_a : 0u;
    if (cnt_a >= UNION_WORDS) {
        for (uint32_t wi = lane; wi < 1024u; wi += 32u) {
            uint64_t a = ~0ull;
            for (uint32_t c = 0; c < np; c++) a &= __ldg(&v.bm_words[(size_t)rec.t[meta_cperm(meta, c)].bmi * 1024 + wi]);
            acc += (uint32_t)__popcll(a);
        }
        st_words += np * 1024u;                                         // warp-uniform: every list's 1024 words, counted once (lane 0 reports)
        return acc;
    }
    const uint32_t sb = meta_cperm(meta, np - 2u);
    const uint32_t cnt_b = slot_cnt(rec.t[sb]);
    if (cnt_b <= 8u * cnt_a) {
        uint4* b4 = reinterpret_cast<uint4*>(bm);
        for (uint32_t i = lane; i < 512u; i += 32u) b4[i] = make_uint4(0u, 0u, 0u, 0u);
        __syncwarp();
        st_visited += cnt_a + cnt_b;
        stream_lists(v, rec, 2u, lane, [&](uint32_t i) { return i ? sb : sa; },
            [&](uint32_t i, uint32_t d, bool valid) {
                if (i == 0) { if (valid) atomicOr(&bm[d >> 5], 1u << (d & 31u)); return; }
                bool ok = valid && ((bm[d >> 5] >> (d & 31u)) & 1u);
                for (uint32_t c = 0; c + 2u < np; c++) {                 // longer lists, rarely reached
                    if (!ok) continue;
                    const LvSlot& t = rec.t[meta_cperm(meta, c)];
                    st_probes++;
                    ok = present_in(v, slot_cnt(t), slot_off(t), t.bmi, d);
                }
                acc += ok ? 1u : 0u;
            },
            [&](uint32_t) { __syncwarp(); });
        __syncwarp();
        return acc;
    }
    st_visited += cnt_a;
    stream_lists(v, rec, 1u, lane, [&](uint32_t) { return sa; },
        [&](uint32_t, uint32_t d, bool valid) {
            bool ok = valid;
            for (uint32_t c = 0; c + 1u < np; c++) {
                if (!ok) continue;
                const LvSlot& t = rec.t[meta_cperm(meta, c)];
                st_probes++;
                ok = present_in(v, slot_cnt(t), slot_off(t), t.bmi, d);
            }
            acc += ok ? 1u : 0u;
        },
        [&](uint32_t) {});
    return acc;
}

// ---- |union| of one record through a warp-private bitmap of the level's 65536 doc ids in shared memory (8 KB) ----
// Every list is read once, sequentially: lists of >= UNION_WORDS postings as their 8 KB of bitmap words (OR-ed in, fresh bits
// counted by popcount), shorter ones as postings (4 B each) that set their bit with a shared-memory atomicOr — the bit was
// clear before <=> the doc is new to the union.  No probes of other lists, no global random access (union_count, union.rs:807-1164,
// computes the same number from bitmap words; for two lists it is df0 + df1 - |AND|, union.rs:1236-1244).
__device__ __forceinline__ uint32_t count_union(const LexView& v, const LvRec& rec, uint32_t* bm, int lane, uint32_t& st_visited, uint32_t& st_words) {
    const uint32_t meta = rec.meta, np = meta_npres(meta);
    if (np == 0) return 0;
    if (np == 1) return lane == 0 ? slot_cnt(rec.t[meta_cperm(meta, 0)]) : 0u;
    uint4* b4 = reinterpret_cast<uint4*>(bm);
    uint32_t acc = 0, nw = 0;
    for (uint32_t c = 0; c < np; c++) {                                  // cperm: count descending -> the word-wise lists come first
        const LvSlot& t = rec.t[meta_cperm(meta, c)];
        if (slot_cnt(t) < UNION_WORDS || t.bmi == NONE) break;
        const uint4* g = reinterpret_cast<const uint4*>(v.bm_words + (size_t)t.bmi * 1024);
#pragma unroll 1
        for (uint32_t i0 = lane; i0 < 512u; i0 += 128u) {                // four 16-byte loads in flight per lane
            uint4 n[4];
#pragma unroll
            for (uint32_t u = 0; u < 4u; u++) n[u] = __ldg(g + i0 + 32u * u);
#pragma unroll
            for (uint32_t u = 0; u < 4u; u++) {
                if (c) {
                    const uint4 o = b4[i0 + 32u * u];
                    acc -= __popc(o.x) + __popc(o.y) + __popc(o.z) + __popc(o.w);
                    n[u].x |= o.x; n[u].y |= o.y; n[u].z |= o.z; n[u].w |= o.w;
                }
                acc += __popc(n[u].x) + __popc(n[u].y) + __popc(n[u].z) + __popc(n[u].w);
                b4[i0 + 32u * u] = n[u];
            }
        }
        st_words += 1024u; nw++;                                         // warp-uniform: the list's 1024 words (lane 0 reports)
    }
    if (nw == 0) for (uint32_t i = lane; i < 512u; i += 32u) b4[i] = make_uint4(0u, 0u, 0u, 0u);
    __syncwarp();
    for (uint32_t c = nw; c < np; c++) st_visited += slot_cnt(rec.t[meta_cperm(meta, c)]);
    // the order in which postings claim their bits does not matter: |union| = number of bits that were clear when claimed
    stream_lists(v, rec, np - nw, lane, [&](uint32_t i) { return meta_cperm(meta, nw + i); },
        [&](uint32_t, uint32_t d, bool valid) {
            if (valid) {
                const uint32_t bit = 1u << (d & 31u);
                acc += (atomicOr(&bm[d >> 5], bit) & bit) ? 0u : 1u;
            }
        },
        [&](uint32_t) {});
    __syncwarp();
    return acc;
}

// Pull what the scoring of a record touches first into L1: the coarse tables of its dense lists (8 lines each) and the first
// 128 postings of every list (4 lines each).  Two instructions per record; the loads that follow hit L1 instead of paying a DRAM
// round trip each (the average list has only ~3 stream iterations, so first-touch latency is most of a short list's time).
__device__ __forceinline__ void prefetch_record(const LexView& v, const LvRec& rec, int lane) {
#ifdef SSB_NO_PREFETCH
    return;
#endif
    {
        const LvSlot& t = rec.t[lane >> 3];
        if (slot_cnt(t) && t.bmi != NONE) asm volatile("prefetch.global.L1 [%0];" :: "l"(v.bm_q8 + (size_t)t.bmi * 1024u + (uint32_t)(lane & 7) * 128u));
    }
    if (lane < 16) {
        const LvSlot& t = rec.t[lane >> 2];
        const uint32_t cnt = slot_cnt(t), ln = (uint32_t)(lane & 3);
        if (cnt > ln * 32u) asm volatile("prefetch.global.L1 [%0];" :: "l"(v.post + slot_off(t) + ln * 32u));
    }
}

// ---- record path (n <= FAST_T live terms), scoring of one item ----
template <bool IS_AND, bool HAS_NOT>
__device__ __forceinline__ void score_records(const LexView& v, WarpSm& w, uint32_t nrec, uint32_t q, uint32_t k, uint64_t ceil,
                                              const uint64_t* theta, int lane, uint64_t& L, Thr& thr, bool& dirty,
                                              uint32_t& st_visited, uint32_t& st_probes, uint32_t& st_recs, uint32_t& st_skipped) {
    uint32_t nq_in = 0;
    prefetch_record(v, w.recs[0], lane);
#pragma unroll 1
    for (uint32_t ri = 0; ; ri++) {
        if (ri + 1u < nrec) prefetch_record(v, w.recs[ri + 1u], lane);      // its lines arrive while this record is scored
        // one extra pass (flush) after the last record — or after the first record the block-max test prunes — drains the queues
        bool flush = ri >= nrec;
        const LvRec& rec = w.recs[flush ? 0u : ri];
        const uint32_t meta = rec.meta;
        if (ri && !flush) { const uint32_t t2 = (uint32_t)(__ldcg(&theta[q]) >> 32); if (t2 > thr.u) thr.set(t2); }   // other warps' progress
        // block-max: records are sorted by bound, so the first one below θ ends the scoring of this item
        // (only strictly smaller bounds prune: intersection.rs:2227-2233, single.rs:386-394)
        if (!flush && ord_f32(rec.bound) < thr.u) { st_skipped += nrec - ri; flush = true; }
        if (!flush) st_recs++;
        const uint32_t np = (IS_AND || flush) ? 1u : meta_npres(meta);
#pragma unroll 1
        for (uint32_t p = 0; p < np; p++) {
            // OR, MAXSCORE: a list is essential while the in-query-order sum of the not-yet-driven bounds can reach θ (the role
            // of union_docid_2/3's "single pass only if max_list_score > heap.min", union.rs:1259-1301, 1371-1412)
            if (!IS_AND && !flush && ord_f32(rec.S[p]) < thr.u) break;
            const uint32_t drv = IS_AND ? meta_anddrv(meta) : meta_perm(meta, p);
            const uint32_t dcnt = flush ? 0u : slot_cnt(rec.t[drv]);
            st_visited += dcnt;
            stream_driver<IS_AND, HAS_NOT>(v, w, (ri << 17) | (p << 20), flush ? 0ull : slot_off(rec.t[drv]), dcnt, rec.idf[drv],
                                           rec.R[IS_AND ? 0u : p], coarse_of<IS_AND>(v, rec, drv, p), flush, nq_in, lane, k, ceil, L, thr, dirty, st_probes);
        }
        if (flush) break;
    }
}

// ---- generic path: up to SSB_MAX_QUERY_TERMS live terms, lane t holds term t, values broadcast by shuffles ----
// SORTED: the top-k key is (sort key, score, doc) in T (L / thr unused).  θ is not a score there, so none of the score bounds prunes
// (MAXSCORE driver break, score test of the insert); a candidate whose sort key is below T.thr is dropped before its score loads and,
// on the OR path, before its probes (AND, Topk: before its probes as well — nothing is counted).
template <bool FIELD_RUNS, bool SORTED, bool GEO>
__device__ __forceinline__ void process_item_generic(const LexView& v, const QueryPlan* pl, const ItemCtx& c, int lane,
                                                  uint64_t& L, uint32_t& thr, bool& dirty, uint32_t& matches_out,
                                                  uint32_t& st_visited, uint32_t& st_probes, SortTop& T, const SortDev& sd) {
    const uint32_t n = c.n, lv = c.lv;
    uint32_t matches = 0;
    TermRegs tr; tr.cnt = 0; tr.off = 0; tr.bmi = NONE; tr.idf = 0.f; tr.ub = 0.f;
    if ((uint32_t)lane < n) {
        QTerm qt = pl->t[lane];
        uint32_t e;
        if (find_entry(v, qt, lv, e)) {
            tr.cnt = __ldg(&v.e_count[e]); tr.off = __ldg(&v.e_off[e]); tr.bmi = __ldg(&v.e_bitmap[e]);
            tr.ub = __fmul_rn(qt.idf, __ldg(&v.e_maxcomp[e]));
        }
        tr.idf = qt.idf;
    }
    if (c.is_and) {
        uint32_t cc = (uint32_t)lane < n ? tr.cnt : 0xFFFFFFFFu;
        uint32_t key = cc; int drv = lane;
        for (int s = 16; s; s >>= 1) {
            uint32_t ok = __shfl_xor_sync(FULL, key, s); int od = __shfl_xor_sync(FULL, drv, s);
            if (ok < key || (ok == key && od < drv)) { key = ok; drv = od; }
        }
        const uint32_t dcnt = __shfl_sync(FULL, tr.cnt, drv);
        const uint64_t doff = shfl64(tr.off, drv);
        st_visited += dcnt;
        for (uint32_t base = 0; base < dcnt; base += 32) {
            const uint32_t p = base + lane;
            const bool active = p < dcnt;
            const uint32_t d = active ? (__ldg(&v.post[doff + p]) & 0xFFFFu) : 0u;
            bool ok = active; float score = 0.f;
            uint64_t hi = 0; bool keep = true;
            if constexpr (SORTED) {
                if (active && c.scoring) hi = doc_sort_hi<GEO>(v, sd, c.docbase | d, c.q);
                keep = c.scoring && !(hi < T.thr);
                ok = active && (keep || c.need_count);
            }
            for (uint32_t t = 0; t < n; t++) {          // query order
                const uint32_t tc = __shfl_sync(FULL, tr.cnt, t); const uint64_t to = shfl64(tr.off, t);
                const uint32_t tb = __shfl_sync(FULL, tr.bmi, t); const float ti = __shfl_sync(FULL, tr.idf, t);
                uint32_t rank = p; bool found = true;
                if ((int)t != drv) { found = ok && probe(v, tc, to, tb, d, rank); st_probes += ok ? 1 : 0; }
                ok = ok && found;
                if (ok && c.scoring && (!SORTED || keep)) score = acc_term(v, score, ti, to + rank);
            }
            if (c.n_filt) {
                // a filtered query is counted here doc by doc: filter, delete set and NOT lists at once (the correction kernels skip it)
                ok = ok && !filters_reject<FIELD_RUNS, GEO>(v, pl, c.filt_first, c.n_facet_filt, c.field_mask, c.n, c.lv, d, c.docbase | d) && !is_deleted(v, c.docbase | d) && !(c.n_not && in_not_lists(v, pl, c.n_not, c.lv, d));
                matches += __popc(__ballot_sync(FULL, ok));
                if constexpr (SORTED) { if (c.scoring) insert_sorted(T, ok && keep, hi, score, c.docbase | d, sd.score_asc, c.k, lane, dirty, c.ceil, c.ceil_lo); }
                else
                if (c.scoring) insert_candidates(L, thr, ok && ord_f32(score) >= thr, score, c.docbase | d, c.k, lane, dirty, c.ceil);
                continue;
            }
            matches += __popc(__ballot_sync(FULL, ok));
            if constexpr (SORTED) {
                if (c.scoring) insert_sorted(T, ok && keep && !is_deleted(v, c.docbase | d) && !(c.n_not && in_not_lists(v, pl, c.n_not, c.lv, d)), hi, score, c.docbase | d,
                                             sd.score_asc, c.k, lane, dirty, c.ceil, c.ceil_lo);
            } else
            if (c.scoring) insert_candidates(L, thr, ok && ord_f32(score) >= thr && !is_deleted(v, c.docbase | d) && !(c.n_not && in_not_lists(v, pl, c.n_not, c.lv, d)), score, c.docbase | d, c.k, lane, dirty, c.ceil);
        }
        if (lane == 0) matches_out += matches;
        return;
    }
    if (c.scoring) {
        uint32_t rk = 0;
        for (uint32_t t = 0; t < n; t++) {
            float ou = __shfl_sync(FULL, tr.ub, t); uint32_t oc = __shfl_sync(FULL, tr.cnt, t);
            bool mine = (uint32_t)lane < n;
            bool before = (oc > 0 && tr.cnt == 0) || ((oc > 0) == (tr.cnt > 0) && (ou > tr.ub || (ou == tr.ub && t < (uint32_t)lane)));
            if (mine && before && t != (uint32_t)lane) rk++;
        }
        if ((uint32_t)lane >= n) rk = 0xFFFFu;
        for (uint32_t p = 0; p < n; p++) {
            const int drv = __ffs(__ballot_sync(FULL, rk == p)) - 1;
            const uint32_t dcnt = __shfl_sync(FULL, tr.cnt, drv);
            if (dcnt == 0) break;
            float S = 0.f;
            for (uint32_t t = 0; t < n; t++) {
                float ou = __shfl_sync(FULL, tr.ub, t); uint32_t orr = __shfl_sync(FULL, rk, t);
                if (orr >= p) S = __fadd_rn(S, ou);
            }
            if (!SORTED && ord_f32(S) < thr) break;
            const uint64_t doff = shfl64(tr.off, drv);
            const float didf = __shfl_sync(FULL, tr.idf, drv);
            st_visited += dcnt;
            for (uint32_t base = 0; base < dcnt; base += 32) {
                const uint32_t pp = base + lane;
                const bool active = pp < dcnt;
                const uint32_t d = active ? (__ldg(&v.post[doff + pp]) & 0xFFFFu) : 0u;
                bool dup = false; float score = 0.f;
                uint64_t hi = 0; bool live = active;
                if constexpr (SORTED) {
                    if (active) hi = doc_sort_hi<GEO>(v, sd, c.docbase | d, c.q);
                    live = active && !(hi < T.thr);
                }
                for (uint32_t t = 0; t < n; t++) {      // query order
                    const uint32_t tc = __shfl_sync(FULL, tr.cnt, t); const uint64_t to = shfl64(tr.off, t);
                    const uint32_t tb = __shfl_sync(FULL, tr.bmi, t); const float ti = __shfl_sync(FULL, tr.idf, t);
                    const uint32_t trk = __shfl_sync(FULL, rk, t);
                    if ((int)t == drv) { if (live) score = acc_term(v, score, didf, doff + pp); continue; }
                    if (tc == 0 || !live || dup) continue;
                    uint32_t rank; st_probes++;
                    if (probe(v, tc, to, tb, d, rank)) {
                        if (trk < p) dup = true;
                        else score = acc_term(v, score, ti, to + rank);
                    }
                }
                if constexpr (SORTED) {
                    insert_sorted(T, live && !dup && !is_deleted(v, c.docbase | d) && !(c.n_not && in_not_lists(v, pl, c.n_not, c.lv, d))
                                     && !(c.n_filt && filters_reject<FIELD_RUNS, GEO>(v, pl, c.filt_first, c.n_facet_filt, c.field_mask, c.n, c.lv, d, c.docbase | d)),
                                  hi, score, c.docbase | d, sd.score_asc, c.k, lane, dirty, c.ceil, c.ceil_lo);
                } else
                insert_candidates(L, thr, active && !dup && ord_f32(score) >= thr && !is_deleted(v, c.docbase | d) && !(c.n_not && in_not_lists(v, pl, c.n_not, c.lv, d))
                                              && !(c.n_filt && filters_reject<FIELD_RUNS, GEO>(v, pl, c.filt_first, c.n_facet_filt, c.field_mask, c.n, c.lv, d, c.docbase | d)), score, c.docbase | d, c.k, lane, dirty, c.ceil);
            }
        }
    }
    if (c.need_count) {
        uint32_t crk = 0;
        for (uint32_t t = 0; t < n; t++) {
            uint32_t oc = __shfl_sync(FULL, tr.cnt, t);
            if ((uint32_t)lane < n && t != (uint32_t)lane && (oc > tr.cnt || (oc == tr.cnt && t < (uint32_t)lane))) crk++;
        }
        if ((uint32_t)lane >= n) crk = 0xFFFFu;
        for (uint32_t p = 0; p < n; p++) {
            const int drv = __ffs(__ballot_sync(FULL, crk == p)) - 1;
            const uint32_t dcnt = __shfl_sync(FULL, tr.cnt, drv);
            if (dcnt == 0) break;
            if (p == 0 && !c.n_filt) { matches += dcnt; continue; }
            const uint64_t doff = shfl64(tr.off, drv);
            st_visited += dcnt;
            for (uint32_t base = 0; base < dcnt; base += 32) {
                const uint32_t pp = base + lane;
                const bool active = pp < dcnt;
                const uint32_t d = active ? (__ldg(&v.post[doff + pp]) & 0xFFFFu) : 0u;
                bool dup = false;
                for (uint32_t t = 0; t < n; t++) {
                    const uint32_t tc = __shfl_sync(FULL, tr.cnt, t); const uint64_t to = shfl64(tr.off, t);
                    const uint32_t tb = __shfl_sync(FULL, tr.bmi, t); const uint32_t trk = __shfl_sync(FULL, crk, t);
                    if (trk >= p || tc == 0 || !active || dup) continue;
                    uint32_t rank; st_probes++;
                    if (probe(v, tc, to, tb, d, rank)) dup = true;
                }
                bool cnt_ok = active && !dup;
                if (c.n_filt && cnt_ok)      // filtered query: every match is tested here (filter, delete set, NOT lists; the correction kernels skip it)
                    cnt_ok = !filters_reject<FIELD_RUNS, GEO>(v, pl, c.filt_first, c.n_facet_filt, c.field_mask, c.n, c.lv, d, c.docbase | d) && !is_deleted(v, c.docbase | d) && !(c.n_not && in_not_lists(v, pl, c.n_not, c.lv, d));
                matches += __popc(__ballot_sync(FULL, cnt_ok));
            }
        }
    }
    if (lane == 0) matches_out += matches;
}

#ifndef SSB_LEX_MINB
#define SSB_LEX_MINB 3
#endif

// claim the next work item: wave order — item i -> (j = i / nq, q = i % nq) = the j-th item of query q, so every query's best
// levels are scored first and its θ is published before most of its other items start
// Work distribution: item index i -> (j = i / nq, q = i % nq), i.e. the first items of all queries, then the second ones, ...
// A warp takes ITEM_CHUNK consecutive indices per atomic; its lanes test them in parallel (most indices of the later waves
// name items a query does not have) and the warp then works through the valid ones.
constexpr uint32_t ITEM_CHUNK = 8;
template <bool FAST, class SM>
__device__ __forceinline__ bool next_item(SM& it, uint32_t* counter, uint64_t total, uint32_t nq, const QueryPlan* __restrict__ plans,
                                          int lane, uint32_t& j, uint32_t& q) {
    unsigned mask = it.it_mask; uint32_t base = it.it_base;      // warp-private shared memory: keeps two registers out of the hot loops
    __syncwarp();
    while (!mask) {
        uint32_t b = 0;
        if (lane == 0) b = atomicAdd(counter, ITEM_CHUNK);
        b = __shfl_sync(FULL, b, 0);
        if ((uint64_t)b >= total) return false;
        const uint64_t i = (uint64_t)b + (uint32_t)lane;
        bool ok = (uint32_t)lane < ITEM_CHUNK && i < total;
        if (ok) {
            const uint32_t jj = (uint32_t)(i / nq), qq = (uint32_t)(i - (uint64_t)jj * nq);
            const QueryPlan* pl = &plans[qq];
            ok = jj < __ldg(&pl->n_items) && ((__ldg(&pl->fast) != 0u) == FAST);
        }
        mask = __ballot_sync(FULL, ok); base = b;
    }
    const uint32_t i = base + (uint32_t)(__ffs(mask) - 1);
    if (lane == 0) { it.it_mask = mask & (mask - 1); it.it_base = base; }
    __syncwarp();
    j = i / nq; q = i - j * nq;
    return true;
}
// stage the item's records in shared memory: 128 B per record, one coalesced word per lane
template <class SM>
__device__ __forceinline__ uint32_t stage_item(SM& w, const LvRec* __restrict__ recs, const uint16_t* __restrict__ item_start,
                                               uint32_t nlv, uint32_t q, uint32_t j, int lane) {
    const uint16_t* is = item_start + (size_t)q * (nlv + 1);
    const uint32_t r0 = __ldg(&is[j]), r1 = __ldg(&is[j + 1]);
    const uint32_t nrec = r1 - r0;
    __syncwarp();
    const uint32_t* src = reinterpret_cast<const uint32_t*>(recs + (size_t)q * nlv + r0);
    uint32_t* dst = reinterpret_cast<uint32_t*>(w.recs);
    for (uint32_t r = 0; r < nrec; r++) dst[r * 32 + lane] = __ldg(src + r * 32 + lane);
    __syncwarp();
    return nrec;
}
// merge the warp's list into the query's global list under the per-query lock, raise θ
__device__ __forceinline__ void publish(uint64_t L, uint32_t q, uint32_t k, int lane, uint64_t* theta, int* lock, uint64_t* glist) {
    if (lane == 0) { while (atomicCAS(&lock[q], 0, 1) != 0) __nanosleep(40); }
    __syncwarp();
    __threadfence();
    uint64_t G = __ldcg(&glist[(size_t)q * LIST + lane]);
    uint64_t M = wl_merge(L, G, lane);
    __stcg(&glist[(size_t)q * LIST + lane], M);
    uint64_t nth = shfl64(M, (int)k - 1);
    __threadfence();
    __syncwarp();
    if (lane == 0) {
        if (nth > __ldcg(&theta[q])) __stcg(&theta[q], nth);
        __threadfence();
        atomicExch(&lock[q], 0);
    }
}

// ---- scoring, queries with <= 4 live terms (ResultType Topk / TopkCount) ----
template <bool IS_AND, bool HAS_NOT>
__global__ void __launch_bounds__(256, SSB_LEX_MINB) lex_score(LexView v, const QueryPlan* __restrict__ plans, const LvRec* __restrict__ recs,
                                                 const uint16_t* __restrict__ item_start, uint32_t nq, uint32_t k, uint32_t* ctr, uint64_t* theta,
                                                 int* lock, uint64_t* glist, LexStats* stats, const uint64_t* __restrict__ ceil_keys) {
    __shared__ __align__(16) WarpSm wsm[8];
    if (v.fast_t == 0) return;                           // several indexed fields: every query takes the generic path
    WarpSm& w = wsm[(threadIdx.x >> 5) & 7];
    const int lane = threadIdx.x & 31;
    const uint64_t total = (uint64_t)(*(volatile uint32_t*)&ctr[1]) * nq;
    uint32_t st_visited = 0, st_probes = 0, st_done = 0, st_skipped = 0, st_recs = 0;   // per warp: far below 2^32 each
    uint32_t j, q;
    if (lane == 0) { w.it_mask = 0; w.it_base = 0; }
    __syncwarp();
    while (next_item<true>(w, &ctr[0], total, nq, plans, lane, j, q)) {
        const QueryPlan* pl = &plans[q];
        const uint64_t ceil = ceil_keys ? __ldg(&ceil_keys[q]) : ~0ull;
        if (ceil == 0) continue;                         // this query's result list is already exhausted
        const uint32_t nrec = stage_item(w, recs, item_start, v.n_levels, q, j, lane);
        if (lane == 0) { w.pl = pl; w.n_not = __ldg(&pl->n_not); w.nq2 = 0; w.n_filt = __ldg(&pl->n_filt); w.filt_first = __ldg(&pl->filt_first); }
        __syncwarp();
        Thr thr; thr.set((uint32_t)(__ldcg(&theta[q]) >> 32));
        if (ord_f32(w.recs[0].bound) < thr.u) { st_skipped += nrec; continue; }   // whole item below θ
        uint64_t L = 0; bool dirty = false;
        st_done++;
        score_records<IS_AND, HAS_NOT>(v, w, nrec, q, k, ceil, theta, lane, L, thr, dirty, st_visited, st_probes, st_recs, st_skipped);
        if (dirty) publish(L, q, k, lane, theta, lock, glist);
    }
    // per-lane counters (probes) are summed over the warp; warp-uniform ones are taken from lane 0
    unsigned long long acc_probes = st_probes;
    for (int s = 16; s; s >>= 1) acc_probes += __shfl_xor_sync(FULL, acc_probes, s);
    if (lane == 0) {
        atomicAdd((unsigned long long*)&stats->postings_visited, (unsigned long long)st_visited);
        atomicAdd((unsigned long long*)&stats->probes, acc_probes);
        atomicAdd((unsigned long long*)&stats->items_processed, (unsigned long long)st_done);
        atomicAdd((unsigned long long*)&stats->items_skipped, (unsigned long long)st_skipped);
        atomicAdd((unsigned long long*)&stats->recs_processed, (unsigned long long)st_recs);
    }
}

// ---- exact match counts, queries with <= 4 live terms (ResultType Count / TopkCount): independent of θ, own kernel ----
__global__ void __launch_bounds__(128, 6) lex_count(LexView v, const QueryPlan* __restrict__ plans, const LvRec* __restrict__ recs,
                                                const uint16_t* __restrict__ item_start, uint32_t nq, uint32_t query_type, uint32_t* ctr,
                                                uint64_t* count, LexStats* stats) {
    __shared__ __align__(16) CountSm csm[4];
    if (v.fast_t == 0) return;                           // several indexed fields: the generic path counts as well
    CountSm& w = csm[(threadIdx.x >> 5) & 3];
    const int lane = threadIdx.x & 31;
    const uint64_t total = (uint64_t)(*(volatile uint32_t*)&ctr[1]) * nq;
    const bool is_and = query_type == SSB_QUERY_INTERSECTION;
    uint64_t acc_visited = 0, acc_probes = 0, acc_words = 0; uint32_t st_recs = 0;
    uint32_t j, q;
    if (lane == 0) { w.it_mask = 0; w.it_base = 0; }
    __syncwarp();
    while (next_item<true>(w, &ctr[2], total, nq, plans, lane, j, q)) {
        const uint32_t nrec = stage_item(w, recs, item_start, v.n_levels, q, j, lane);
        uint32_t matches = 0, st_visited = 0, st_probes = 0, st_words = 0;
        for (uint32_t ri = 0; ri < nrec; ri++)
            matches += is_and ? count_intersection(v, w.recs[ri], w.bm, lane, st_visited, st_probes, st_words)
                              : count_union(v, w.recs[ri], w.bm, lane, st_visited, st_words);
        st_recs += nrec;
        for (int s = 16; s; s >>= 1) matches += __shfl_xor_sync(FULL, matches, s);
        if (lane == 0 && matches) atomicAdd((unsigned long long*)&count[q], (unsigned long long)matches);
        acc_visited += st_visited; acc_probes += st_probes; acc_words += st_words;
    }
    for (int s = 16; s; s >>= 1) acc_probes += __shfl_xor_sync(FULL, acc_probes, s);
    if (lane == 0) {
        atomicAdd((unsigned long long*)&stats->postings_visited, (unsigned long long)acc_visited);
        atomicAdd((unsigned long long*)&stats->probes, (unsigned long long)acc_probes);
        atomicAdd((unsigned long long*)&stats->dense_words, (unsigned long long)acc_words);
        atomicAdd((unsigned long long*)&stats->recs_processed, (unsigned long long)st_recs);
    }
}

// ---- queries with 5..16 live terms: one level per item, per-term state in lanes (scoring and counting) ----
// FIELD_RUNS: phrase batch on an index with several fields (the phrase check walks per-field position runs)
// SORTED: a sorted batch (every query is here; theta / glist / ceil_keys hold 128-bit keys).  The score bound of a level means nothing
// there; under Topk a level is skipped when its sort-key bound is below θ.hi (strictly: ties in hi go through the exact insert).
// GEO: the batch has a POINT filter or sorts by a POINT criterion (geo_rejects_impl / point_sort_key in the call graph)
template <bool FIELD_RUNS, bool SORTED, bool GEO = false>
__global__ void __launch_bounds__(256) lex_generic(LexView v, const QueryPlan* __restrict__ plans, const LvRec* __restrict__ recs,
                                                  const uint16_t* __restrict__ item_start, uint32_t nq, uint32_t query_type, uint32_t result_type,
                                                  uint32_t k, uint32_t* ctr, uint64_t* theta, int* lock, uint64_t* count, uint64_t* glist,
                                                  LexStats* stats, const uint64_t* __restrict__ ceil_keys, SortDev sort) {
    if (*(volatile uint32_t*)&ctr[4] == 0) return;       // no query of this batch has more than FAST_T live terms
    __shared__ __align__(16) WarpSm wsm[8];
    WarpSm& w = wsm[(threadIdx.x >> 5) & 7];
    const int lane = threadIdx.x & 31;
    const uint64_t total = (uint64_t)(*(volatile uint32_t*)&ctr[1]) * nq;
    const bool want_topk = result_type != SSB_RESULT_COUNT && k > 0;
    const bool need_count = result_type != SSB_RESULT_TOPK;
    uint32_t st_visited = 0, st_probes = 0, st_done = 0, st_skipped = 0;
    uint32_t j, q;
    if (lane == 0) { w.it_mask = 0; w.it_base = 0; }
    __syncwarp();
    while (next_item<false>(w, &ctr[3], total, nq, plans, lane, j, q)) {
        const QueryPlan* pl = &plans[q];
        const uint32_t n_live = __ldg(&pl->n_live);
        if constexpr (SORTED) {
            const uint64_t ch = ceil_keys ? __ldg(&ceil_keys[2 * q]) : ~0ull, cl = ceil_keys ? __ldg(&ceil_keys[2 * q + 1]) : ~0ull;
            if (ch == 0 && cl == 0) continue;
            const uint32_t nrec = stage_item(w, recs, item_start, v.n_levels, q, j, lane);
            SortTop T{0, 0, 0};
            uint64_t L = 0; uint32_t thr = 0; bool dirty = false; uint32_t matches = 0;
            for (uint32_t ri = 0; ri < nrec; ri++) {
                const uint64_t th = __ldcg(&theta[2 * q]);
                if (th > T.thr) T.thr = th;
                ItemCtx c;
                c.ceil = ch; c.ceil_lo = cl; c.q = q; c.n = n_live; c.k = k; c.lv = w.recs[ri].lv; c.bound_ord = 0; c.n_not = __ldg(&pl->n_not);
                c.n_facet_filt = __ldg(&pl->n_filt); c.filt_first = __ldg(&pl->filt_first); c.field_mask = __ldg(&pl->field_mask);
                c.n_filt = c.n_facet_filt + (c.field_mask ? 1u : 0u) + (__ldg(&pl->n_phr) ? 1u : 0u);
                c.scoring = want_topk && !(rec_sort_bound(w.recs[ri]) < T.thr);
                c.need_count = need_count; c.is_and = query_type == SSB_QUERY_INTERSECTION; c.docbase = w.recs[ri].docbase;
                if (!c.scoring && !need_count) { st_skipped++; continue; }
                st_done++;
                process_item_generic<FIELD_RUNS, true, GEO>(v, pl, c, lane, L, thr, dirty, matches, st_visited, st_probes, T, sort);
            }
            if (dirty) publish_sorted(T, q, k, lane, theta, lock, glist);
            if (need_count && lane == 0 && matches) atomicAdd((unsigned long long*)&count[q], (unsigned long long)matches);
            continue;
        }
        const uint64_t ceil = ceil_keys ? __ldg(&ceil_keys[q]) : ~0ull;
        if (ceil == 0) continue;
        const uint32_t nrec = stage_item(w, recs, item_start, v.n_levels, q, j, lane);
        uint32_t thr = (uint32_t)(__ldcg(&theta[q]) >> 32);
        uint64_t L = 0; bool dirty = false; uint32_t matches = 0;
        SortTop T;
        for (uint32_t ri = 0; ri < nrec; ri++) {
            ItemCtx c;
            c.ceil = ceil; c.q = q; c.n = n_live; c.k = k; c.lv = w.recs[ri].lv; c.bound_ord = ord_f32(w.recs[ri].bound); c.n_not = __ldg(&pl->n_not);
            c.n_facet_filt = __ldg(&pl->n_filt); c.filt_first = __ldg(&pl->filt_first); c.field_mask = __ldg(&pl->field_mask);
            c.n_filt = c.n_facet_filt + (c.field_mask ? 1u : 0u) + (__ldg(&pl->n_phr) ? 1u : 0u);
            c.scoring = want_topk && c.bound_ord >= thr;
            c.need_count = need_count; c.is_and = query_type == SSB_QUERY_INTERSECTION; c.docbase = w.recs[ri].docbase;
            if (!c.scoring && !need_count) { st_skipped++; continue; }
            st_done++;
            process_item_generic<FIELD_RUNS, false, GEO>(v, pl, c, lane, L, thr, dirty, matches, st_visited, st_probes, T, sort);
        }
        if (dirty) publish(L, q, k, lane, theta, lock, glist);
        if (need_count && lane == 0 && matches) atomicAdd((unsigned long long*)&count[q], (unsigned long long)matches);
    }
    unsigned long long pr = st_probes;
    for (int s = 16; s; s >>= 1) pr += __shfl_xor_sync(FULL, pr, s);
    if (lane == 0) {
        atomicAdd((unsigned long long*)&stats->postings_visited, (unsigned long long)st_visited);
        atomicAdd((unsigned long long*)&stats->probes, pr);
        atomicAdd((unsigned long long*)&stats->items_processed, (unsigned long long)st_done);
        atomicAdd((unsigned long long*)&stats->items_skipped, (unsigned long long)st_skipped);
    }
}

// does doc d of local level lv match the query's n positive terms (AND: all of them, OR: any)?
__device__ __forceinline__ bool matches_terms(const LexView& v, const QueryPlan* pl, uint32_t n, bool is_and, uint32_t lv, uint32_t d) {
    bool any = false, all = true;
    for (uint32_t t = 0; t < n; t++) {
        const bool pres = term_has(v, pl->t[t], lv, d);
        any = any || pres; all = all && pres;
    }
    return is_and ? all : any;
}

// ---- exact counts with NOT lists: the count kernels count every match of the positive terms; the matches that sit in a NOT list are
// subtracted here.  One warp per (query, local level); a NOT list's postings are enumerated (each doc once: docs already seen in an
// earlier NOT list are skipped), deleted docs are left to lex_del_count. ----
__global__ void __launch_bounds__(256) lex_not_count(LexView v, const QueryPlan* __restrict__ plans, uint32_t nq, uint32_t query_type, const uint32_t* ctr,
                                                    uint64_t* count) {
    if (*(volatile const uint32_t*)&ctr[5] == 0) return;
    const int lane = threadIdx.x & 31;
    const uint64_t wid = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const uint64_t n_warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    const bool is_and = query_type == SSB_QUERY_INTERSECTION;
    for (uint64_t it = wid; it < (uint64_t)nq * v.n_levels; it += n_warps) {
        const uint32_t q = (uint32_t)(it / v.n_levels), lv = (uint32_t)(it % v.n_levels);
        const QueryPlan* pl = &plans[q];
        const uint32_t n_not = pl->n_not, n = pl->n_live;
        if (!n_not || !n || pl->n_filt || pl->field_mask || pl->n_phr) continue;                      // filtered queries were counted doc by doc in lex_generic
        const uint32_t docbase = __ldg(&v.level_ids[lv]) << 16;
        uint32_t sub = 0;
        for (uint32_t i = 0; i < n_not; i++) {
            uint32_t e;
            if (!find_entry(v, pl->tn[i], lv, e)) continue;
            for_each_posting(v, __ldg(&v.e_off[e]), __ldg(&v.e_count[e]), lane, [&](uint32_t d, bool valid) {
                if (!valid) return;
                if (i && in_not_lists(v, pl, i, lv, d)) return;          // counted with an earlier NOT list
                if (is_deleted(v, docbase | d)) return;
                sub += matches_terms(v, pl, n, is_and, lv, d) ? 1u : 0u;
            });
        }
        for (int s = 16; s; s >>= 1) sub += __shfl_xor_sync(FULL, sub, s);
        if (lane == 0 && sub) atomicAdd((unsigned long long*)&count[q], 0ull - (unsigned long long)sub);
    }
}

// ---- exact counts with a delete set: the count kernels count every match; the deleted docs that match are subtracted here,
// one thread per (query, deleted doc) — the reference does the same walk over delete_hashset (union_count, union.rs:975-1000) ----
__global__ void lex_del_count(LexView v, const QueryPlan* __restrict__ plans, uint32_t nq, uint32_t query_type, uint64_t* count) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (uint64_t)nq * v.n_del) return;
    const uint32_t q = (uint32_t)(i / v.n_del), doc = __ldg(&v.del_docs[i % v.n_del]);
    const QueryPlan* pl = &plans[q];
    const uint32_t n = pl->n_live;
    if (n == 0 || pl->n_filt || pl->field_mask || pl->n_phr) return;                               // (filtered queries were counted doc by doc in lex_generic)
    uint32_t lo = 0, hi = v.n_levels;                               // local level index of the doc's level id
    const uint32_t lid = doc >> 16, d = doc & 0xFFFFu;
    while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (__ldg(&v.level_ids[m]) < lid) lo = m + 1; else hi = m; }
    if (lo >= v.n_levels || __ldg(&v.level_ids[lo]) != lid) return;  // level not on this shard
    if (matches_terms(v, pl, n, query_type == SSB_QUERY_INTERSECTION, lo, d)) atomicAdd((unsigned long long*)&count[q], ~0ull);   // -1
}

__global__ void copy_out(const uint64_t* __restrict__ glist, const uint64_t* __restrict__ count, uint32_t nq, uint32_t k,
                         uint64_t* keys_out, uint64_t* count_out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nq * LIST) { uint32_t j = i & 31; keys_out[i] = j < k ? glist[i] : 0; }
    if (count_out && i < nq) count_out[i] = count[i];
}

// ================================================================= facet counts (ssb_search_lexical_facets; facet_count, add_result.rs:487-640)
// A pass of its own after lex_plan<false> (Count): every scoring and counting kernel above keeps its code.  One warp per (query, record):
// the level's matches as a bitmap of its 65536 doc ids in shared memory (as CountSm), then the set bits in doc order through the same
// predicates the count path runs, then one bin per doc and request.  Range bins go to a warp-private shared histogram flushed with one
// global atomic per nonzero bin at the end of the record; value bins (ids) go to the query's dense histogram in global memory.
constexpr uint32_t FACET_WARPS = 4;
struct FacetCall {
    const FacetReqDev* req; uint32_t n_req;
    const uint64_t* starts; uint32_t n_starts;      // RANGES / POINT starts in key space
    const double* bases; uint32_t n_point;          // [n_queries][n_point][2]
    uint32_t* hist; uint32_t hist_words, range_words;   // [chunk][hist_words]: the range bins first, then the value bins
    uint64_t* stats;                                // {postings read, dense words read, counted docs, StringSet CSR bytes read}
};
struct FacetWarpSm { uint32_t bm[2048]; uint16_t list[1024]; };

// SETS: the call has a VALUES request on a StringSet facet (search.rs:3615-3640: each doc counts under each member occurrence of its
// combination); csr [2 * n_req]: per request the facet's set offsets and member ids as addresses (0: not a StringSet facet).  Its own
// instantiation, and the table an argument of its own, so that the other instantiations keep their code and registers.
template <bool FIELD_RUNS, bool GEO, bool SETS>
__global__ void __launch_bounds__(FACET_WARPS * 32) lex_facets(LexView v, const QueryPlan* __restrict__ plans, const LvRec* __restrict__ recs,
                                                                uint32_t q0, uint32_t nqc, uint32_t query_type, FacetCall fc,
                                                                const uint64_t* __restrict__ csr) {
    extern __shared__ __align__(16) uint8_t fsm_raw[];
    uint64_t* sstart = reinterpret_cast<uint64_t*>(fsm_raw);                                   // [n_starts]
    FacetReqDev* sreq = reinterpret_cast<FacetReqDev*>(sstart + fc.n_starts);                  // [n_req]
    FacetWarpSm* wsm = reinterpret_cast<FacetWarpSm*>(sreq + fc.n_req);                        // [FACET_WARPS]
    uint32_t* rhist_all = reinterpret_cast<uint32_t*>(wsm + FACET_WARPS);                      // [FACET_WARPS][range_words]
    for (uint32_t i = threadIdx.x; i < fc.n_starts; i += blockDim.x) sstart[i] = fc.starts[i];
    for (uint32_t i = threadIdx.x; i < fc.n_req; i += blockDim.x) sreq[i] = fc.req[i];
    for (uint32_t i = threadIdx.x; i < FACET_WARPS * fc.range_words; i += blockDim.x) rhist_all[i] = 0;
    __syncthreads();
    const uint32_t wi = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    uint32_t* bm = wsm[wi].bm;
    uint64_t* bm64 = reinterpret_cast<uint64_t*>(bm);
    uint16_t* list = wsm[wi].list;
    uint32_t* rhist = rhist_all + (size_t)wi * fc.range_words;
    const uint32_t nlv = v.n_levels;
    const bool is_and = query_type == SSB_QUERY_INTERSECTION;
    uint64_t st_post = 0, st_words = 0, st_docs = 0, st_csr = 0;
    const uint64_t n_warps = (uint64_t)gridDim.x * FACET_WARPS;
    for (uint64_t it = (uint64_t)blockIdx.x * FACET_WARPS + wi; it < (uint64_t)nqc * nlv; it += n_warps) {
        const uint32_t ql = (uint32_t)(it / nlv), j = (uint32_t)(it % nlv), q = q0 + ql;
        const QueryPlan* pl = &plans[q];
        if (j >= __ldg(&pl->n_recs)) continue;
        const uint32_t lv = __ldg(&recs[(size_t)q * nlv + j].lv);
        const uint32_t docbase = __ldg(&recs[(size_t)q * nlv + j].docbase);
        const uint32_t n = __ldg(&pl->n_live);
        // lane t: the list of query term t at this level (a record exists: OR some list, AND every list is there)
        uint32_t cnt = 0, bmi = NONE; uint64_t off = 0;
        if ((uint32_t)lane < n) {
            uint32_t e;
            if (find_entry(v, pl->t[lane], lv, e)) { cnt = __ldg(&v.e_count[e]); off = __ldg(&v.e_off[e]); bmi = __ldg(&v.e_bitmap[e]); }
        }
        // ---- 1. the match bitmap ----
        if (!is_and) {
            for (uint32_t i = lane; i < 2048u; i += 32u) bm[i] = 0u;
            __syncwarp();
            for (uint32_t t = 0; t < n; t++) {
                const uint32_t tc = __shfl_sync(FULL, cnt, t), tb = __shfl_sync(FULL, bmi, t); const uint64_t to = shfl64(off, t);
                if (tc == 0) continue;
                if (tb != NONE) {
                    for (uint32_t i = lane; i < 1024u; i += 32u) bm64[i] |= __ldg(&v.bm_words[(size_t)tb * 1024 + i]);
                    st_words += 1024u;                                         // the list's 1024 words, once per warp (lane 0 reports)
                } else {
                    for_each_posting(v, to, tc, lane, [&](uint32_t d, bool valid) { if (valid) atomicOr(&bm[d >> 5], 1u << (d & 31u)); });
                    st_post += tc;
                }
                __syncwarp();
            }
        } else {
            // the shortest list drives; all lists dense (the shortest has a bitmap): word AND, else its postings probe the others
            uint32_t key = (uint32_t)lane < n ? cnt : 0xFFFFFFFFu; int drv = lane;
            for (int s = 16; s; s >>= 1) {
                const uint32_t ok = __shfl_xor_sync(FULL, key, s); const int od = __shfl_xor_sync(FULL, drv, s);
                if (ok < key || (ok == key && od < drv)) { key = ok; drv = od; }
            }
            const uint32_t dcnt = __shfl_sync(FULL, cnt, drv), dbmi = __shfl_sync(FULL, bmi, drv); const uint64_t doff = shfl64(off, drv);
            if (dcnt == 0) continue;
            if (dbmi != NONE) {
                for (uint32_t i = lane; i < 1024u; i += 32u) {
                    uint64_t a = ~0ull;
                    for (uint32_t t = 0; t < n; t++) a &= __ldg(&v.bm_words[(size_t)__shfl_sync(FULL, bmi, t) * 1024 + i]);
                    bm64[i] = a;
                }
                st_words += 1024u * n;
            } else {
                for (uint32_t i = lane; i < 2048u; i += 32u) bm[i] = 0u;
                __syncwarp();
                for_each_posting(v, doff, dcnt, lane, [&](uint32_t d, bool valid) {
                    bool ok = valid;
                    for (uint32_t t = 0; t < n; t++) {
                        const uint32_t tc = __shfl_sync(FULL, cnt, t), tb = __shfl_sync(FULL, bmi, t); const uint64_t to = shfl64(off, t);
                        if ((int)t != drv && ok) ok = present_in(v, tc, to, tb, d);
                    }
                    if (ok) atomicOr(&bm[d >> 5], 1u << (d & 31u));
                });
                st_post += dcnt;
            }
        }
        __syncwarp();
        // NOT lists and the delete set clear their bits
        const uint32_t n_not = __ldg(&pl->n_not);
        for (uint32_t i = 0; i < n_not; i++) {
            uint32_t e;
            if (!find_entry(v, pl->tn[i], lv, e)) continue;
            const uint32_t tc = __ldg(&v.e_count[e]), tb = __ldg(&v.e_bitmap[e]); const uint64_t to = __ldg(&v.e_off[e]);
            if (tb != NONE) { for (uint32_t w = lane; w < 1024u; w += 32u) bm64[w] &= ~__ldg(&v.bm_words[(size_t)tb * 1024 + w]); st_words += 1024u; }
            else { for_each_posting(v, to, tc, lane, [&](uint32_t d, bool valid) { if (valid) atomicAnd(&bm[d >> 5], ~(1u << (d & 31u))); }); st_post += tc; }
            __syncwarp();
        }
        if (v.del_slot) {
            const uint32_t slot = __ldg(&v.del_slot[docbase >> 16]);
            if (slot != NONE) for (uint32_t w = lane; w < 1024u; w += 32u) bm64[w] &= ~__ldg(&v.del_words[(size_t)slot * 1024 + w]);
            __syncwarp();
        }
        // ---- 2. the set bits in doc order, 1024 doc ids at a time: the per-doc predicates, then 3. the bins ----
        const uint32_t nf = __ldg(&pl->n_filt), f0 = __ldg(&pl->filt_first), fmask = __ldg(&pl->field_mask), n_phr = __ldg(&pl->n_phr);
        const bool filtered = nf || fmask || n_phr;
        uint32_t* qhist = fc.hist + (size_t)ql * fc.hist_words;
        for (uint32_t w0 = 0; w0 < 2048u; w0 += 32u) {
            uint32_t word = bm[w0 + lane];
            const uint32_t c = __popc(word);
            uint32_t incl = c;
            for (int s = 1; s < 32; s <<= 1) { const uint32_t y = __shfl_up_sync(FULL, incl, s); if (lane >= s) incl += y; }
            const uint32_t total = __shfl_sync(FULL, incl, 31);
            if (total == 0) continue;
            uint32_t pos = incl - c;
            while (word) { const uint32_t b = __ffs(word) - 1; word &= word - 1; list[pos++] = (uint16_t)(((w0 + lane) << 5) | b); }
            __syncwarp();
            for (uint32_t i0 = 0; i0 < total; i0 += 32u) {
                const bool act = i0 + lane < total;
                const uint32_t d = act ? list[i0 + lane] : 0u, doc = docbase | d;
                bool ok = act;
                if (filtered && ok) ok = !filters_reject<FIELD_RUNS, GEO>(v, pl, f0, nf, fmask, n, lv, d, doc);
                const uint64_t row = (uint64_t)doc - v.facet_first_doc;
                ok = ok && doc >= v.facet_first_doc && row < v.facet_rows;          // no facet row: not counted
                const uint32_t n_ok = __popc(__ballot_sync(FULL, ok));
                if (lane == 0) st_docs += n_ok;
                for (uint32_t r = 0; r < fc.n_req; r++) {
                    const FacetReqDev& R = sreq[r];
                    if (R.kind == FREQ_VALUES && R.length == 0) continue;
                    const uint64_t key = ok ? __ldg(&v.facet_keys[(size_t)R.facet * v.facet_rows + row]) : 0ull;
                    if (SETS && R.kind == FREQ_VALUES && __ldg(&csr[2 * r])) {
                        // member j of every lane's combination in one round, warp-aggregated by member id: one atomic per distinct member
                        const uint64_t* so = reinterpret_cast<const uint64_t*>(__ldg(&csr[2 * r]));
                        const uint32_t* sm = reinterpret_cast<const uint32_t*>(__ldg(&csr[2 * r + 1]));
                        const uint64_t b = ok ? __ldg(&so[key]) : 0ull, nm = ok ? __ldg(&so[key + 1]) - b : 0ull;
                        if (ok) st_csr += 16 + nm * 4;
                        const uint32_t rounds = __reduce_max_sync(FULL, (uint32_t)nm);
                        for (uint32_t j = 0; j < rounds; j++) {
                            const uint32_t m = j < nm ? __ldg(&sm[b + j]) : 0xFFFFFFFFu;
                            const unsigned grp = __match_any_sync(FULL, m);
                            if (m != 0xFFFFFFFFu && lane == __ffs(grp) - 1) atomicAdd(&qhist[R.hist_off + m], (uint32_t)__popc(grp));
                        }
                        continue;
                    }
                    if (R.kind == FREQ_VALUES) {                               // warp-aggregated: one atomic per distinct id
                        const unsigned grp = __match_any_sync(FULL, ok ? key : ~0ull);
                        if (ok && lane == __ffs(grp) - 1) atomicAdd(&qhist[R.hist_off + key], (uint32_t)__popc(grp));
                        continue;
                    }
                    bool c2 = ok; uint64_t kk = key;
                    if (R.kind == FREQ_POINT) {
                        if (c2) {
                            const double* b = fc.bases + ((size_t)q * fc.n_point + R.point_idx) * 2;
                            const double dist = geo_distance(key, __ldg(&b[0]), __ldg(&b[1]), [&] { return R.radius; });
                            c2 = dist == dist;                                   // a NaN distance is not counted
                            kk = f64_order_key(dist);
                        }
                    } else if (R.is_float) c2 = c2 && key != ~0ull;             // NaN value
                    uint32_t lo = 0, hi = R.n_bins;                              // the first start above the key
                    while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (sstart[R.start_first + m] <= kk) lo = m + 1; else hi = m; }
                    if (c2 && lo > 0) atomicAdd(&rhist[R.hist_off + lo - 1], 1u);
                }
            }
            __syncwarp();
        }
        for (uint32_t i = lane; i < fc.range_words; i += 32u)
            if (rhist[i]) { atomicAdd(&qhist[i], rhist[i]); rhist[i] = 0; }
        __syncwarp();
    }
    if (lane == 0) {
        atomicAdd((unsigned long long*)&fc.stats[0], (unsigned long long)st_post);
        atomicAdd((unsigned long long*)&fc.stats[1], (unsigned long long)st_words);
        atomicAdd((unsigned long long*)&fc.stats[2], (unsigned long long)st_docs);
    }
    if (SETS && st_csr) atomicAdd((unsigned long long*)&fc.stats[3], (unsigned long long)st_csr);
}

// One CTA per (query of the chunk, request).  RANGES: the bins as they are.  VALUES: the `length` ids with count > 0 (and, with a prefix,
// a value-order rank in [rank_lo, rank_hi); StringSet member ids: the id itself) of largest key (count << 32 | ~id): count descending, id ascending.  A radix select over the
// keys' bytes finds the length-th largest key, the ids at or above it are sorted in shared memory.  Deterministic.
struct RankPtrs { const uint32_t* p[SSB_MAX_FACETS]; };
__global__ void __launch_bounds__(256) facet_select(const FacetReqDev* __restrict__ req, uint32_t n_req, const uint32_t* __restrict__ hist,
                                                    uint32_t hist_words, RankPtrs rank, ssb_facet_count* out, uint32_t out_stride, uint32_t* n_out) {
    __shared__ uint32_t h[256];
    __shared__ uint64_t sel[SSB_MAX_FACET_LENGTH];
    __shared__ uint64_t s_prefix; __shared__ uint32_t s_need, s_all, s_n;
    const uint32_t r = blockIdx.x, ql = blockIdx.y;
    const FacetReqDev R = req[r];
    const uint32_t* qh = hist + (size_t)ql * hist_words + R.hist_off;
    ssb_facet_count* o = out + (size_t)ql * out_stride + R.out_off;
    if (R.kind != FREQ_VALUES) {
        for (uint32_t i = threadIdx.x; i < R.n_bins; i += blockDim.x) { ssb_facet_count c; c.value = i; c.pad = 0; c.count = qh[i]; o[i] = c; }
        if (threadIdx.x == 0) n_out[(size_t)ql * n_req + r] = R.n_bins;
        return;
    }
    if (R.length == 0) { if (threadIdx.x == 0) n_out[(size_t)ql * n_req + r] = 0; return; }
    const uint32_t* rk = rank.p[R.facet];
    auto key_of = [&](uint32_t id) -> uint64_t {                      // 0 = not eligible
        const uint32_t c = qh[id];
        if (c == 0) return 0ull;
        if (R.has_prefix) { const uint32_t x = rk ? __ldg(&rk[id]) : id; if (x < R.rank_lo || x >= R.rank_hi) return 0ull; }
        return ((uint64_t)c << 32) | (0xFFFFFFFFu - id);
    };
    if (threadIdx.x == 0) { s_prefix = 0; s_need = R.length; s_all = 0; s_n = 0; }
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) h[i] = 0;
        __syncthreads();
        const uint64_t pre = s_prefix;
        for (uint32_t id = threadIdx.x; id < R.n_bins; id += blockDim.x) {
            const uint64_t k = key_of(id);
            if (k && (shift == 56 || (k >> (shift + 8)) == (pre >> (shift + 8)))) atomicAdd(&h[(k >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            if (shift == 56) { uint32_t tot = 0; for (int b = 0; b < 256; b++) tot += h[b]; if (tot <= s_need) s_all = 1; }
            if (!s_all) {
                uint32_t acc = 0;
                for (int b = 255; b >= 0; b--) {
                    if (acc + h[b] >= s_need) { s_prefix |= (uint64_t)b << shift; s_need -= acc; break; }
                    acc += h[b];
                }
            }
        }
        __syncthreads();
        if (s_all) break;
    }
    const uint64_t thr = s_all ? 1ull : s_prefix;                    // the smallest key taken
    for (uint32_t id = threadIdx.x; id < R.n_bins; id += blockDim.x) {
        const uint64_t k = key_of(id);
        if (k && k >= thr) sel[atomicAdd(&s_n, 1u)] = k;
    }
    __syncthreads();
    const uint32_t m = s_n;
    uint32_t p2 = 1; while (p2 < m) p2 <<= 1;
    for (uint32_t i = m + threadIdx.x; i < p2; i += blockDim.x) sel[i] = 0;
    __syncthreads();
    for (uint32_t size = 2; size <= p2; size <<= 1)                  // bitonic sort, descending
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t i = threadIdx.x; i < p2 / 2; i += blockDim.x) {
                const uint32_t lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const bool desc = (lo & size) == 0;
                const uint64_t a = sel[lo], b = sel[hi];
                if (desc ? (a < b) : (a > b)) { sel[lo] = b; sel[hi] = a; }
            }
            __syncthreads();
        }
    for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) {
        ssb_facet_count c; c.value = 0xFFFFFFFFu - (uint32_t)sel[i]; c.pad = 0; c.count = sel[i] >> 32; o[i] = c;
    }
    if (threadIdx.x == 0) n_out[(size_t)ql * n_req + r] = m;
}

// ================================================================= host side
int32_t launch_facet_select(const FacetSet& fs, const FacetReqDev* req, uint32_t n_req, const uint32_t* hist, uint32_t hist_words, uint32_t nq,
                            ssb_facet_count* out, uint32_t out_stride, uint32_t* n_out, cudaStream_t st) {
    RankPtrs rk{};
    for (uint32_t f = 0; f < fs.n_facets && f < SSB_MAX_FACETS; f++) rk.p[f] = facet_is_stringset(fs.types[f]) ? nullptr : fs.d_rank[f];
    facet_select<<<dim3(n_req, nq), 256, 0, st>>>(req, n_req, hist, hist_words, rk, out, out_stride, n_out);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

LexIndex::~LexIndex() {
    for (auto& l : levels_) { cudaFree(l.d_term_keys); cudaFree(l.d_posting_offsets); }
    free_committed();
}

void LexIndex::free_committed() {
    cudaFree(d_dict_keys_); cudaFree(d_term_first_); cudaFree(d_term_idf_); cudaFree(d_term_df_);
    cudaFree(d_e_level_); cudaFree(d_e_off_); cudaFree(d_e_count_); cudaFree(d_e_maxcomp_); cudaFree(d_e_bitmap_);
    cudaFree(d_bm_words_); cudaFree(d_bm_); cudaFree(d_bm_q8_); cudaFree(d_level_ids_); cudaFree(d_cache_);
    d_dict_keys_ = nullptr; d_term_first_ = nullptr; d_term_idf_ = nullptr; d_term_df_ = nullptr;
    d_e_level_ = nullptr; d_e_off_ = nullptr; d_e_count_ = nullptr; d_e_maxcomp_ = nullptr; d_e_bitmap_ = nullptr;
    d_bm_words_ = nullptr; d_bm_ = nullptr; d_bm_q8_ = nullptr; d_level_ids_ = nullptr; d_cache_ = nullptr;
    cudaFree(d_lvl_pos_base_); d_lvl_pos_base_ = nullptr;
    committed_ = false;
}

// copy n bytes from a host-or-device pointer into device memory
static cudaError_t to_device(void* dst, const void* src, size_t n, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    return cudaMemcpyAsync(dst, src, n, cudaMemcpyDefault, st);
}

int32_t LexIndex::set_fields(uint32_t n_fields, const float* boosts) {
    if (n_fields == 0 || n_fields > 4) { set_error("set_field_boosts: 1..4 indexed fields"); return SSB_E_UNSUPPORTED; }
    if (!levels_.empty()) { set_error("set_field_boosts: call it before the first level is added"); return SSB_E_STATE; }
    n_fields_ = n_fields;
    for (uint32_t f = 0; f < 4; f++) boosts_[f] = (boosts && f < n_fields) ? boosts[f] : 1.f;
    for (uint32_t f = 0; f < n_fields; f++) if (!(boosts_[f] >= 0.f) || boosts_[f] > 1.0e6f) { set_error("set_field_boosts: boosts must be in [0, 1e6]"); return SSB_E_INVALID; }
    return SSB_OK;
}

int32_t LexIndex::set_ngram_config(uint32_t similarity, uint32_t df_rule) {
    if (similarity > SSB_LEXSIM_BM25F_PROXIMITY || df_rule > SSB_NGRAM_DF_LAST_LEVEL) { set_error("set_ngram_config: unknown similarity / df rule"); return SSB_E_INVALID; }
    if (!levels_.empty()) { set_error("set_ngram_config: call it before the first level is added"); return SSB_E_STATE; }
    lex_sim_ = similarity; ng_rule_ = df_rule;
    return SSB_OK;
}

int32_t LexIndex::add_level_ngrams(const ssb_level_desc* d, const ssb_level_ngrams* ng) {
    if (!ng) return add_level(d);
    if (!d) { set_error("add_level: null level"); return SSB_E_INVALID; }
    if (n_fields_ > 1 || d->n_fields > 1) { set_error("add_level_ngrams: n-gram lists need an index with one indexed field"); return SSB_E_UNSUPPORTED; }
    // the level's n-gram keys: the terms whose key has low bits set
    std::vector<uint64_t> keys(d->n_terms); std::vector<uint32_t> offs((size_t)d->n_terms + 1, 0u);
    if (d->n_terms && d->term_keys && d->posting_offsets) {
        SSB_CUDA_TRY(cudaMemcpy(keys.data(), d->term_keys, (size_t)d->n_terms * 8, cudaMemcpyDefault));
        SSB_CUDA_TRY(cudaMemcpy(offs.data(), d->posting_offsets, ((size_t)d->n_terms + 1) * 4, cudaMemcpyDefault));
    }
    std::vector<uint32_t> ng_terms;
    for (uint32_t t = 0; t < d->n_terms; t++) if (keys[t] & 7u) ng_terms.push_back(t);
    if (ng_terms.empty()) return add_level(d);
    if (plain_lowbit_) { set_error("add_level_ngrams: an earlier level added without n-gram data carried keys with low bits set"); return SSB_E_INVALID; }
    if (!ng->component_tfs || !ng->component_df_bytes) { set_error("add_level_ngrams: null component_tfs / component_df_bytes"); return SSB_E_INVALID; }
    std::vector<uint8_t> dfb((size_t)d->n_terms * 3);
    SSB_CUDA_TRY(cudaMemcpy(dfb.data(), ng->component_df_bytes, dfb.size(), cudaMemcpyDefault));
    const uint64_t base = n_post_;
    SSB_TRY(add_level(d));                                                 // validates the level (offsets ascend) and appends it
    const uint32_t np = offs[d->n_terms];
    std::vector<uint64_t> seg; seg.reserve(ng_terms.size() * 3);
    uint64_t n_tf = 0;
    for (uint32_t t : ng_terms) {
        const uint32_t cnt = offs[t + 1] - offs[t];
        if (!cnt) continue;
        NgSeg g{}; g.key = keys[t]; g.post_off = base + offs[t]; g.tf_off = n_ng_tf_ + n_tf; g.cnt = cnt;
        for (int c = 0; c < 3; c++) g.dfb[c] = dfb[(size_t)t * 3 + c];
        ng_segs_.push_back(g);
        seg.push_back(offs[t]); seg.push_back(n_tf); seg.push_back(cnt);
        n_tf += cnt;
    }
    if (!n_tf) return SSB_OK;
    // the component tfs stay on the host (a re-commit recomputes the components from them); only commit uploads them, for its kernel
    std::vector<uint16_t> all((size_t)np * 3);
    SSB_CUDA_TRY(cudaMemcpy(all.data(), ng->component_tfs, all.size() * 2, cudaMemcpyDefault));
    h_ng_tf_.reserve(h_ng_tf_.size() + n_tf * 3);
    for (size_t j = 0; j < seg.size(); j += 3) h_ng_tf_.insert(h_ng_tf_.end(), all.begin() + 3 * seg[j], all.begin() + 3 * (seg[j] + seg[j + 2]));
    n_ng_tf_ += n_tf;
    return SSB_OK;
}

int32_t LexIndex::add_level_plain(const ssb_level_desc* d) {
    bool low = false;
    if (d && d->n_terms && d->term_keys) {
        std::vector<uint64_t> keys(d->n_terms);
        SSB_CUDA_TRY(cudaMemcpy(keys.data(), d->term_keys, (size_t)d->n_terms * 8, cudaMemcpyDefault));
        for (uint64_t k : keys) low = low || (k & 7u) != 0;
    }
    if (low && has_ngrams()) { set_error("add_level: keys with low bits set on an index with n-gram lists (ssb_lexical_add_level_ngrams)"); return SSB_E_INVALID; }
    SSB_TRY(add_level(d));
    plain_lowbit_ = plain_lowbit_ || low;
    return SSB_OK;
}

int32_t LexIndex::add_level(const ssb_level_desc* d) {
    const uint32_t nf = n_fields_;
    if (d && (d->n_fields > 1 ? d->n_fields : 1u) != nf) { set_error("add_level: the level carries %u field(s), the index %u", d->n_fields > 1 ? d->n_fields : 1u, nf); return SSB_E_INVALID; }
    if (!d || d->n_docs == 0 || d->n_docs > 65536) { set_error("add_level: n_docs must be in 1..65536"); return SSB_E_INVALID; }
    if (d->level_id >= 65536) { set_error("add_level: level_id must be < 65536 (doc id = level_id << 16 | local)"); return SSB_E_INVALID; }
    if (d->n_terms && (!d->term_keys || !d->posting_offsets)) { set_error("add_level: null term_keys / posting_offsets"); return SSB_E_INVALID; }
    if (levels_.size() >= MAX_LEVELS) { set_error("add_level: more than %u levels per GPU unsupported", MAX_LEVELS); return SSB_E_UNSUPPORTED; }
    for (auto& l : levels_) if (l.level_id == d->level_id) { set_error("add_level: duplicate level_id %u", d->level_id); return SSB_E_INVALID; }
    if (!levels_.empty() && d->level_id < levels_.back().level_id) { set_error("add_level: levels must be added in ascending level_id order"); return SSB_E_INVALID; }
    // ---- the whole input contract is checked BEFORE anything is appended to the arenas (a violated contract would make the
    // scoring kernel read out of bounds or mis-rank silently): offsets start at 0 and ascend, term keys are unique inside
    // the level, ids ascend strictly inside a term and are < n_docs, tf >= 1
    DevTmp<uint64_t> t_keys, t_sorted; DevTmp<uint32_t> t_offs, t_bad;
    SSB_CUDA_TRY(t_keys.alloc(d->n_terms)); SSB_CUDA_TRY(t_offs.alloc((size_t)d->n_terms + 1)); SSB_CUDA_TRY(t_bad.alloc(1));
    SSB_CUDA_TRY(cudaMemsetAsync(t_bad.p, 0, 4, st_));
    SSB_CUDA_TRY(to_device(t_keys.p, d->term_keys, (size_t)d->n_terms * 8, st_));
    if (d->n_terms) SSB_CUDA_TRY(to_device(t_offs.p, d->posting_offsets, ((size_t)d->n_terms + 1) * 4, st_));
    else SSB_CUDA_TRY(cudaMemsetAsync(t_offs.p, 0, 4, st_));
    uint32_t np = 0, bad = 0;
    if (d->n_terms) {
        validate_offsets<<<(d->n_terms + 255) / 256, 256, 0, st_>>>(t_offs.p, d->n_terms, t_bad.p);
        SSB_CUDA_TRY(cudaGetLastError());
        SSB_CUDA_TRY(t_sorted.alloc(d->n_terms));
        SSB_CUDA_TRY(cudaMemcpyAsync(t_sorted.p, t_keys.p, (size_t)d->n_terms * 8, cudaMemcpyDeviceToDevice, st_));
        thrust::sort(thrust::cuda::par.on(st_), thrust::device_ptr<uint64_t>(t_sorted.p), thrust::device_ptr<uint64_t>(t_sorted.p + d->n_terms));
        validate_keys_sorted_unique<<<(d->n_terms + 255) / 256, 256, 0, st_>>>(t_sorted.p, d->n_terms, t_bad.p);
        SSB_CUDA_TRY(cudaGetLastError());
        SSB_CUDA_TRY(cudaMemcpyAsync(&np, t_offs.p + d->n_terms, 4, cudaMemcpyDeviceToHost, st_));
        SSB_CUDA_TRY(cudaMemcpyAsync(&bad, t_bad.p, 4, cudaMemcpyDeviceToHost, st_));
        SSB_CUDA_TRY(cudaStreamSynchronize(st_));
        if (bad) { set_error("add_level %u: malformed directory (%u violations: posting_offsets must start at 0 and ascend, term_keys must be unique)", d->level_id, bad); return SSB_E_INVALID; }
    }
    if (np && (!d->doc_ids || !d->tfs || !d->doc_len_bytes)) { set_error("add_level: null doc_ids / tfs / doc_len_bytes"); return SSB_E_INVALID; }
    const uint16_t* d_ids = nullptr; const uint16_t* d_tfs = nullptr; const uint8_t* d_len = nullptr;
    DevTmp<uint16_t> t_ids, t_tfs; DevTmp<uint8_t> t_len;
    if (np) {
        if (is_device_ptr(d->doc_ids)) d_ids = d->doc_ids;
        else { SSB_CUDA_TRY(t_ids.alloc(np)); d_ids = t_ids.p; SSB_CUDA_TRY(to_device(t_ids.p, d->doc_ids, (size_t)np * 2, st_)); }
        if (is_device_ptr(d->tfs)) d_tfs = d->tfs;
        else { SSB_CUDA_TRY(t_tfs.alloc((size_t)np * nf)); d_tfs = t_tfs.p; SSB_CUDA_TRY(to_device(t_tfs.p, d->tfs, (size_t)np * nf * 2, st_)); }
        if (is_device_ptr(d->doc_len_bytes)) d_len = d->doc_len_bytes;
        else { SSB_CUDA_TRY(t_len.alloc((size_t)d->n_docs * nf)); d_len = t_len.p; SSB_CUDA_TRY(to_device(t_len.p, d->doc_len_bytes, (size_t)d->n_docs * nf, st_)); }
        validate_level<<<(np + 255) / 256, 256, 0, st_>>>(d_ids, d_tfs, t_offs.p, d->n_terms, np, d->n_docs, t_bad.p, nf);
        SSB_CUDA_TRY(cudaGetLastError());
        SSB_CUDA_TRY(cudaMemcpyAsync(&bad, t_bad.p, 4, cudaMemcpyDeviceToHost, st_));
        SSB_CUDA_TRY(cudaStreamSynchronize(st_));
        if (bad) {
            set_error("add_level %u: malformed postings (%u violations: ids must ascend strictly inside a term and be < n_docs, tf >= 1)", d->level_id, bad);
            return SSB_E_INVALID;
        }
        // validated: append (n_post_ advances only after the kernels were enqueued without error)
        SSB_TRY(post_.reserve(n_post_ + np + 160, n_post_, st_));     // +160: the 16-byte vector loads of the stream may run past the end
        SSB_TRY(pay_.reserve(n_post_ + np + 160, n_post_, st_));
        if (nf > 1) SSB_TRY(payf_.reserve((n_post_ + np) * nf + 16, n_post_ * nf, st_));
        build_postings<<<(np + 255) / 256, 256, 0, st_>>>(d_ids, d_tfs, d_len, post_.p + n_post_, pay_.p + n_post_, np, nf, d->n_docs,
                                                          nf > 1 ? payf_.p + n_post_ * nf : nullptr);
        SSB_CUDA_TRY(cudaGetLastError());
        SSB_CUDA_TRY(cudaStreamSynchronize(st_));
    } else {
        SSB_TRY(post_.reserve(n_post_ + 160, n_post_, st_));
        SSB_TRY(pay_.reserve(n_post_ + 160, n_post_, st_));
    }
    // term positions (phrase queries): all levels or none
    const int has_pos = d->positions ? 1 : 0;
    if (np) {
        if (has_positions_ >= 0 && has_positions_ != has_pos) { set_error("add_level %u: either every level carries positions or none", d->level_id); return SSB_E_INVALID; }
    }
    uint64_t level_positions = 0;
    if (np && has_pos) {
        SSB_TRY(pos_off_.reserve(n_post_ + np, n_post_, st_));
        uint32_t* off = pos_off_.p + n_post_;
        widen_tf<<<(np + 255) / 256, 256, 0, st_>>>(d_tfs, off, np, nf);          // a posting's positions: Σ_f tf_f, field by field
        SSB_CUDA_TRY(cudaGetLastError());
        uint32_t last_tf = 0, last_off = 0;
        SSB_CUDA_TRY(cudaMemcpyAsync(&last_tf, off + np - 1, 4, cudaMemcpyDeviceToHost, st_));
        thrust::exclusive_scan(thrust::cuda::par.on(st_), thrust::device_ptr<uint32_t>(off), thrust::device_ptr<uint32_t>(off + np), thrust::device_ptr<uint32_t>(off));
        SSB_CUDA_TRY(cudaMemcpyAsync(&last_off, off + np - 1, 4, cudaMemcpyDeviceToHost, st_));
        SSB_CUDA_TRY(cudaStreamSynchronize(st_));
        level_positions = (uint64_t)last_off + last_tf;
        if (level_positions >= 0xFFFFFFFFull) { set_error("add_level %u: more than 2^32 positions in one level", d->level_id); return SSB_E_UNSUPPORTED; }
        SSB_TRY(positions_.reserve(n_positions_ + level_positions + 8, n_positions_, st_));
        SSB_CUDA_TRY(to_device(positions_.p + n_positions_, d->positions, (size_t)level_positions * 2, st_));
        SSB_CUDA_TRY(cudaMemsetAsync(t_bad.p, 0, 4, st_));
        validate_positions<<<(np + 255) / 256, 256, 0, st_>>>(positions_.p + n_positions_, off, d_tfs, np, nf, t_bad.p);
        SSB_CUDA_TRY(cudaGetLastError());
        SSB_CUDA_TRY(cudaMemcpyAsync(&bad, t_bad.p, 4, cudaMemcpyDeviceToHost, st_));
        SSB_CUDA_TRY(cudaStreamSynchronize(st_));
        if (bad) {
            if (nf > 1) set_error("add_level %u: %u postings whose positions do not ascend strictly inside one field's run", d->level_id, bad);
            else set_error("add_level %u: %u postings whose positions do not ascend strictly", d->level_id, bad);
            return SSB_E_INVALID;
        }
    }
    if (np) has_positions_ = has_pos;
    h_lvl_pos_base_.push_back(n_positions_);
    n_positions_ += level_positions;
    LexLevel l{};
    l.level_id = d->level_id; l.n_docs = d->n_docs; l.n_terms = d->n_terms; l.post_base = n_post_; l.n_post = np;
    l.d_term_keys = t_keys.release(); l.d_posting_offsets = t_offs.release();
    n_post_ += np;
    levels_.push_back(l);
    committed_ = false;
    return SSB_OK;
}

// DOCUMENT_LENGTH_COMPRESSION (byte4_to_int, index.rs:4255-4279)
static uint32_t byte4_to_int(uint32_t b) {
    if (b < 24) return b;
    const uint32_t x = b - 24, bits = x & 7, shift = x >> 3;
    return shift == 0 ? 24 + bits : 24 + ((bits | 8) << (shift - 1));
}

static void host_bm25_cache(uint64_t n_docs, uint64_t len_sum, float* cache) {
    // commit.rs:318-325; DOCUMENT_LENGTH_COMPRESSION = byte4_to_int (index.rs:4255-4279).  volatile keeps every
    // f32 operation individually rounded regardless of host compiler contraction settings.
    volatile float avgdl = (float)len_sum / (float)n_docs;
    const float K = 1.2f, B = 0.75f;
    for (int i = 0; i < 256; i++) {
        const uint32_t v = byte4_to_int((uint32_t)i);
        volatile float quot = (float)v / avgdl;
        volatile float bq = B * quot;
        volatile float omb = 1.0f - B;
        volatile float inner = omb + bq;
        cache[i] = K * inner;
    }
}

static float host_idf(uint64_t n_docs, uint32_t df) {
    // search.rs:3225-3230
    volatile float a = (float)n_docs - (float)df;
    volatile float num = a + 0.5f;
    volatile float den = (float)df + 0.5f;
    volatile float r = num / den;
    volatile float r1 = r + 1.0f;
    return logf(r1);
}

LexView LexIndex::view() const {
    LexView v{};
    v.dict_keys = d_dict_keys_; v.n_terms = n_terms_; v.term_first = d_term_first_; v.term_idf = d_term_idf_; v.term_df = d_term_df_;
    v.e_level = d_e_level_; v.e_off = d_e_off_; v.e_count = d_e_count_; v.e_maxcomp = d_e_maxcomp_; v.e_bitmap = d_e_bitmap_;
    v.post = post_.p; v.pay = pay_.p; v.comp = comp_.p; v.bm_words = d_bm_words_; v.bm = d_bm_; v.bm_q8 = d_bm_q8_; v.q8_step = q8_step_ > 0.f ? q8_step_ : Q8_STEP; v.level_ids = d_level_ids_;
    v.n_levels = (uint32_t)levels_.size(); v.cache = d_cache_;
    v.k1p = 1.2f + 1.0f;
    v.payf = payf_.p; v.compf = compf_.p; v.n_fields = n_fields_; v.fast_t = n_fields_ > 1 ? 0u : FAST_T;
    for (int f = 0; f < 4; f++) v.boost[f] = boosts_[f];
    if (del_ && del_->n) { v.del_slot = del_->d_slot; v.del_words = del_->d_words; v.del_docs = del_->d_docs; v.n_del = del_->n; }
    if (has_positions_ == 1 && d_lvl_pos_base_) { v.positions = positions_.p; v.pos_off = pos_off_.p; v.lvl_pos_base = d_lvl_pos_base_; }
    if (facets_ && facets_->n_facets) { v.facet_keys = facets_->d_keys; v.facet_rows = facets_->n_rows; v.facet_first_doc = facets_->first_doc; v.n_facets = facets_->n_facets; }
    return v;
}

// the n-gram lists at commit: each key's component dfs from the df bytes of its first or last level (ng_rule_), the component idfs over
// n_docs (search.rs:3231-3269), then fill_ngram_bounds on every segment; the coarse bound step grows with the largest component
int32_t LexIndex::commit_ngrams(uint64_t n_docs) {
    h_ng_keys_.clear();
    if (ng_segs_.empty()) return SSB_OK;
    std::vector<uint32_t> order(ng_segs_.size());
    for (uint32_t i = 0; i < order.size(); i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return ng_segs_[a].key < ng_segs_[b].key; });   // levels ascend in a key
    std::vector<NgSegDev> segs(ng_segs_.size());
    for (size_t a = 0; a < order.size();) {
        size_t b = a;
        while (b < order.size() && ng_segs_[order[b]].key == ng_segs_[order[a]].key) b++;
        const NgSeg& src = ng_segs_[order[ng_rule_ == SSB_NGRAM_DF_LAST_LEVEL ? b - 1 : a]];
        const uint32_t ty = (uint32_t)(src.key & 7u);
        const uint32_t n_comp = lex_sim_ == SSB_LEXSIM_BM25F ? (ty <= SSB_NGRAM_RF ? 2u : 3u) : 0u;
        float idf[3] = {0.f, 0.f, 0.f};
        for (uint32_t c = 0; c < n_comp; c++) idf[c] = host_idf(n_docs, byte4_to_int(src.dfb[c]));
        for (size_t j = a; j < b; j++) {
            const NgSeg& g = ng_segs_[order[j]];
            NgSegDev& o = segs[order[j]];
            o.post_off = g.post_off; o.tf_off = g.tf_off; o.cnt = g.cnt; o.n_comp = n_comp; o.pad = 0;
            for (int c = 0; c < 3; c++) o.idf[c] = idf[c];
        }
        h_ng_keys_.push_back(src.key);
        a = b;
    }
    DevTmp<NgSegDev> t_segs; DevTmp<uint32_t> t_max; DevTmp<uint16_t> t_tf;
    SSB_CUDA_TRY(t_segs.alloc(segs.size())); SSB_CUDA_TRY(t_max.alloc(1)); SSB_CUDA_TRY(t_tf.alloc(h_ng_tf_.size()));
    SSB_CUDA_TRY(to_device(t_segs.p, segs.data(), segs.size() * sizeof(NgSegDev), st_));
    SSB_CUDA_TRY(to_device(t_tf.p, h_ng_tf_.data(), h_ng_tf_.size() * 2, st_));
    SSB_CUDA_TRY(cudaMemsetAsync(t_max.p, 0, 4, st_));
    LexView v{};
    v.pay = pay_.p; v.cache = d_cache_; v.k1p = 1.2f + 1.0f;
    fill_ngram_bounds<<<(unsigned)((n_ng_tf_ + 255) / 256), 256, 0, st_>>>(v, t_segs.p, (uint32_t)segs.size(), t_tf.p, n_ng_tf_, post_.p, comp_.p, t_max.p);
    SSB_CUDA_TRY(cudaGetLastError());
    uint32_t maxbits = 0;
    SSB_CUDA_TRY(cudaMemcpyAsync(&maxbits, t_max.p, 4, cudaMemcpyDeviceToHost, st_));
    SSB_CUDA_TRY(cudaStreamSynchronize(st_));
    float maxc; memcpy(&maxc, &maxbits, 4);
    // build_bitmaps clamps a word's coarse bound to 255 steps: the step must reach the largest fp16 bound (1 % covers the round-up)
    if (maxc * 1.01f / 255.0f > q8_step_) q8_step_ = maxc * 1.01f / 255.0f;
    return SSB_OK;
}

// the dictionary idf of every n-gram key is 1.0 (score = 1.0 * component sum)
void LexIndex::ngram_idf_one(std::vector<float>& idf) const {
    for (uint64_t key : h_ng_keys_) {
        const auto it = std::lower_bound(h_dict_keys_.begin(), h_dict_keys_.end(), key);
        if (it != h_dict_keys_.end() && *it == key) idf[it - h_dict_keys_.begin()] = 1.0f;
    }
}

int32_t LexIndex::commit(uint64_t n_docs, uint64_t len_sum) {
    if (n_docs == 0) { set_error("commit: n_docs must be > 0"); return SSB_E_INVALID; }
    free_committed();
    n_docs_ = n_docs; len_sum_ = len_sum;
    const uint32_t nlv = (uint32_t)levels_.size();
    uint64_t total64 = 0;
    for (auto& l : levels_) total64 += l.n_terms;
    if (total64 >= 0xFFFFFFFFull) { set_error("commit: too many (term, level) entries"); return SSB_E_UNSUPPORTED; }
    if (n_post_ >= (1ull << 44)) { set_error("commit: more than 2^44 postings per GPU unsupported"); return SSB_E_UNSUPPORTED; }
    const uint32_t total = (uint32_t)total64;
    n_entries_ = total;
    auto pol = thrust::cuda::par.on(st_);

    float cache[256];
    host_bm25_cache(n_docs, len_sum, cache);
    SSB_CUDA_TRY(cudaMalloc(&d_cache_, 256 * 4));
    SSB_CUDA_TRY(cudaMemcpyAsync(d_cache_, cache, 256 * 4, cudaMemcpyHostToDevice, st_));
    std::vector<uint32_t> lids(nlv ? nlv : 1); std::vector<uint64_t> lbase(nlv ? nlv : 1); std::vector<const uint32_t*> loffs(nlv ? nlv : 1);
    for (uint32_t i = 0; i < nlv; i++) { lids[i] = levels_[i].level_id; lbase[i] = levels_[i].post_base; loffs[i] = levels_[i].d_posting_offsets; }
    if (has_positions_ == 1) {
        SSB_CUDA_TRY(cudaMalloc(&d_lvl_pos_base_, (h_lvl_pos_base_.size() + 1) * 8));
        SSB_CUDA_TRY(cudaMemcpyAsync(d_lvl_pos_base_, h_lvl_pos_base_.data(), h_lvl_pos_base_.size() * 8, cudaMemcpyHostToDevice, st_));
    }
    SSB_CUDA_TRY(cudaMalloc(&d_level_ids_, lids.size() * 4));
    SSB_CUDA_TRY(cudaMemcpyAsync(d_level_ids_, lids.data(), lids.size() * 4, cudaMemcpyHostToDevice, st_));

    // per-posting fp16 upper bounds of the score component (needs the cache, i.e. avgdl)
    if (n_post_) {
        LexView v{};
        v.pay = pay_.p; v.cache = d_cache_; v.k1p = 1.2f + 1.0f;
        v.n_fields = n_fields_; v.payf = payf_.p; for (int f = 0; f < 4; f++) v.boost[f] = boosts_[f];
        if (n_fields_ > 1) { SSB_TRY(compf_.reserve(n_post_ * n_fields_ + 16, 0, st_, true)); v.compf = compf_.p; }
        SSB_TRY(comp_.reserve(n_post_ + 160, 0, st_, true));
        fill_bounds<<<(unsigned)((n_post_ + 255) / 256), 256, 0, st_>>>(v, post_.p, comp_.p, n_post_);
        SSB_CUDA_TRY(cudaGetLastError());
    }
    q8_step_ = Q8_STEP;
    SSB_TRY(commit_ngrams(n_docs));
    if (post_.p) SSB_CUDA_TRY(cudaMemsetAsync(post_.p + n_post_, 0, 160 * 4, st_));   // tail read by the vector loads

    size_t alloc_n = total ? total : 1;
    DevTmp<uint64_t> t_keys, t_vals, t_lbase, t_ukeys; DevTmp<const uint32_t*> t_loffs; DevTmp<uint32_t> t_epc, t_df;
    SSB_CUDA_TRY(t_keys.alloc(alloc_n)); SSB_CUDA_TRY(t_vals.alloc(alloc_n));
    SSB_CUDA_TRY(t_lbase.alloc(lbase.size())); SSB_CUDA_TRY(t_loffs.alloc(loffs.size()));
    uint64_t *d_keys = t_keys.p, *d_vals = t_vals.p, *d_lbase = t_lbase.p; const uint32_t** d_loffs = t_loffs.p;
    SSB_CUDA_TRY(cudaMemcpyAsync(d_lbase, lbase.data(), lbase.size() * 8, cudaMemcpyHostToDevice, st_));
    SSB_CUDA_TRY(cudaMemcpyAsync(d_loffs, loffs.data(), loffs.size() * sizeof(void*), cudaMemcpyHostToDevice, st_));
    uint32_t pos = 0;
    for (uint32_t i = 0; i < nlv; i++) {
        if (levels_[i].n_terms) gather_dict<<<(levels_[i].n_terms + 255) / 256, 256, 0, st_>>>(levels_[i].d_term_keys, levels_[i].n_terms, i, d_keys + pos, d_vals + pos);
        pos += levels_[i].n_terms;
    }
    SSB_CUDA_TRY(cudaGetLastError());
    // stable: entries of one term stay in ascending level order
    thrust::stable_sort_by_key(pol, thrust::device_ptr<uint64_t>(d_keys), thrust::device_ptr<uint64_t>(d_keys + total), thrust::device_ptr<uint64_t>(d_vals));

    SSB_CUDA_TRY(cudaMalloc(&d_e_level_, alloc_n * 4)); SSB_CUDA_TRY(cudaMalloc(&d_e_off_, alloc_n * 8));
    SSB_CUDA_TRY(cudaMalloc(&d_e_count_, alloc_n * 4)); SSB_CUDA_TRY(cudaMalloc(&d_e_maxcomp_, alloc_n * 4));
    SSB_CUDA_TRY(cudaMalloc(&d_e_bitmap_, alloc_n * 4));
    if (total) build_entries<<<(total + 255) / 256, 256, 0, st_>>>(d_vals, total, d_loffs, d_lbase, d_e_level_, d_e_off_, d_e_count_);
    SSB_CUDA_TRY(cudaGetLastError());

    // dictionary: unique keys, entries per term, df per term
    SSB_CUDA_TRY(t_ukeys.alloc(alloc_n)); SSB_CUDA_TRY(t_epc.alloc(alloc_n + 1)); SSB_CUDA_TRY(t_df.alloc(alloc_n));
    uint64_t* d_ukeys = t_ukeys.p; uint32_t *d_epc = t_epc.p, *d_df = t_df.p;
    uint32_t nt = 0;
    if (total) {
        auto e1 = thrust::reduce_by_key(pol, thrust::device_ptr<uint64_t>(d_keys), thrust::device_ptr<uint64_t>(d_keys + total),
                                        thrust::constant_iterator<uint32_t>(1), thrust::device_ptr<uint64_t>(d_ukeys), thrust::device_ptr<uint32_t>(d_epc));
        nt = (uint32_t)(e1.first - thrust::device_ptr<uint64_t>(d_ukeys));
        thrust::reduce_by_key(pol, thrust::device_ptr<uint64_t>(d_keys), thrust::device_ptr<uint64_t>(d_keys + total),
                              thrust::device_ptr<uint32_t>(d_e_count_), thrust::make_discard_iterator(), thrust::device_ptr<uint32_t>(d_df));
    }
    n_terms_ = nt;
    size_t nt_alloc = nt ? nt : 1;
    SSB_CUDA_TRY(cudaMalloc(&d_dict_keys_, nt_alloc * 8)); SSB_CUDA_TRY(cudaMalloc(&d_term_first_, (nt_alloc + 1) * 4));
    SSB_CUDA_TRY(cudaMalloc(&d_term_idf_, nt_alloc * 4)); SSB_CUDA_TRY(cudaMalloc(&d_term_df_, nt_alloc * 4));
    SSB_CUDA_TRY(cudaMemcpyAsync(d_dict_keys_, d_ukeys, (size_t)nt * 8, cudaMemcpyDeviceToDevice, st_));
    SSB_CUDA_TRY(cudaMemcpyAsync(d_term_df_, d_df, (size_t)nt * 4, cudaMemcpyDeviceToDevice, st_));
    SSB_CUDA_TRY(cudaMemsetAsync(d_term_first_, 0, 4, st_));
    if (nt) thrust::inclusive_scan(pol, thrust::device_ptr<uint32_t>(d_epc), thrust::device_ptr<uint32_t>(d_epc + nt), thrust::device_ptr<uint32_t>(d_term_first_ + 1));
    h_dict_keys_.resize(nt); h_term_df_.resize(nt);
    SSB_CUDA_TRY(cudaMemcpyAsync(h_dict_keys_.data(), d_dict_keys_, (size_t)nt * 8, cudaMemcpyDeviceToHost, st_));
    SSB_CUDA_TRY(cudaMemcpyAsync(h_term_df_.data(), d_term_df_, (size_t)nt * 4, cudaMemcpyDeviceToHost, st_));
    SSB_CUDA_TRY(cudaStreamSynchronize(st_));
    h_local_df_ = h_term_df_;
    {   // idf on the host (same libm as the oracle)
        std::vector<float> idf(nt_alloc);
        for (uint32_t t = 0; t < nt; t++) idf[t] = host_idf(n_docs, h_term_df_[t]);
        ngram_idf_one(idf);
        SSB_CUDA_TRY(cudaMemcpyAsync(d_term_idf_, idf.data(), (size_t)nt * 4, cudaMemcpyHostToDevice, st_));
        SSB_CUDA_TRY(cudaStreamSynchronize(st_));
    }

    // bitmaps for dense lists
    n_bitmaps_ = 0;
    if (total) {
        DevTmp<uint32_t> t_flags, t_scan, t_dense;
        SSB_CUDA_TRY(t_flags.alloc(alloc_n)); SSB_CUDA_TRY(t_scan.alloc(alloc_n));
        uint32_t *d_flags = t_flags.p, *d_scan = t_scan.p;
        mark_dense<<<(total + 255) / 256, 256, 0, st_>>>(d_e_count_, total, d_flags);
        thrust::exclusive_scan(pol, thrust::device_ptr<uint32_t>(d_flags), thrust::device_ptr<uint32_t>(d_flags + total), thrust::device_ptr<uint32_t>(d_scan));
        uint32_t last_flag = 0, last_scan = 0;
        SSB_CUDA_TRY(cudaMemcpyAsync(&last_flag, d_flags + total - 1, 4, cudaMemcpyDeviceToHost, st_));
        SSB_CUDA_TRY(cudaMemcpyAsync(&last_scan, d_scan + total - 1, 4, cudaMemcpyDeviceToHost, st_));
        SSB_CUDA_TRY(cudaStreamSynchronize(st_));
        n_bitmaps_ = last_flag + last_scan;
        assign_bitmap<<<(total + 255) / 256, 256, 0, st_>>>(d_e_count_, d_scan, total, d_e_bitmap_);
        SSB_CUDA_TRY(cudaGetLastError());
        if (n_bitmaps_) {
            SSB_CUDA_TRY(cudaMalloc(&d_bm_words_, (size_t)n_bitmaps_ * 1024 * 8));
            SSB_CUDA_TRY(cudaMalloc(&d_bm_, (size_t)n_bitmaps_ * 512 * sizeof(BmSec)));
            SSB_CUDA_TRY(cudaMalloc(&d_bm_q8_, (size_t)n_bitmaps_ * 1024));
            SSB_CUDA_TRY(t_dense.alloc(n_bitmaps_));
            uint32_t* d_dense = t_dense.p;
            compact_dense<<<(total + 255) / 256, 256, 0, st_>>>(d_e_bitmap_, total, d_dense);
            build_bitmaps<<<n_bitmaps_, 256, 0, st_>>>(d_e_bitmap_, d_e_off_, d_e_count_, total, post_.p, d_bm_words_, d_bm_, d_bm_q8_, q8_step_, d_dense);
            SSB_CUDA_TRY(cudaGetLastError());
            SSB_CUDA_TRY(cudaStreamSynchronize(st_));
        }
        SSB_CUDA_TRY(cudaStreamSynchronize(st_));
    }

    if (total) {
        LexView v = view();
        entry_maxcomp<<<(total + 7) / 8, 256, 0, st_>>>(v, total, d_e_maxcomp_);
        SSB_CUDA_TRY(cudaGetLastError());
    }
    SSB_CUDA_TRY(cudaStreamSynchronize(st_));
    committed_ = true;
    refresh_live_docs();
    return SSB_OK;
}

int32_t LexIndex::dict_export(uint64_t* keys, uint32_t* dfs, uint64_t cap) const {
    if (!committed_) { set_error("dict_export before commit"); return SSB_E_STATE; }
    if (cap < n_terms_) { set_error("dict_export: capacity too small"); return SSB_E_INVALID; }
    if (keys) memcpy(keys, h_dict_keys_.data(), (size_t)n_terms_ * 8);
    if (dfs) memcpy(dfs, h_term_df_.data(), (size_t)n_terms_ * 4);
    return SSB_OK;
}

int32_t LexIndex::set_global_df(const uint64_t* keys, const uint32_t* dfs, uint64_t n) {
    if (!committed_) { set_error("set_global_df before commit"); return SSB_E_STATE; }
    std::vector<float> idf(n_terms_ ? n_terms_ : 1);
    for (uint64_t i = 0; i < n; i++) {
        size_t lo = 0, hi = n_terms_;
        while (lo < hi) { size_t m = (lo + hi) / 2; if (h_dict_keys_[m] < keys[i]) lo = m + 1; else hi = m; }
        if (lo < n_terms_ && h_dict_keys_[lo] == keys[i]) h_term_df_[lo] = dfs[i];
    }
    for (uint32_t t = 0; t < n_terms_; t++) idf[t] = host_idf(n_docs_, h_term_df_[t]);
    ngram_idf_one(idf);                                                    // n-gram keys: the components carry the idfs
    SSB_CUDA_TRY(cudaMemcpyAsync(d_term_idf_, idf.data(), (size_t)n_terms_ * 4, cudaMemcpyHostToDevice, st_));
    SSB_CUDA_TRY(cudaMemcpyAsync(d_term_df_, h_term_df_.data(), (size_t)n_terms_ * 4, cudaMemcpyHostToDevice, st_));
    SSB_CUDA_TRY(cudaStreamSynchronize(st_));
    return SSB_OK;
}

int32_t LexIndex::ensure_workspace(LexWorkspace& ws, cudaStream_t st, uint32_t nq, uint32_t total_terms) const {
    const size_t cq = nq > max_batch_ ? nq : max_batch_;
    const size_t ct = total_terms > cq * 4 ? total_terms : cq * 4;
    const size_t nl1 = levels_.empty() ? 1 : levels_.size();
    SSB_TRY(ws.plans.reserve(cq, 0, st, true));
    SSB_TRY(ws.recs.reserve(cq * nl1, 0, st, true));
    SSB_TRY(ws.item_start.reserve(cq * (nl1 + 1), 0, st, true));
    SSB_TRY(ws.theta.reserve(cq * 2, 0, st, true));
    SSB_TRY(ws.lock.reserve(cq, 0, st, true));
    SSB_TRY(ws.count.reserve(cq, 0, st, true));
    SSB_TRY(ws.ctr.reserve(8, 0, st, true));
    SSB_TRY(ws.qoff.reserve(cq + 1, 0, st, true));
    SSB_TRY(ws.qkeys.reserve(ct, 0, st, true));
    SSB_TRY(ws.qflags.reserve(ct, 0, st, true));
    SSB_TRY(ws.stats.reserve(1, 0, st, true));
    return SSB_OK;
}

int32_t LexIndex::prepare_sort(const ssb_sort_criterion* crit, uint32_t n, bool has_bases, SortDev* out, bool* sorted) const {
    SortDev s{};
    SSB_TRY(sort_of_criteria(facets_, crit, n, has_bases, &s, sorted));
    if (!*sorted) return SSB_OK;
    bool any_facet = false;
    for (uint32_t j = 0; j < s.n; j++) any_facet = any_facet || s.src[j] == SORT_SRC_FACET;
    if (any_facet) {
        for (const LexLevel& l : levels_) {                           // a sorted doc must have a facet value
            const uint64_t d0 = (uint64_t)l.level_id << 16;
            if (l.n_docs && (d0 < facets_->first_doc || d0 + l.n_docs > (uint64_t)facets_->first_doc + facets_->n_rows)) {
                set_error("search_lexical_sorted: the facet rows do not cover level %u", l.level_id); return SSB_E_STATE;
            }
        }
    }
    *out = s;
    return SSB_OK;
}

int32_t LexIndex::stage_sort_bases(LexWorkspace& ws, cudaStream_t st, const double* bases, uint32_t nq, SortDev* sort) {
    if (!sort_has_point(*sort) || nq == 0) return SSB_OK;
    if (is_device_ptr(bases)) { set_error("search_lexical_sorted: bases must be a host array"); return SSB_E_INVALID; }
    SSB_TRY(ws.bases.reserve((size_t)nq * 2, 0, st, true));
    SSB_CUDA_TRY(cudaMemcpyAsync(ws.bases.p, bases, (size_t)nq * 16, cudaMemcpyHostToDevice, st));
    sort->bases = ws.bases.p;
    return SSB_OK;
}

int32_t LexIndex::stage_filters(LexWorkspace& ws, cudaStream_t st, const ssb_lex_batch* q, LexView& v, bool* any, bool* geo_any) const {
    const uint32_t nq = q->n_queries;
    if (is_device_ptr(q->filter_offsets) || (q->filters && is_device_ptr(q->filters)) || (q->filter_set_values && is_device_ptr(q->filter_set_values))) { set_error("search_lexical: filter arrays must be host arrays"); return SSB_E_INVALID; }
    const uint32_t nf = q->filter_offsets[nq];
    *any = false; *geo_any = false;
    if (nf == 0) return SSB_OK;
    if (!q->filters) { set_error("search_lexical: null filters"); return SSB_E_INVALID; }
    if (!facets_ || !facets_->n_facets) { set_error("search_lexical: facet filters need ssb_set_facets"); return SSB_E_STATE; }
    std::vector<FiltDev> fd(nf);
    std::vector<uint64_t> geo;                                       // POINT payloads (GEO_WORDS each) and MEMBERS payloads, staged behind the SET values
    uint32_t n_sets = 0;
    for (uint32_t i = 0; i < nq; i++) {
        if (q->filter_offsets[i + 1] < q->filter_offsets[i] || q->filter_offsets[i + 1] > nf) { set_error("query %u: filter_offsets must ascend", i); return SSB_E_INVALID; }
        if (q->filter_offsets[i + 1] - q->filter_offsets[i] > SSB_MAX_FILTERS_PER_QUERY) { set_error("query %u: more than %u facet filters", i, SSB_MAX_FILTERS_PER_QUERY); return SSB_E_UNSUPPORTED; }
    }
    for (uint32_t i = 0; i < nf; i++) {
        const ssb_facet_filter& f = q->filters[i];
        if (f.facet >= facets_->n_facets) { set_error("facet filter %u: facet %u of %u", i, f.facet, facets_->n_facets); return SSB_E_INVALID; }
        SSB_TRY(encode_filter(f, i, facets_->types[f.facet], q->filter_set_values, &fd[i], geo, facets_->n_sets[f.facet], facets_->n_values[f.facet]));
        if (fd[i].kind == FILT_MEMBERS) { fd[i].lo = (uint64_t)facets_->d_set_off[f.facet]; fd[i].hi = (uint64_t)facets_->d_set_mem[f.facet]; }
        *geo_any = *geo_any || fd[i].kind == FILT_POINT || fd[i].kind == FILT_MEMBERS;   // the out-of-line tests: the GEO instantiations
        if (f.kind == SSB_FILTER_SET && (uint64_t)f.set_first + f.set_count > n_sets) n_sets = f.set_first + f.set_count;
    }
    for (uint32_t i = 0; i < nf; i++) if (fd[i].kind == FILT_POINT || fd[i].kind == FILT_MEMBERS) fd[i].set_first += n_sets;
    const uint32_t n_staged = n_sets + (uint32_t)geo.size();
    SSB_TRY(ws.foff.reserve((size_t)nq + 1, 0, st, true));
    SSB_TRY(ws.filt.reserve(nf, 0, st));
    SSB_TRY(ws.fsets.reserve(n_staged, 0, st));
    // pageable host sources: cudaMemcpyAsync returns after staging them, the vectors may go out of scope
    SSB_CUDA_TRY(cudaMemcpyAsync(ws.foff.p, q->filter_offsets, ((size_t)nq + 1) * 4, cudaMemcpyHostToDevice, st));
    SSB_CUDA_TRY(cudaMemcpyAsync(ws.filt.p, fd.data(), (size_t)nf * sizeof(FiltDev), cudaMemcpyHostToDevice, st));
    if (n_sets) SSB_CUDA_TRY(cudaMemcpyAsync(ws.fsets.p, q->filter_set_values, (size_t)n_sets * 8, cudaMemcpyHostToDevice, st));
    if (!geo.empty()) SSB_CUDA_TRY(cudaMemcpyAsync(ws.fsets.p + n_sets, geo.data(), geo.size() * 8, cudaMemcpyHostToDevice, st));
    v.filt = ws.filt.p; v.filt_sets = ws.fsets.p;
    *any = true;
    return SSB_OK;
}

int32_t LexIndex::stage_batch(LexWorkspace& ws, cudaStream_t st, const ssb_lex_batch* q, LexView& v, bool* filtered, bool* geo,
                              const uint32_t** fmask_dev) const {
    const uint32_t nq = q->n_queries;
    uint32_t total_terms = 0;
    const bool off_dev = is_device_ptr(q->term_offsets);
    if (off_dev) SSB_CUDA_TRY(cudaMemcpy(&total_terms, q->term_offsets + nq, 4, cudaMemcpyDeviceToHost));
    else {
        total_terms = q->term_offsets[nq];
        for (uint32_t i = 0; i < nq; i++) {
            if (q->term_offsets[i + 1] < q->term_offsets[i]) { set_error("query %u: term_offsets must ascend", i); return SSB_E_INVALID; }
            uint32_t n_pos = q->term_offsets[i + 1] - q->term_offsets[i], n_neg = 0;
            if (q->term_flags && !is_device_ptr(q->term_flags))
                for (uint32_t t = q->term_offsets[i]; t < q->term_offsets[i + 1]; t++) if (q->term_flags[t] & SSB_TERM_NOT) { n_neg++; n_pos--; }
            if (n_pos > SSB_MAX_QUERY_TERMS || n_neg > SSB_MAX_NOT_TERMS) {
                set_error("query %u has %u terms + %u NOT terms (max %u + %u per query)", i, n_pos, n_neg, SSB_MAX_QUERY_TERMS, SSB_MAX_NOT_TERMS);
                return SSB_E_UNSUPPORTED;
            }
        }
    }
    if (total_terms && !q->term_keys) { set_error("search_lexical: null term_keys"); return SSB_E_INVALID; }
    if ((uint64_t)nq * (levels_.size() ? levels_.size() : 1) >= 0xFFFFFFFFull) { set_error("batch too large: n_queries * n_levels must be < 2^32"); return SSB_E_UNSUPPORTED; }
    SSB_TRY(ensure_workspace(ws, st, nq, total_terms));
    SSB_CUDA_TRY(to_device(ws.qoff.p, q->term_offsets, ((size_t)nq + 1) * 4, st));
    SSB_CUDA_TRY(to_device(ws.qkeys.p, q->term_keys, (size_t)total_terms * 8, st));
    if (q->term_flags) SSB_CUDA_TRY(to_device(ws.qflags.p, q->term_flags, (size_t)total_terms, st));
    v = view();
    *filtered = false; *geo = false; *fmask_dev = nullptr;
    if (q->filter_offsets) SSB_TRY(stage_filters(ws, st, q, v, filtered, geo));
    if (q->field_masks && n_fields_ > 1) {                   // field_filter: one bitmask of indexed fields per query (host array)
        if (is_device_ptr(q->field_masks)) { set_error("search_lexical: field_masks must be a host array"); return SSB_E_INVALID; }
        SSB_TRY(ws.fmask.reserve(nq, 0, st, true));
        SSB_CUDA_TRY(cudaMemcpyAsync(ws.fmask.p, q->field_masks, (size_t)nq * 4, cudaMemcpyHostToDevice, st));
        *fmask_dev = ws.fmask.p;
    }
    return SSB_OK;
}

int32_t LexIndex::plan_batch(LexWorkspace& ws, cudaStream_t st, const ssb_lex_batch* q, bool topk_only, const SortDev* sort, uint64_t* glist,
                            Batch* b, uint64_t* launches) const {
    if (!committed_) { set_error("search before ssb_lexical_commit"); return SSB_E_STATE; }
    if (!q || (q->n_queries && (!q->term_offsets || !glist))) { set_error("search_lexical: null argument"); return SSB_E_INVALID; }
    if (q->query_type > SSB_QUERY_PHRASE) { set_error("bad query_type"); return SSB_E_INVALID; }
    b->phrase = q->query_type == SSB_QUERY_PHRASE ? 1u : 0u;
    if (b->phrase && has_positions_ != 1) { set_error("phrase query: the index holds no term positions (ssb_level_desc.positions)"); return SSB_E_STATE; }
    if (b->phrase && q->term_flags) { set_error("phrase query: NOT terms are not accepted inside a phrase batch"); return SSB_E_UNSUPPORTED; }
    b->qt_eff = b->phrase ? (uint32_t)SSB_QUERY_INTERSECTION : q->query_type;   // a phrase is an intersection + the position check
    b->nq = q->n_queries;
    if (b->nq == 0) return SSB_OK;
    const uint32_t* fmask_dev = nullptr;
    SSB_TRY(stage_batch(ws, st, q, b->v, &b->filtered, &b->geo, &fmask_dev));
    b->geo = b->geo || (sort && sort_has_point(*sort));
    // a batch with a POINT filter plans without flag bit 1: EVERY filtered query of that batch (its range / set filters too) leaves the
    // lex_score record path for lex_generic<.., GEO>, so that lex_score keeps its code and registers; unfiltered queries stay on it
    const uint32_t topk_flag = topk_only && !b->geo ? 2u : 0u;
    SSB_CUDA_TRY(cudaMemsetAsync(ws.ctr.p, 0, 32, st));
    uint32_t n_pow2 = 2; while (n_pow2 < b->v.n_levels) n_pow2 <<= 1;
    const size_t plan_smem = (size_t)b->v.n_levels * (8 + 2 * FAST_T) + 16 + (size_t)n_pow2 * 8;
    auto plan = sort ? lex_plan<true> : lex_plan<false>;
    if (plan_smem > 48 * 1024) SSB_CUDA_TRY(cudaFuncSetAttribute(plan, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan_smem));
    plan<<<b->nq, 128, plan_smem, st>>>(b->v, ws.qoff.p, ws.qkeys.p, q->term_flags ? ws.qflags.p : nullptr, b->filtered ? ws.foff.p : nullptr, fmask_dev,
                                        b->phrase | topk_flag | (has_ngrams() ? 4u : 0u), b->qt_eff, ws.plans.p, ws.recs.p, ws.item_start.p, ws.ctr.p, ws.theta.p, ws.lock.p,
                                        ws.count.p, glist, n_pow2, ITEM_W, 2, GMAX, sort ? *sort : SortDev{});
    SSB_CUDA_TRY(cudaGetLastError());
    if (launches) *launches += 1;
    return SSB_OK;
}

int32_t LexIndex::search_keys(LexWorkspace& ws, cudaStream_t st, const ssb_lex_batch* q, uint32_t k, uint32_t result_type,
                              uint64_t* keys_out_dev, uint64_t* count_dev, uint64_t* launches, const uint64_t* ceil_dev, const SortDev* sort) const {
    if (k > SSB_K_MAX) { set_error("k=%u exceeds SSB_K_MAX=%u", k, SSB_K_MAX); return SSB_E_UNSUPPORTED; }
    if (result_type > SSB_RESULT_TOPKCOUNT) { set_error("bad result_type"); return SSB_E_INVALID; }
    if (result_type != SSB_RESULT_COUNT && k == 0) result_type = SSB_RESULT_COUNT;   // search.rs:2472-2478
    // keys_out_dev doubles as the per-query global list (32 u64 per query, 32 x 2 sorted); copy_out masks the entries >= k afterwards
    uint64_t* glist = keys_out_dev;
    Batch b;
    SSB_TRY(plan_batch(ws, st, q, result_type == SSB_RESULT_TOPK, sort, glist, &b, launches));
    if (b.nq == 0) return SSB_OK;
    SSB_CUDA_TRY(cudaMemsetAsync(ws.stats.p, 0, sizeof(LexStats), st));   // lex_plan keeps no stats
    const uint32_t nq = b.nq, kk = k ? k : 1;
    const LexView& v = b.v;
    if (ws.ev0) cudaEventRecord(ws.ev0, st);
    const bool need_count = result_type != SSB_RESULT_TOPK;
    // a sorted batch: every query takes lex_generic with 128-bit keys; keys_out_dev is left unmasked (callers read the first k entries)
    if (!sort) {
        if (result_type != SSB_RESULT_COUNT) {
            // batches that carry NOT terms ('-' operator) run their own instantiation: the common kernel stays free of the out-of-line probe
            const bool hn = q->term_flags != nullptr || b.filtered;
            auto score = b.qt_eff == SSB_QUERY_INTERSECTION ? (hn ? lex_score<true, true> : lex_score<true, false>)
                                                            : (hn ? lex_score<false, true> : lex_score<false, false>);
            score<<<n_sms_ * SSB_LEX_MINB, 256, 0, st>>>(v, ws.plans.p, ws.recs.p, ws.item_start.p, nq, kk, ws.ctr.p, ws.theta.p, ws.lock.p, glist, ws.stats.p, ceil_dev);
            SSB_CUDA_TRY(cudaGetLastError());
            if (launches) *launches += 1;
        }
        if (need_count) {
            lex_count<<<n_sms_ * 6, 128, 0, st>>>(v, ws.plans.p, ws.recs.p, ws.item_start.p, nq, b.qt_eff, ws.ctr.p, ws.count.p, ws.stats.p);
            SSB_CUDA_TRY(cudaGetLastError());
            if (launches) *launches += 1;
        }
    }
    // unsorted: queries with 5..16 live terms (the kernel returns at once when the batch has none)
    const bool runs = b.phrase && n_fields_ > 1;
    auto generic = sort ? (runs ? (b.geo ? lex_generic<true, true, true> : lex_generic<true, true>) : (b.geo ? lex_generic<false, true, true> : lex_generic<false, true>))
                        : (runs ? (b.geo ? lex_generic<true, false, true> : lex_generic<true, false>) : (b.geo ? lex_generic<false, false, true> : lex_generic<false, false>));
    generic<<<n_sms_ * 2, 256, 0, st>>>(v, ws.plans.p, ws.recs.p, ws.item_start.p, nq, b.qt_eff, result_type, kk, ws.ctr.p, ws.theta.p, ws.lock.p, ws.count.p, glist,
                                        ws.stats.p, ceil_dev, sort ? *sort : SortDev{});
    SSB_CUDA_TRY(cudaGetLastError());
    if (launches) *launches += 1;
    if (need_count) {     // returns at once unless some query of the batch carries NOT terms
        lex_not_count<<<n_sms_ * 4, 256, 0, st>>>(v, ws.plans.p, nq, b.qt_eff, ws.ctr.p, ws.count.p);
        SSB_CUDA_TRY(cudaGetLastError());
        if (launches) *launches += 1;
        if (v.n_del) {
            const uint64_t pairs = (uint64_t)nq * v.n_del;
            lex_del_count<<<(unsigned)((pairs + 255) / 256), 256, 0, st>>>(v, ws.plans.p, nq, b.qt_eff, ws.count.p);
            SSB_CUDA_TRY(cudaGetLastError());
            if (launches) *launches += 1;
        }
    }
    if (ws.ev1) cudaEventRecord(ws.ev1, st);
    if (sort) {
        if (count_dev) SSB_CUDA_TRY(cudaMemcpyAsync(count_dev, ws.count.p, (size_t)nq * 8, cudaMemcpyDeviceToDevice, st));
        return SSB_OK;
    }
    copy_out<<<(nq * LIST + 255) / 256, 256, 0, st>>>(glist, ws.count.p, nq, result_type == SSB_RESULT_COUNT ? 0 : k, keys_out_dev, count_dev);
    SSB_CUDA_TRY(cudaGetLastError());
    if (launches) *launches += 1;
    return SSB_OK;
}

constexpr size_t FACET_HIST_BYTES = 256ull << 20;   // per search context: the histograms of one query chunk

int32_t LexIndex::facet_counts(LexWorkspace& ws, cudaStream_t st, const ssb_lex_batch* q, const ssb_facet_request* req, uint32_t n_req,
                               const double* bases, ssb_facet_count* out, uint32_t* n_out, uint64_t* launches, uint64_t* kernel_ns,
                               uint64_t* alg_bytes) const {
    if (!q || (n_req && !req) || (q->n_queries && n_req && (!out || !n_out))) { set_error("search_lexical_facets: null argument"); return SSB_E_INVALID; }
    if (n_req > SSB_MAX_FACET_REQUESTS) { set_error("search_lexical_facets: %u requests, at most %u", n_req, SSB_MAX_FACET_REQUESTS); return SSB_E_UNSUPPORTED; }
    // ---- the batch and its plans (Count: every match, no top-k) ----
    SSB_TRY(ws.fglist.reserve((size_t)q->n_queries * LIST, 0, st, true));
    Batch b;
    SSB_TRY(plan_batch(ws, st, q, false, nullptr, ws.fglist.p, &b, launches));
    const uint32_t nq = b.nq;
    if (nq == 0 || n_req == 0) return SSB_OK;
    if (!facets_ || !facets_->n_facets) { set_error("search_lexical_facets: facet counts need ssb_set_facets"); return SSB_E_STATE; }
    if (bases && is_device_ptr(bases)) { set_error("search_lexical_facets: bases must be a host array"); return SSB_E_INVALID; }
    // ---- the requests: keys, and the layout of a query's histogram (range bins, then value bins) and output (request order) ----
    const FacetSet& fs = *facets_;
    std::vector<FacetReqDev> rd(n_req);
    std::vector<uint64_t> starts;
    FacetCall fc{};
    std::vector<uint64_t> csr(2 * (size_t)n_req, 0);                 // per request a StringSet facet's CSR addresses
    bool any_set = false;                                            // a StringSet request: the lex_facets<.., true> instantiation
    uint32_t range_words = 0, n_point = 0; uint64_t value_words = 0, out_stride = 0;
    for (uint32_t i = 0; i < n_req; i++) {
        const uint32_t f = req[i].facet;
        if (f >= fs.n_facets) { set_error("facet request %u: facet %u of %u", i, f, fs.n_facets); return SSB_E_INVALID; }
        const bool set = facet_is_stringset(fs.types[f]);
        const uint64_t max_key = set ? (uint64_t)fs.n_values[f] - 1 : fs.max_key[f];   // a StringSet facet bins its member ids
        if (req[i].kind == SSB_FACET_COUNT_VALUES && req[i].length && (max_key + 1) * 4 > FACET_HIST_BYTES) {
            set_error("facet request %u: %llu value ids, above the %zu MiB facet workspace", i, (unsigned long long)max_key + 1, FACET_HIST_BYTES >> 20);
            return SSB_E_UNSUPPORTED;
        }
        const bool has_order = set ? fs.n_sets[f] != 0 : fs.d_rank[f] && fs.max_key[f] < fs.n_rank[f];
        SSB_TRY(encode_facet_request(req[i], i, fs.types[f], has_order, max_key, bases != nullptr, &rd[i], starts));
        if (set) { csr[2 * i] = (uint64_t)fs.d_set_off[f]; csr[2 * i + 1] = (uint64_t)fs.d_set_mem[f]; any_set = true; }
        if (rd[i].kind != FREQ_VALUES) { rd[i].hist_off = range_words; range_words += rd[i].n_bins; }
        if (rd[i].kind == FREQ_POINT) rd[i].point_idx = n_point++;
        rd[i].out_off = (uint32_t)out_stride;
        out_stride += rd[i].kind == FREQ_VALUES ? rd[i].length : rd[i].n_bins;
    }
    for (uint32_t i = 0; i < n_req; i++)
        if (rd[i].kind == FREQ_VALUES && rd[i].length) { rd[i].hist_off = (uint32_t)(range_words + value_words); value_words += rd[i].n_bins; }
    const uint64_t hist_words = range_words + value_words;
    if (hist_words * 4 > FACET_HIST_BYTES) {
        set_error("search_lexical_facets: one query's histograms take %llu bytes, above the %zu MiB facet workspace", (unsigned long long)hist_words * 4, FACET_HIST_BYTES >> 20);
        return SSB_E_UNSUPPORTED;
    }
    const uint32_t chunk = (uint32_t)std::min<uint64_t>(nq, FACET_HIST_BYTES / 4 / (hist_words ? hist_words : 1));
    SSB_TRY(ws.fhist.reserve(FACET_HIST_BYTES / 4, 0, st, true));
    SSB_TRY(ws.freq.reserve(SSB_MAX_FACET_REQUESTS, 0, st, true));
    SSB_TRY(ws.fstarts.reserve((size_t)SSB_MAX_FACET_REQUESTS * SSB_MAX_FACET_RANGES, 0, st, true));
    SSB_TRY(ws.fstats.reserve(4, 0, st, true));
    SSB_TRY(ws.fcsr.reserve(2 * SSB_MAX_FACET_REQUESTS, 0, st, true));
    SSB_TRY(ws.fout.reserve((size_t)chunk * (out_stride ? out_stride : 1), 0, st, true));
    SSB_TRY(ws.fnout.reserve((size_t)chunk * n_req, 0, st, true));
    SSB_CUDA_TRY(cudaMemcpyAsync(ws.fcsr.p, csr.data(), csr.size() * 8, cudaMemcpyHostToDevice, st));
    SSB_CUDA_TRY(cudaMemcpyAsync(ws.freq.p, rd.data(), n_req * sizeof(FacetReqDev), cudaMemcpyHostToDevice, st));
    if (!starts.empty()) SSB_CUDA_TRY(cudaMemcpyAsync(ws.fstarts.p, starts.data(), starts.size() * 8, cudaMemcpyHostToDevice, st));
    if (n_point) {
        SSB_TRY(ws.fbases.reserve((size_t)nq * n_point * 2, 0, st, true));
        SSB_CUDA_TRY(cudaMemcpyAsync(ws.fbases.p, bases, (size_t)nq * n_point * 16, cudaMemcpyHostToDevice, st));
    }
    SSB_CUDA_TRY(cudaMemsetAsync(ws.fstats.p, 0, 4 * 8, st));
    // ---- per query chunk: the counts, the selection, the copy out ----
    const bool runs = b.phrase && n_fields_ > 1;
    auto kern = any_set ? (runs ? (b.geo ? lex_facets<true, true, true> : lex_facets<true, false, true>) : (b.geo ? lex_facets<false, true, true> : lex_facets<false, false, true>))
                        : (runs ? (b.geo ? lex_facets<true, true, false> : lex_facets<true, false, false>) : (b.geo ? lex_facets<false, true, false> : lex_facets<false, false, false>));
    const size_t smem = starts.size() * 8 + n_req * sizeof(FacetReqDev) + FACET_WARPS * (sizeof(FacetWarpSm) + (size_t)range_words * 4);
    if (smem > 48 * 1024) SSB_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    fc.req = ws.freq.p; fc.n_req = n_req; fc.starts = ws.fstarts.p; fc.n_starts = (uint32_t)starts.size(); fc.bases = ws.fbases.p; fc.n_point = n_point;
    fc.hist = ws.fhist.p; fc.hist_words = (uint32_t)hist_words; fc.range_words = range_words; fc.stats = ws.fstats.p;
    cudaEvent_t e0 = ws.ev0, e1 = ws.ev1;
    float ms_sum = 0.f;
    for (uint32_t q0 = 0; q0 < nq; q0 += chunk) {
        const uint32_t nqc = std::min(chunk, nq - q0);
        SSB_CUDA_TRY(cudaMemsetAsync(ws.fhist.p, 0, (size_t)nqc * hist_words * 4, st));
        if (e0) cudaEventRecord(e0, st);
        kern<<<n_sms_ * 4, FACET_WARPS * 32, smem, st>>>(b.v, ws.plans.p, ws.recs.p, q0, nqc, b.qt_eff, fc, ws.fcsr.p);
        SSB_CUDA_TRY(cudaGetLastError());
        if (e1) cudaEventRecord(e1, st);
        SSB_TRY(launch_facet_select(fs, ws.freq.p, n_req, ws.fhist.p, (uint32_t)hist_words, nqc, ws.fout.p, (uint32_t)out_stride, ws.fnout.p, st));
        if (launches) *launches += 2;
        if (out_stride) SSB_CUDA_TRY(cudaMemcpyAsync(out + (size_t)q0 * out_stride, ws.fout.p, (size_t)nqc * out_stride * sizeof(ssb_facet_count), cudaMemcpyDeviceToHost, st));
        SSB_CUDA_TRY(cudaMemcpyAsync(n_out + (size_t)q0 * n_req, ws.fnout.p, (size_t)nqc * n_req * 4, cudaMemcpyDeviceToHost, st));
        SSB_CUDA_TRY(cudaStreamSynchronize(st));
        float ms = 0.f;
        if (e0 && e1 && cudaEventElapsedTime(&ms, e0, e1) == cudaSuccess) ms_sum += ms; else cudaGetLastError();
    }
    uint64_t fst[4] = {0, 0, 0, 0};
    SSB_CUDA_TRY(cudaMemcpy(fst, ws.fstats.p, 4 * 8, cudaMemcpyDeviceToHost));
    if (kernel_ns) *kernel_ns = (uint64_t)((double)ms_sum * 1e6);
    if (alg_bytes) *alg_bytes = fst[0] * 4 + fst[1] * 8 + fst[2] * n_req * 8 + fst[3];
    return SSB_OK;
}

LexStats LexIndex::read_stats(const LexWorkspace& ws, cudaStream_t st) {
    LexStats s{};
    if (ws.stats.p) { cudaMemcpyAsync(&s, ws.stats.p, sizeof(s), cudaMemcpyDeviceToHost, st); cudaStreamSynchronize(st); }
    return s;
}

}  // namespace ssb
