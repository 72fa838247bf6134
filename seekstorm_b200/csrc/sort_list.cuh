// sort_list.cuh — the 128-bit top-k lists of sorted batches: keys {hi, lo} with hi the packed sort key (sort_pack_hi, facets.cuh) and lo a
// pack_key word, warp lists descending like the wl_* helpers of common.cuh, and their merge into a query's global list under its lock.
// Included by bm25.cu (sorted lexical batches) and empty_query.cu (empty-query batches).
#pragma once
#include "common.cuh"

namespace ssb {

// ---- sorted batches: 128-bit top-k keys (hi = packed sort key, lo = pack_key(score, doc)), warp lists descending like wl_* ----
__device__ __forceinline__ bool gt128(uint64_t ah, uint64_t al, uint64_t bh, uint64_t bl) { return ah > bh || (ah == bh && al > bl); }
__device__ __forceinline__ void wl_insert128(uint64_t& Lh, uint64_t& Ll, uint64_t ch, uint64_t cl, int lane) {
    const int pos = __popc(__ballot_sync(FULL, !gt128(ch, cl, Lh, Ll)));   // entries >= cand stay in front
    if (__any_sync(FULL, Lh == ch && Ll == cl)) return;
    const uint64_t uh = shfl64_up1(Lh), ul = shfl64_up1(Ll);
    if (lane == pos) { Lh = ch; Ll = cl; }
    else if (lane > pos) { Lh = uh; Ll = ul; }
}
__device__ __forceinline__ void wl_merge128(uint64_t& Ah, uint64_t& Al, uint64_t Bh, uint64_t Bl, int lane) {
    const uint64_t rh = shfl64(Bh, 31 - lane), rl = shfl64(Bl, 31 - lane);
    if (gt128(rh, rl, Ah, Al)) { Ah = rh; Al = rl; }                   // bitonic, holds the top 32 of the union
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) {
        const uint64_t ph = shfl64_xor(Ah, s), pl = shfl64_xor(Al, s);
        const bool keep_max = (lane & s) == 0;
        if (keep_max == gt128(ph, pl, Ah, Al)) { Ah = ph; Al = pl; }
    }
}
// the warp's list of one sorted item; thr = a lower bound of θ.hi (global θ.hi, or the local list's k-th hi once it is full)
struct SortTop { uint64_t h, l, thr; };
// insert the lanes' candidates (cand) below the paging ceiling (ch, cl) into the warp list; raise thr from the k-th entry
__device__ __forceinline__ void insert_sorted(SortTop& T, bool cand, uint64_t hi, float score, uint32_t doc, bool score_asc,
                                              uint32_t k, int lane, bool& dirty, uint64_t ch, uint64_t cl) {
    const uint64_t lo = pack_key(score, doc) ^ (score_asc ? 0xFFFFFFFF00000000ull : 0ull);
    unsigned m = __ballot_sync(FULL, cand && gt128(ch, cl, hi, lo));
    if (!m) return;
    while (m) {
        const int src = __ffs(m) - 1; m &= m - 1;
        wl_insert128(T.h, T.l, shfl64(hi, src), shfl64(lo, src), lane);
    }
    dirty = true;
    const uint64_t kth = shfl64(T.h, (int)k - 1);
    if (kth > T.thr) T.thr = kth;
}
// merge the warp's list into the query's global list (glist [q][32][2], theta [q][2]) under the per-query lock.  Readers outside the lock
// load θ.hi alone — the pair can tear, θ.hi never decreases — and prune only docs with hi < θ.hi.
__device__ __forceinline__ void publish_sorted(const SortTop& T, uint32_t q, uint32_t k, int lane, uint64_t* theta, int* lock, uint64_t* glist) {
    if (lane == 0) { while (atomicCAS(&lock[q], 0, 1) != 0) __nanosleep(40); }
    __syncwarp();
    __threadfence();
    uint64_t* g = glist + ((size_t)q * LIST + lane) * 2;
    uint64_t Mh = T.h, Ml = T.l;
    wl_merge128(Mh, Ml, __ldcg(&g[0]), __ldcg(&g[1]), lane);
    __stcg(&g[0], Mh); __stcg(&g[1], Ml);
    const uint64_t nh = shfl64(Mh, (int)k - 1), nl = shfl64(Ml, (int)k - 1);
    __threadfence();
    __syncwarp();
    if (lane == 0) {
        if (gt128(nh, nl, __ldcg(&theta[2 * q]), __ldcg(&theta[2 * q + 1]))) { __stcg(&theta[2 * q + 1], nl); __stcg(&theta[2 * q], nh); }
        __threadfence();
        atomicExch(&lock[q], 0);
    }
}

}  // namespace ssb
