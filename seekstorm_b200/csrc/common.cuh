// common.cuh — shared device/host helpers for libseekstorm_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "../../include/seekstorm_b200.h"

namespace ssb {

// ---------------------------------------------------------------- errors
void set_error(const char* fmt, ...);

#define SSB_CUDA_TRY(expr)                                                                   \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            ssb::set_error("%s:%d CUDA error %d (%s) in %s", __FILE__, __LINE__, (int)_e,   \
                           cudaGetErrorString(_e), #expr);                                   \
            return _e == cudaErrorMemoryAllocation ? SSB_E_NOMEM : SSB_E_CUDA;               \
        }                                                                                    \
    } while (0)

#define SSB_TRY(expr)                      \
    do {                                   \
        int32_t _r = (expr);               \
        if (_r != SSB_OK) return _r;       \
    } while (0)

constexpr unsigned FULL = 0xffffffffu;
constexpr int LIST = 32;  // lane-distributed top-k list length (== SSB_K_MAX)

// ---------------------------------------------------------------- packed top-k keys
// key = (ordered(score) << 32) | (0xFFFFFFFF - doc_id); larger key = better under the canonical rule
// (score desc, doc id asc).  0 = empty slot.
__host__ __device__ __forceinline__ uint32_t ord_f32(float s) {
#ifdef __CUDA_ARCH__
    uint32_t u = __float_as_uint(s);
#else
    uint32_t u; memcpy(&u, &s, 4);
#endif
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float unord_f32(uint32_t o) {
    uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}
__host__ __device__ __forceinline__ uint64_t pack_key(float score, uint32_t doc) {
    return ((uint64_t)ord_f32(score) << 32) | (uint64_t)(0xFFFFFFFFu - doc);
}
__host__ __device__ __forceinline__ uint32_t key_doc(uint64_t k) { return 0xFFFFFFFFu - (uint32_t)k; }
__host__ __device__ __forceinline__ float key_score(uint64_t k) { return unord_f32((uint32_t)(k >> 32)); }

#ifdef __CUDACC__
// ---------------------------------------------------------------- warp-distributed sorted list (desc)
__device__ __forceinline__ uint64_t shfl64(uint64_t v, int src) {
    uint32_t lo = __shfl_sync(FULL, (uint32_t)v, src), hi = __shfl_sync(FULL, (uint32_t)(v >> 32), src);
    return ((uint64_t)hi << 32) | lo;
}
__device__ __forceinline__ uint64_t shfl64_up1(uint64_t v) {
    uint32_t lo = __shfl_up_sync(FULL, (uint32_t)v, 1), hi = __shfl_up_sync(FULL, (uint32_t)(v >> 32), 1);
    return ((uint64_t)hi << 32) | lo;
}
__device__ __forceinline__ uint64_t shfl64_xor(uint64_t v, int m) {
    uint32_t lo = __shfl_xor_sync(FULL, (uint32_t)v, m), hi = __shfl_xor_sync(FULL, (uint32_t)(v >> 32), m);
    return ((uint64_t)hi << 32) | lo;
}
// Insert cand (warp-uniform) into the descending list L (lane i holds the i-th largest).
__device__ __forceinline__ void wl_insert(uint64_t& L, uint64_t cand, int lane) {
    unsigned gt = __ballot_sync(FULL, L >= cand);   // >=: an identical key is never inserted twice
    int pos = __popc(gt);
    if (__any_sync(FULL, L == cand)) return;
    uint64_t up = shfl64_up1(L);
    if (lane == pos) L = cand;
    else if (lane > pos) L = up;
}
// Sort 32 keys (one per lane) descending with a shuffle bitonic network (15 compare-exchange steps).
__device__ __forceinline__ uint64_t wl_sort_desc(uint64_t v, int lane) {
#pragma unroll
    for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
            const uint64_t p = shfl64_xor(v, j);
            const bool keep_max = ((lane & k) == 0) == ((lane & j) == 0);
            v = keep_max ? (v > p ? v : p) : (v < p ? v : p);
        }
    }
    return v;
}
// Merge two descending lists -> the 32 largest of their union, descending.
__device__ __forceinline__ uint64_t wl_merge(uint64_t A, uint64_t B, int lane) {
    uint64_t Br = shfl64(B, 31 - lane);
    uint64_t M = A > Br ? A : Br;                  // bitonic, holds the top 32 of the union
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) {
        uint64_t P = shfl64_xor(M, s);
        bool keep_max = (lane & s) == 0;
        M = keep_max ? (M > P ? M : P) : (M < P ? M : P);
    }
    return M;
}

// Block-wide merge of the descending lists of ONE query (256 threads = 8 warps): list l at base[l * stride].  Every warp returns the
// top 32 of their union.  merge_lists (one CTA per query after a scan) and refine_candidates (the lists a seeded 256-query filter pass
// left per CTA) both run it.
constexpr uint32_t MERGE_MAX_LISTS = 2048;   // heads-first path (more lists: plain walk)
struct MergeSmem {
    uint64_t part[8][LIST];                  // per-warp partial merges
    uint16_t ne[MERGE_MAX_LISTS];            // indices of the non-empty lists
    uint32_t n_ne;
};
__device__ __forceinline__ uint64_t merge_lists_block(const uint64_t* __restrict__ base, uint32_t n_lists, size_t stride, MergeSmem& sm) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) sm.n_ne = 0;
    __syncthreads();
    // Phase 1: the lists are sorted best-first, so a list is empty iff its head is 0 — all heads are probed at once (2-3 independent loads
    // per thread for the 592 lists of a tensor-core scan) and only the non-empty lists are fetched in phase 2.  Measured on the 256-query
    // filter batch: 27.9 -> 23.9 us per launch under ncu — a modest gain, because with sample-seeded thresholds nearly every list of a scan
    // still receives 1-3 entries (~k * rows / sample_rows inserts per query in total); exact scans with tight thresholds and the multi-GPU
    // merge profit more.  (A block-wide selection over the first 4 entries of every list would be the next step.)
    const bool small = n_lists <= MERGE_MAX_LISTS;
    if (small) {
        for (uint32_t l = threadIdx.x; l < n_lists; l += 256)
            if (__ldg(&base[(size_t)l * stride]) != 0ull) sm.ne[atomicAdd(&sm.n_ne, 1u)] = (uint16_t)l;
        __syncthreads();
    }
    const uint32_t cnt = small ? sm.n_ne : n_lists;
    uint64_t L = 0;
    // Phase 2: four independent loads in flight per warp; the merge order does not matter (the result is the top 32 of the union)
    for (uint32_t i = warp; i < cnt; i += 32) {
        uint64_t B[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const uint32_t k = i + 8 * u;
            B[u] = k < cnt ? __ldg(&base[(size_t)(small ? (uint32_t)sm.ne[k] : k) * stride + lane]) : 0ull;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) if (__any_sync(FULL, B[u] != 0)) L = wl_merge(L, B[u], lane);
    }
    sm.part[warp][lane] = L;
    __syncthreads();
    L = sm.part[0][lane];
    for (int w = 1; w < 8; w++) L = wl_merge(L, sm.part[w][lane], lane);
    return L;
}

// delete set probe (shard.delete_hashset, vector.rs:1450-1451 / add_result.rs:3435): level table + one bitmap word; only on the
// rare candidate-insert paths
__device__ __forceinline__ bool doc_deleted(const uint32_t* __restrict__ del_slot, const uint64_t* __restrict__ del_words, uint32_t doc) {
    if (!del_slot) return false;
    const uint32_t slot = __ldg(&del_slot[doc >> 16]);
    if (slot == 0xFFFFFFFFu) return false;
    return ((__ldg(&del_words[(size_t)slot * 1024 + ((doc & 0xFFFFu) >> 6)]) >> (doc & 63u)) & 1ull) != 0;
}

// IVF probe (vec_ivf.cu): is the row's cluster NOT selected for this query?  sel = [nq][words] bit per (query, cluster), null = AnnMode::All
__device__ __forceinline__ bool ivf_skipped(const uint32_t* __restrict__ sel, uint32_t words, uint32_t q, const uint32_t* __restrict__ row_cluster, uint32_t row) {
    if (!sel) return false;
    const uint32_t c = __ldg(&row_cluster[row]);
    return ((__ldg(&sel[(size_t)q * words + (c >> 5)]) >> (c & 31u)) & 1u) == 0u;
}

// ---------------------------------------------------------------- PTX: mbarrier + TMA
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra.uni WAIT_DONE;\n"
        "bra.uni WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// 2-D tiled TMA load: box -> smem, completion on mbarrier (complete_tx::bytes)
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
#endif  // __CUDACC__

// host: encode a 2-D row-major f32 tensor map (cuTensorMapEncodeTiled resolved at runtime, no libcuda link)
// generic 2-D row-major tensor map: elem_bytes 4 (f32) or 2 (bf16); swizzle_bytes 0 / 64 / 128
int32_t encode_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes, uint64_t inner_elems, uint64_t rows,
                       uint64_t row_pitch_bytes, uint32_t box_inner, uint32_t box_rows, int swizzle_bytes);
int32_t encode_tmap_2d_f32(CUtensorMap* out, const void* base, uint64_t inner_elems, uint64_t rows,
                           uint64_t row_pitch_bytes, uint32_t box_inner, uint32_t box_rows, int swizzle128);

}  // namespace ssb
