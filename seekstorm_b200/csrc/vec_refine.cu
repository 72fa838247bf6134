// vec_refine.cu — second half of the FILTER vector scan (DESIGN.md §3.2c): exact re-scoring of the candidates the fp16 filter
// scan (scan_tc<NQ, PREC_F16F>, vec_scan_tc.cu) kept, and the exact fallback for queries whose candidate set did not fit.
//
// Reference semantics: search_vector_shard scores EVERY record with dot_f32 (vector.rs:1397-1467, vector_similarity.rs:1006-1008,
// 1120-1142) and keeps the k best (TopK, vector.rs:410-497).  The filter scan computes s^ = h(a).h(b) (h = round to fp16) for every record instead and
// guarantees |s - s^| <= eps_q, so the exact top-k is contained in C = {r : s^_r >= (k-th best s^) - 2 eps_q}.  refine_candidates
// evaluates the f32 dot product of the query with the <= 32 rows of C from the f32 corpus — the returned scores are plain f32 dot
// products (closer to the reference's than the 3-product split of the exact tensor-core scan) — and re-sorts under the canonical rule.
// |C| > 32 cannot be represented in the 32-entry list: it shows as "the 32nd entry is still inside the margin"; those queries are
// re-run by fallback_scan, a plain f32 scan (one corpus pass per 4 flagged queries), always enqueued and exiting at once when the
// flag list is empty — no host round trip, so the *_keys entry points stay asynchronous.  Flags are rare by construction: 2 eps_q is
// ~1.2e-3 for unit 768-d vectors (0.03 standard deviations of a random cosine), the candidate set of a top-10 query over 1M x 768
// Gaussian rows holds 10-12 rows; dense near-ties (many copies of one vector) are what the fallback is for.
#include "common.cuh"
#include "vec_scan.h"

namespace ssb {
namespace vec {
namespace rf {

constexpr int RTHREADS = 256;   // refine: 8 warps x 4 candidates
constexpr int RCAND = LIST / (RTHREADS / 32);
constexpr int QF = 4;           // fallback: queries per corpus pass
constexpr int FTHREADS = 256;

__device__ __forceinline__ float dot4(const float4 a, const float4 b, float s) {
    s = fmaf(a.x, b.x, s); s = fmaf(a.y, b.y, s); s = fmaf(a.z, b.z, s); return fmaf(a.w, b.w, s);
}

// one CTA per query.  The approximate list is keys[q] (merged by merge_lists), or, when `lists` is set, the merge of the n_lists per-CTA
// lists a seeded 256-query filter pass leaves in its scratch ([nq_pad / qt][n_lists][qt][32]): merged here, with no launch in between
__global__ void __launch_bounds__(RTHREADS)
refine_candidates(const float* __restrict__ rows, const uint32_t* __restrict__ doc_ids, uint32_t dpad, const float* __restrict__ queries,
                  const float* __restrict__ margin, const uint64_t* keys, const uint64_t* __restrict__ lists, uint32_t n_lists, uint32_t qt,
                  uint64_t* keys_out, uint32_t k, uint32_t* __restrict__ fb_state) {
    __shared__ uint64_t ex[LIST];
    __shared__ MergeSmem msm;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t q = blockIdx.x;
    // approximate keys, descending; low word = 0xFFFFFFFF - row
    const uint64_t mine = lists ? merge_lists_block(lists + (size_t)(q / qt) * n_lists * qt * LIST + (size_t)(q % qt) * LIST, n_lists, (size_t)qt * LIST, msm)
                                : keys[(size_t)q * LIST + lane];
    const float* qv = queries + (size_t)q * dpad;
    uint64_t ck[RCAND]; const float* rp[RCAND]; float s[RCAND];
#pragma unroll
    for (int c = 0; c < RCAND; c++) {
        ck[c] = shfl64(mine, warp * RCAND + c);
        rp[c] = rows + (size_t)(ck[c] ? key_doc(ck[c]) : 0u) * dpad;   // empty slot: row 0, result discarded
        s[c] = 0.f;
    }
    if (ck[0]) {   // lists are dense from the front: nothing to do for this warp when its first slot is empty
        for (uint32_t i = lane * 4; i < dpad; i += 128) {
            const float4 b = *reinterpret_cast<const float4*>(qv + i);
#pragma unroll
            for (int c = 0; c < RCAND; c++) s[c] = dot4(__ldg(reinterpret_cast<const float4*>(rp[c] + i)), b, s[c]);
        }
    }
#pragma unroll
    for (int c = 0; c < RCAND; c++) {
        float v = s[c];
        for (int m = 16; m; m >>= 1) v += __shfl_xor_sync(FULL, v, m);
        if (lane == 0) {
            uint64_t key = 0;
            if (ck[c] && v == v) { const uint32_t row = key_doc(ck[c]); key = pack_key(v, doc_ids ? __ldg(&doc_ids[row]) : row); }
            ex[warp * RCAND + c] = key;
        }
    }
    __syncthreads();
    if (warp == 0) {
        keys_out[(size_t)q * LIST + lane] = wl_sort_desc(ex[lane], lane);   // (every warp read its `keys` before the barrier: aliasing is fine)
        // candidate-set overflow: the list is full and its last entry is still a candidate
        const uint64_t kth = shfl64(mine, (int)k - 1), last = shfl64(mine, LIST - 1);
        if (lane == 0 && last && kth) {
            const float m = margin[q], th = __fsub_rd(key_score(kth), m);
            if (!(m == m) || key_score(last) >= th) fb_state[1 + atomicAdd(&fb_state[0], 1u)] = q;
        }
    }
}

// exact f32 scan for the flagged queries; every CTA exits at once when there are none
__global__ void __launch_bounds__(FTHREADS)
fallback_scan(const float* __restrict__ rows, const uint32_t* __restrict__ doc_ids, uint64_t n_rows, uint32_t dpad,
              const float* __restrict__ queries, const uint32_t* __restrict__ fb_state, uint64_t* __restrict__ fb_lists /*[slot][gridDim.x][32]*/,
              uint32_t k, const uint32_t* __restrict__ del_slot, const uint64_t* __restrict__ del_words,
              const uint32_t* __restrict__ ivf_sel, uint32_t ivf_words, const uint32_t* __restrict__ row_cluster) {
    const uint32_t nf = fb_state[0];
    if (nf == 0) return;
    extern __shared__ __align__(16) float qs[];            // [QF][dpad]
    __shared__ uint64_t sm[FTHREADS / 32][QF][LIST];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (uint32_t base = 0; base < nf; base += QF) {
        for (uint32_t i = threadIdx.x; i < QF * dpad; i += FTHREADS) {
            const uint32_t j = i / dpad;
            qs[i] = base + j < nf ? queries[(size_t)fb_state[1 + base + j] * dpad + (i - j * dpad)] : 0.f;
        }
        __syncthreads();
        uint64_t L[QF];
#pragma unroll
        for (int j = 0; j < QF; j++) L[j] = 0;
        for (uint64_t row = (uint64_t)blockIdx.x * (FTHREADS / 32) + warp; row < n_rows; row += (uint64_t)gridDim.x * (FTHREADS / 32)) {
            float s[QF];
#pragma unroll
            for (int j = 0; j < QF; j++) s[j] = 0.f;
            const float* r = rows + row * dpad;
            for (uint32_t i = lane * 4; i < dpad; i += 128) {
                const float4 a = __ldg(reinterpret_cast<const float4*>(r + i));
#pragma unroll
                for (int j = 0; j < QF; j++) s[j] = dot4(a, *reinterpret_cast<const float4*>(qs + j * dpad + i), s[j]);
            }
#pragma unroll
            for (int j = 0; j < QF; j++) for (int m = 16; m; m >>= 1) s[j] += __shfl_xor_sync(FULL, s[j], m);
            const uint32_t doc = doc_ids ? __ldg(&doc_ids[row]) : (uint32_t)row;
            if (doc_deleted(del_slot, del_words, doc)) continue;
#pragma unroll
            for (int j = 0; j < QF; j++) {
                if (!(s[j] == s[j]) || base + j >= nf) continue;
                if (ivf_skipped(ivf_sel, ivf_words, fb_state[1 + base + j], row_cluster, (uint32_t)row)) continue;
                const uint64_t key = pack_key(s[j], doc);
                if (key > shfl64(L[j], (int)k - 1)) wl_insert(L[j], key, lane);
            }
        }
#pragma unroll
        for (int j = 0; j < QF; j++) sm[warp][j][lane] = L[j];
        __syncthreads();
        if (warp < QF && base + warp < nf) {
            uint64_t M = sm[0][warp][lane];
            for (int w = 1; w < FTHREADS / 32; w++) M = wl_merge(M, sm[w][warp][lane], lane);
            fb_lists[((size_t)(base + warp) * gridDim.x + blockIdx.x) * LIST + lane] = M;
        }
        __syncthreads();
    }
}

// one warp per flagged query: merge the per-CTA lists and replace the query's result list
__global__ void __launch_bounds__(32)
fallback_merge(const uint32_t* __restrict__ fb_state, const uint64_t* __restrict__ fb_lists, uint32_t n_lists, uint64_t* __restrict__ keys) {
    const uint32_t nf = fb_state[0];
    const int lane = threadIdx.x;
    for (uint32_t slot = blockIdx.x; slot < nf; slot += gridDim.x) {
        uint64_t L = 0;
        for (uint32_t l = 0; l < n_lists; l++) {
            const uint64_t B = fb_lists[((size_t)slot * n_lists + l) * LIST + lane];
            if (__any_sync(FULL, B != 0)) L = wl_merge(L, B, lane);
        }
        keys[(size_t)fb_state[1 + slot] * LIST + lane] = L;
    }
}

// one warp per returned (query, doc): the doc's rows in record order, each scored like the scan that produced the hit — f32: the plain
// f32 dot product of refine_candidates (Euclidean: the negated sum of squared differences); int8: the exact int32 dot product through
// the scaled epilogue of scan_tc, so that the winning row's score is the hit's score bit for bit
__global__ void __launch_bounds__(256)
best_rows(BestRowArgs a) {
    const uint32_t h = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (h >= a.n_hits) return;
    const uint4 hit = a.hits[h];
    const uint32_t q = hit.x;
    const uint32_t m = __ldg(&a.field_mask[q]);
    uint32_t best = 0xFFFFFFFFu; float best_s = 0.f;
    for (uint32_t e = hit.y; e < hit.y + hit.z; e++) {
        const uint32_t row = __ldg(&a.doc_rows[e]);
        if (m != 0u && ((m >> __ldg(&a.row_field[row])) & 1u) == 0u) continue;
        float sc;
        if (a.rows_i8) {
            const int* rr = reinterpret_cast<const int*>(a.rows_i8 + (size_t)row * a.dpad8);
            const int* qq = reinterpret_cast<const int*>(a.queries_i8 + (size_t)q * a.dpad8);
            int di = 0;
            for (uint32_t i = lane; i < a.dpad8 / 4; i += 32) di = __dp4a(__ldg(&rr[i]), __ldg(&qq[i]), di);
            for (int o = 16; o; o >>= 1) di += __shfl_xor_sync(FULL, di, o);
            if (!a.i8_scaled) sc = (float)di;
            else {
                if (a.i8_scaled == 3) di = di - a.row_aff[2 * row] * a.q_aff[2 * q + 1] + a.q_aff[2 * q] * a.row_aff[2 * row + 1];
                const float dotf = __fmul_rn(__fmul_rn((float)di, a.q_scale[q]), a.row_scale[row]);
                sc = a.i8_scaled >= 2 ? -fmaxf(__fsub_rn(__fadd_rn(a.q_norm[q], a.row_norm[row]), __fmul_rn(2.0f, dotf)), 0.0f) : dotf;
            }
        } else {
            const float* r = a.rows + (size_t)row * a.dpad;
            const float* qv = a.queries + (size_t)q * a.dpad;
            float s = 0.f;
            for (uint32_t i = lane * 4; i < a.dpad; i += 128) {
                const float4 x = __ldg(reinterpret_cast<const float4*>(r + i)), y = *reinterpret_cast<const float4*>(qv + i);
                if (a.euclid) {
                    const float4 d = make_float4(y.x - x.x, y.y - x.y, y.z - x.z, y.w - x.w);
                    s = dot4(d, d, s);
                } else s = dot4(x, y, s);
            }
            for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(FULL, s, o);
            sc = a.euclid ? -s : s;
        }
        if (sc == sc && (best == 0xFFFFFFFFu || sc > best_s)) { best = row; best_s = sc; }
    }
    if (lane == 0) a.best_row[h] = best;
}

}  // namespace rf

int32_t launch_best_rows(const BestRowArgs& a, cudaStream_t st) {
    if (a.n_hits == 0) return SSB_OK;
    rf::best_rows<<<(a.n_hits + 7) / 8, 256, 0, st>>>(a);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

size_t refine_scratch_words(int n_sms, uint32_t nq_pad) { return (size_t)nq_pad * (size_t)n_sms * LIST + (nq_pad + 2) / 2 + 1; }

int32_t launch_refine(const RefineArgs& a, cudaStream_t st) {
    if (a.nq == 0) return SSB_OK;
    SSB_CUDA_TRY(cudaMemsetAsync(a.fb_state, 0, 4, st));
    rf::refine_candidates<<<a.nq, rf::RTHREADS, 0, st>>>(a.rows, a.doc_ids, a.dpad, a.queries_padded, a.margin, a.keys, a.lists, a.n_lists, a.qt,
                                                         a.keys_out, a.k, a.fb_state);
    SSB_CUDA_TRY(cudaGetLastError());
    const int smem = rf::QF * (int)a.dpad * 4;
    if (smem > 200 * 1024) { set_error("filter scan: vector_dims too large for the fallback scan"); return SSB_E_UNSUPPORTED; }
    if (smem > 40 * 1024) SSB_CUDA_TRY(cudaFuncSetAttribute(rf::fallback_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    rf::fallback_scan<<<a.n_sms, rf::FTHREADS, smem, st>>>(a.rows, a.doc_ids, a.n_rows, a.dpad, a.queries_padded, a.fb_state, a.fb_lists, a.k,
                                                           a.del_slot, a.del_words, a.ivf_sel, a.ivf_words, a.row_cluster);
    SSB_CUDA_TRY(cudaGetLastError());
    rf::fallback_merge<<<64, 32, 0, st>>>(a.fb_state, a.fb_lists, (uint32_t)a.n_sms, a.keys_out);
    SSB_CUDA_TRY(cudaGetLastError());
    if (a.launches) *a.launches += 3;
    return SSB_OK;
}

}  // namespace vec
}  // namespace ssb
