// vec_ivf.cu — IVF cluster probe of the vector search (AnnMode::Nprobe / Similaritythreshold / NprobeSimilaritythreshold).
//
// Reference (vector.rs:1300-1392): per level the record area is split into clusters (contiguous record ranges, the table in front of
// the level, vector.rs:1066-1094); a cluster's medoid is its first record.  For one query the reference scores the query against the
// medoid of every cluster of the level (:1316-1368), keeps the n_probe best in a TopK (strict `>` replacement = score desc, earlier
// cluster wins ties; medoids scoring below the pre-mapped cluster threshold are rejected, vector.rs:388-399, 421) and then scans only the
// records of the selected clusters (:1395-1467).
//
// Here: the scan kernels are batched — 16 to 256 queries share one pass over the corpus — so the union of the clusters a batch selects is
// (nearly) the whole corpus and skipping bytes is not where the GPU saves time.  The probe is therefore a SELECTION MASK: ivf_score_medoids
// + ivf_select write one bit per (query, cluster), the scans run unchanged and test the bit only where a row is about to become a
// candidate (the rare path, next to the delete-set probe).  A row of an unselected cluster can therefore never enter a list or move a
// threshold: the result is exactly the reference's result for the same AnnMode, recall loss included.
#include "common.cuh"
#include "vec_scan.h"

namespace ssb {
namespace vec {
namespace ivf {

// scores[q][c] of every (query, medoid) pair with the reference's scalar arithmetic: left-to-right sum of individually rounded products
// (dot_f32, vector_similarity.rs:1006-1008) or of squared differences (euclidean, :912-918), so that the cluster ranking is not perturbed
// by a different summation tree.  Block = 32 clusters x 8 queries, 32-dim tiles through shared memory.
template <int SIM>
__global__ void __launch_bounds__(256)
ivf_score_medoids(const float* __restrict__ medoids, uint32_t n_clusters, const float* __restrict__ queries, uint32_t nq, uint32_t dpad,
                  float* __restrict__ scores /*[nq][n_clusters]*/) {
    __shared__ float med[32][33];
    __shared__ float qv[8][32];
    const int tc = threadIdx.x & 31, tq = threadIdx.x >> 5;
    const uint32_t c0 = blockIdx.x * 32, q0 = blockIdx.y * 8;
    float s = 0.0f;
    for (uint32_t d0 = 0; d0 < dpad; d0 += 32) {
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int r = tq * 4 + i;                     // 8 warps x 4 rows = 32 medoids, lane = dim
            med[r][tc] = c0 + r < n_clusters ? medoids[(size_t)(c0 + r) * dpad + d0 + tc] : 0.f;
        }
        qv[tq][tc] = q0 + tq < nq ? queries[(size_t)(q0 + tq) * dpad + d0 + tc] : 0.f;
        __syncthreads();
#pragma unroll
        for (int d = 0; d < 32; d++) {
            if (SIM == SSB_SIM_EUCLIDEAN) { const float df = __fsub_rn(qv[tq][d], med[tc][d]); s = __fadd_rn(s, __fmul_rn(df, df)); }
            else s = __fadd_rn(s, __fmul_rn(qv[tq][d], med[tc][d]));
        }
        __syncthreads();
    }
    if (c0 + tc < n_clusters && q0 + tq < nq) scores[(size_t)(q0 + tq) * n_clusters + c0 + tc] = SIM == SSB_SIM_EUCLIDEAN ? -s : s;
}

// one warp per (level, query): rank the level's clusters, set the bits of the selected ones, add up their vector counts
__global__ void __launch_bounds__(32)
ivf_select(const float* __restrict__ scores, uint32_t n_clusters, const uint32_t* __restrict__ lvl_begin /*[n_levels + 1]*/,
           const uint32_t* __restrict__ cl_count, uint32_t n_probe, int has_thr, float thr,
           uint32_t* __restrict__ sel /*[nq][words]*/, uint32_t words, unsigned long long* __restrict__ observed /*[nq]*/) {
    extern __shared__ uint64_t keys[];
    const int lane = threadIdx.x;
    const uint32_t q = blockIdx.y, b = lvl_begin[blockIdx.x], n = lvl_begin[blockIdx.x + 1] - b;
    const float* sc = scores + (size_t)q * n_clusters + b;
    for (uint32_t i = lane; i < n; i += 32) {
        const float s = sc[i];
        const bool pass = s == s && !(has_thr && s < thr);     // TopK::push rejects score < threshold (vector.rs:421)
        keys[i] = pass ? pack_key(s, i) : 0ull;                   // larger key = better: score desc, cluster id asc
    }
    __syncwarp();
    unsigned long long obs = 0;
    for (uint32_t i = lane; i < n; i += 32) {
        const uint64_t ki = keys[i];
        if (!ki) continue;
        uint32_t rank = 0;
        if (n_probe < n) for (uint32_t j = 0; j < n; j++) rank += keys[j] > ki;
        if (rank < n_probe) {
            atomicOr(&sel[(size_t)q * words + ((b + i) >> 5)], 1u << ((b + i) & 31));
            obs += cl_count[b + i];
        }
    }
    for (int m = 16; m; m >>= 1) obs += __shfl_xor_sync(FULL, obs, m);
    if (lane == 0 && obs) atomicAdd(&observed[q], obs);
}

__global__ void gather_rows(const float* __restrict__ src, const uint32_t* __restrict__ idx, uint32_t n, uint32_t dpad, float* __restrict__ dst) {
    const uint32_t r = blockIdx.x;
    if (r >= n) return;
    for (uint32_t i = threadIdx.x; i < dpad; i += blockDim.x) dst[(size_t)r * dpad + i] = src[(size_t)idx[r] * dpad + i];
}

// out[q][c] = fields of cluster c that query q scans: its mask (0 = every field) if the probe selected c, else none
__global__ void field_sel(const uint32_t* __restrict__ sel, uint32_t sel_words, const uint32_t* __restrict__ fmask, uint32_t n_cl,
                          uint32_t nq, uint32_t* __restrict__ out) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_cl) return;
    for (uint32_t q = blockIdx.y; q < nq; q += gridDim.y) {   // any batch size: the grid's y extent is capped below 65536
        const uint32_t m = fmask[q] ? fmask[q] : 0xFFFFFFFFu;
        const bool on = !sel || ((sel[(size_t)q * sel_words + (c >> 5)] >> (c & 31u)) & 1u);
        out[(size_t)q * n_cl + c] = on ? m : 0u;
    }
}

}  // namespace ivf

int32_t launch_field_sel(const uint32_t* sel, uint32_t sel_words, const uint32_t* fmask, uint32_t nq_pad, uint32_t n_cl, uint32_t* out, cudaStream_t st) {
    if (nq_pad == 0 || n_cl == 0) return SSB_OK;
    ivf::field_sel<<<dim3((n_cl + 127) / 128, nq_pad < 4096u ? nq_pad : 4096u), 128, 0, st>>>(sel, sel_words, fmask, n_cl, nq_pad, out);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

int32_t launch_gather_rows(const float* src, const uint32_t* idx_dev, uint32_t n, uint32_t dpad, float* dst, cudaStream_t st) {
    if (n == 0) return SSB_OK;
    ivf::gather_rows<<<n, 128, 0, st>>>(src, idx_dev, n, dpad, dst);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

int32_t launch_ivf_select(const IvfArgs& a, cudaStream_t st) {
    if (a.nq == 0 || a.n_clusters == 0) return SSB_OK;
    SSB_CUDA_TRY(cudaMemsetAsync(a.sel, 0, (size_t)a.nq_pad * a.words * 4, st));
    SSB_CUDA_TRY(cudaMemsetAsync(a.observed, 0, (size_t)a.nq * 8, st));
    const dim3 g1((a.n_clusters + 31) / 32, (a.nq + 7) / 8);
    if (a.similarity == SSB_SIM_EUCLIDEAN) ivf::ivf_score_medoids<SSB_SIM_EUCLIDEAN><<<g1, 256, 0, st>>>(a.medoids, a.n_clusters, a.queries_padded, a.nq, a.dpad, a.scores);
    else ivf::ivf_score_medoids<SSB_SIM_DOT><<<g1, 256, 0, st>>>(a.medoids, a.n_clusters, a.queries_padded, a.nq, a.dpad, a.scores);
    SSB_CUDA_TRY(cudaGetLastError());
    const uint32_t n_probe = (a.ann_mode == SSB_ANN_NPROBE || a.ann_mode == SSB_ANN_NPROBE_SIMILARITY_THRESHOLD) ? a.n_probe : 0xFFFFFFFFu;
    const int has_thr = a.ann_mode == SSB_ANN_SIMILARITY_THRESHOLD || a.ann_mode == SSB_ANN_NPROBE_SIMILARITY_THRESHOLD;
    const size_t smem = (size_t)a.max_level_clusters * 8;
    if (smem > 200 * 1024) { set_error("IVF probe: a level holds too many clusters (%u)", a.max_level_clusters); return SSB_E_UNSUPPORTED; }
    if (smem > 40 * 1024) SSB_CUDA_TRY(cudaFuncSetAttribute(ivf::ivf_select, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ivf::ivf_select<<<dim3(a.n_levels, a.nq), 32, smem, st>>>(a.scores, a.n_clusters, a.lvl_begin, a.cl_count, n_probe, has_thr, a.cluster_threshold,
                                                             a.sel, a.words, (unsigned long long*)a.observed);
    SSB_CUDA_TRY(cudaGetLastError());
    if (a.launches) *a.launches += 2;
    return SSB_OK;
}

}  // namespace vec
}  // namespace ssb
