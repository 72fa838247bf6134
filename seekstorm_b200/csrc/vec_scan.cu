// vec_scan.cu — brute-force f32 vector scan with fused top-k (sm_90a).
//
// Replaces the record loop of search_vector_shard (vector.rs:1397-1467): for every record,
// similarity = dot_f32 / -euclidean_f32 (vector_similarity.rs:1006-1008, 912-918, 1120-1142) and
// TopK::push (vector.rs:410-497), for a batch of queries per corpus pass.
//
// Layout: corpus = row-major f32 [n_rows, Dpad] (Dpad = dims rounded up to 32, zero padded), no AoS
// header (the reference's 24-byte VectorHeader + embedding record, vector.rs:62-73, is split at load:
// doc ids live in a separate u32 array).  HBM-bound: algorithmic bytes per pass = n_rows*dims*4.
//
// Kernel scan_ffma: persistent CTAs (one per SM), 8 consumer warps + 1 TMA producer warp.
//   producer: cp.async.bulk.tensor.2d of two [256 rows x 32 floats] corpus boxes (SWIZZLE_128B, 64 KB) and
//             the [16 queries x 32 floats] query box into a 3-stage mbarrier ring.
//   consumers: warp w owns rows (w>>1)*128 + lane + 32*{0..3} of the tile and queries (w&1)*8..+8
//             (4 x 8 register tile per lane): FP32 FFMA accumulation (even-k / odd-k pairs) over the k-chunks
//             (conflict-free swizzled LDS.128 for rows, broadcast LDS.128 for queries; the 4x8 tile
//             keeps shared-memory wavefronts at ~55 % of the HBM-time budget), then a warp-shuffle
//             top-k insert per finished tile.
//   per-warp lists -> scratch; merge_lists kernel reduces them to the final per-query top-k.
#include <limits.h>
#include "common.cuh"
#include "vec_scan.h"

namespace ssb {
namespace vec {

constexpr int KC = 32;                  // floats per k-chunk (128 B = one swizzle row)
constexpr int TILE_ROWS = 512;          // rows per pipeline stage (two 256-row TMA boxes)
constexpr int BOX_ROWS = 256;
constexpr int QT = (int)queries_per_pass(Scan::Ffma);   // queries per pass (16)
constexpr int STAGES = 3;
constexpr int CWARPS = 8;
constexpr int THREADS = (CWARPS + 1) * 32;
constexpr int A_BYTES = TILE_ROWS * KC * 4;  // 64 KB
constexpr int Q_BYTES = QT * KC * 4;         // 2 KB
constexpr int STAGE_TX = A_BYTES + Q_BYTES;
constexpr int LISTS_BYTES = CWARPS * 8 * LIST * 8;   // per-warp top-k lists (8 queries x 32 keys) live in smem
constexpr int SMEM_BYTES = STAGES * (A_BYTES + Q_BYTES) + LISTS_BYTES + 2 * STAGES * 8;

// pairs of FP32 lanes (even-k / odd-k partial sums): Hopper has no packed FP32x2 instructions, so each pair is two scalar
// round-to-nearest operations (the same rounding per component)
__device__ __forceinline__ void ffma2(float2& c, float2 a, float2 b) {
    c.x = __fmaf_rn(a.x, b.x, c.x);
    c.y = __fmaf_rn(a.y, b.y, c.y);
}
__device__ __forceinline__ float2 fsub2(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }


template <int SIM>
__global__ void __launch_bounds__(THREADS, 1)
scan_ffma(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmQ,
          uint32_t n_rows, uint32_t n_kchunks, uint32_t n_tiles, uint32_t k,
          const uint32_t* __restrict__ doc_ids, uint64_t* __restrict__ scratch /*[gridDim.y][gridDim.x*CWARPS/2][QT][32]*/,
          const uint32_t* __restrict__ thr_init /*[gridDim.y*QT] or null*/, uint32_t nq_valid,
          const uint64_t* __restrict__ ceil_keys /*[gridDim.y*QT] or null*/,
          const uint32_t* __restrict__ del_slot, const uint64_t* __restrict__ del_words,
          const uint32_t* __restrict__ ivf_sel, uint32_t ivf_words, const uint32_t* __restrict__ row_cluster /*IVF selection mask or null*/,
          uint32_t sample_mode /* 1: threshold-seeding pass — keep the row-group score maxima, no lists */) {
    // no static shared memory in this kernel: the dynamic segment starts at offset 0 of the CTA window, so the
    // 1024-byte alignment SWIZZLE_128B needs holds and the pointers stay in the shared address space (LDS, not LD)
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* sA = smem;                                  // [STAGES][A_BYTES]
    uint8_t* sQ = smem + STAGES * A_BYTES;               // [STAGES][Q_BYTES]
    uint64_t* sL = (uint64_t*)(sQ + STAGES * Q_BYTES);   // [CWARPS][8][32] (9 warps -> one SMSP hosts 3: 168 regs/thread max)
    uint64_t* full = sL + CWARPS * 8 * LIST;             // [STAGES]
    uint64_t* empty = full + STAGES;                     // [STAGES]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t group = blockIdx.y;                   // which block of QT queries

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], CWARPS); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == CWARPS) {
        // ===== TMA producer =====
        if (lane == 0) {
            tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmQ);
            uint32_t it = 0;
            for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                for (uint32_t kc = 0; kc < n_kchunks; ++kc, ++it) {
                    uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
                    mbar_wait(&empty[s], ph ^ 1u);
                    mbar_arrive_expect_tx(&full[s], STAGE_TX);
                    tma_load_2d(sA + s * A_BYTES, &tmA, (int)(kc * KC), (int)(tile * TILE_ROWS), &full[s]);
                    tma_load_2d(sA + s * A_BYTES + BOX_ROWS * KC * 4, &tmA, (int)(kc * KC), (int)(tile * TILE_ROWS + BOX_ROWS), &full[s]);
                    tma_load_2d(sQ + s * Q_BYTES, &tmQ, (int)(kc * KC), (int)(group * QT), &full[s]);
                }
            }
        }
    } else {
        // ===== consumers: warp = (row group of 128 rows) x (query half); lane owns 4 rows x 8 queries =====
        const int rg = warp >> 1;            // row group 0..3
        const int qh = (warp & 1) * 8;       // first query of this warp's half
        const int r0 = rg * 128 + lane;      // rows r0 + 32*j, j = 0..3; all share (row & 7)
        const int sw = r0 & 7;
        float2 acc[4][8];                    // even-k / odd-k partial sums
        uint64_t* myL = sL + (size_t)warp * 8 * LIST + lane;   // myL[q * LIST]
        uint32_t thr[8];
#pragma unroll
        for (int q = 0; q < 8; q++) {
            myL[q * LIST] = 0;
            // zero-padded query slots score 0 on every row: give them an unreachable threshold so they never insert
            thr[q] = group * QT + qh + q >= nq_valid ? 0xFFFFFFFFu : (thr_init ? __ldg(&thr_init[group * QT + qh + q]) : 0u);
#pragma unroll
            for (int j = 0; j < 4; j++) acc[j][q] = make_float2(0.f, 0.f);
        }

        uint32_t it = 0;
        for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            for (uint32_t kc = 0; kc < n_kchunks; ++kc, ++it) {
                uint32_t s = it % STAGES, ph = (it / STAGES) & 1u;
                mbar_wait(&full[s], ph);
                const float4* A = (const float4*)(sA + s * A_BYTES);
                const float4* Q = (const float4*)(sQ + s * Q_BYTES);
#pragma unroll
                for (int kk = 0; kk < 8; kk++) {
                    float4 a[4];
#pragma unroll
                    for (int j = 0; j < 4; j++) a[j] = A[(r0 + 32 * j) * 8 + (kk ^ sw)];
#pragma unroll
                    for (int q = 0; q < 8; q++) {
                        const float4 qv = Q[(qh + q) * 8 + kk];
#pragma unroll
                        for (int j = 0; j < 4; j++) {
                            if (SIM == SSB_SIM_EUCLIDEAN) {
                                float2 d0 = fsub2(make_float2(qv.x, qv.y), make_float2(a[j].x, a[j].y));
                                float2 d1 = fsub2(make_float2(qv.z, qv.w), make_float2(a[j].z, a[j].w));
                                ffma2(acc[j][q], d0, d0);
                                ffma2(acc[j][q], d1, d1);
                            } else {
                                ffma2(acc[j][q], make_float2(a[j].x, a[j].y), make_float2(qv.x, qv.y));
                                ffma2(acc[j][q], make_float2(a[j].z, a[j].w), make_float2(qv.z, qv.w));
                            }
                        }
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[s]);

                if (kc + 1 == n_kchunks && sample_mode) {
                    // sample mode: lane (j*8 + q) keeps the best ordered-uint score of row group j (32 rows) for query q
                    uint32_t keep = 0;
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const uint32_t row = tile * TILE_ROWS + (uint32_t)r0 + 32u * j;
                        const bool valid = row < n_rows;
#pragma unroll
                        for (int q = 0; q < 8; q++) {
                            const float sum = acc[j][q].x + acc[j][q].y;
                            const float sc = (SIM == SSB_SIM_EUCLIDEAN) ? -sum : sum;
                            acc[j][q] = make_float2(0.f, 0.f);
                            uint32_t so = (valid && sc == sc) ? ord_f32(sc) : 0u;
                            if (ceil_keys && so) {
                                const uint64_t key = ((uint64_t)so << 32) | (uint64_t)(0xFFFFFFFFu - (doc_ids ? __ldg(&doc_ids[row]) : row));
                                if (key >= __ldg(&ceil_keys[group * QT + qh + q])) so = 0u;
                            }
                            const uint32_t mx = __reduce_max_sync(FULL, so);
                            if (lane == j * 8 + q) keep = mx;
                        }
                    }
                    uint32_t* gmax = (uint32_t*)scratch;               // [gridDim.y * QT][n_tiles * 16]
                    gmax[(size_t)(group * QT + qh + (lane & 7)) * (n_tiles * 16) + (tile * 16 + rg * 4 + (lane >> 3))] = keep;
                    continue;
                }
                if (kc + 1 == n_kchunks) {
                    // ---- tile finished: fused top-k (TopK::push, vector.rs:410-497) ----
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        uint32_t row = tile * TILE_ROWS + (uint32_t)r0 + 32u * j;
                        bool valid = row < n_rows;
#pragma unroll
                        for (int q = 0; q < 8; q++) {
                            float sum = acc[j][q].x + acc[j][q].y;
                            float sc = (SIM == SSB_SIM_EUCLIDEAN) ? -sum : sum;
                            acc[j][q] = make_float2(0.f, 0.f);
                            uint32_t so = ord_f32(sc);
                            unsigned m = __ballot_sync(FULL, valid && so >= thr[q] && sc == sc);
                            if (m) {                                   // rare after warm-up
                                // paging: keys >= ceil were returned by an earlier page (0 = this query is exhausted)
                                const uint64_t ceil = ceil_keys ? __ldg(&ceil_keys[group * QT + qh + q]) : ~0ull;
                                uint64_t Lq = myL[q * LIST];
                                while (m) {
                                    int src = __ffs(m) - 1;
                                    m &= m - 1;
                                    uint32_t so_s = __shfl_sync(FULL, so, src);
                                    uint32_t row_s = __shfl_sync(FULL, row, src);
                                    uint32_t doc = doc_ids ? __ldg(&doc_ids[row_s]) : row_s;
                                    uint64_t key = ((uint64_t)so_s << 32) | (uint64_t)(0xFFFFFFFFu - doc);
                                    if (key < ceil && !doc_deleted(del_slot, del_words, doc) && !ivf_skipped(ivf_sel, ivf_words, group * QT + qh + q, row_cluster, row_s))
                                        wl_insert(Lq, key, lane);
                                }
                                myL[q * LIST] = Lq;
                                const uint32_t kth = (uint32_t)(shfl64(Lq, (int)k - 1) >> 32);
                                if (kth > thr[q]) thr[q] = kth;
                            }
                        }
                    }
                }
            }
        }
        // ---- publish the warp's lists: scratch[group][list][q][lane], list = (cta*4 + rg) ----
        if (sample_mode) return;                          // scratch holds the group maxima, not lists
        const uint32_t n_lists = gridDim.x * (CWARPS / 2);
        uint64_t* out = scratch + ((size_t)group * n_lists + (size_t)blockIdx.x * (CWARPS / 2) + rg) * QT * LIST;
#pragma unroll
        for (int q = 0; q < 8; q++) out[(qh + q) * LIST + lane] = myL[q * LIST];
    }
}

// Merge `n_lists` descending 32-lists per query into one.  in: [n_groups][n_lists][qt][32] when
// qt_major==0 ... generic form: list l of query q lives at in[(q / qt) * n_lists * qt * 32 + l * qt * 32 + (q % qt) * 32].
__global__ void __launch_bounds__(256)
merge_lists(const uint64_t* __restrict__ in, uint32_t n_lists, uint32_t qt, uint64_t* __restrict__ out /*[nq][32]*/) {
    __shared__ MergeSmem sm;
    const uint32_t q = blockIdx.x;
    const uint64_t L = merge_lists_block(in + (size_t)(q / qt) * n_lists * qt * LIST + (size_t)(q % qt) * LIST, n_lists, (size_t)qt * LIST, sm);
    if (threadIdx.x < 32) out[(size_t)q * LIST + threadIdx.x] = L;
}

// queries [nq][dims] (row stride qstride) -> padded [nq_pad][dpad], optionally L2-normalised
// (normalize_f32, vector_similarity.rs:70-74; applied to the query at search.rs:1464-1475).
__global__ void prep_queries(const float* __restrict__ q, uint32_t nq, uint32_t dims, uint64_t qstride,
                             float* __restrict__ out, uint32_t nq_pad, uint32_t dpad, int normalize) {
    const int lane = threadIdx.x & 31;
    uint32_t row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= nq_pad) return;
    float* o = out + (size_t)row * dpad;
    if (row >= nq) { for (uint32_t i = lane; i < dpad; i += 32) o[i] = 0.f; return; }
    const float* src = q + (size_t)row * qstride;
    float f = 1.f;
    if (normalize) {
        float s = 0.f;
        for (uint32_t i = lane; i < dims; i += 32) { float v = src[i]; s = fmaf(v, v, s); }
        for (int m = 16; m; m >>= 1) s += __shfl_xor_sync(FULL, s, m);
        f = 1.0f / sqrtf(s);
    }
    for (uint32_t i = lane; i < dpad; i += 32) o[i] = i < dims ? src[i] * f : 0.f;
}

// corpus rows in place: [n][dpad]; normalise first `dims` entries (vector.rs:585-596), zero the padding
__global__ void normalize_rows(float* __restrict__ rows, uint64_t n, uint32_t dims, uint32_t dpad, int normalize) {
    const int lane = threadIdx.x & 31;
    uint64_t row = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n) return;
    float* r = rows + row * dpad;
    float f = 1.f;
    if (normalize) {
        float s = 0.f;
        for (uint32_t i = lane; i < dims; i += 32) { float v = r[i]; s = fmaf(v, v, s); }
        for (int m = 16; m; m >>= 1) s += __shfl_xor_sync(FULL, s, m);
        f = 1.0f / sqrtf(s);
    }
    for (uint32_t i = lane; i < dpad; i += 32) r[i] = i < dims ? r[i] * f : 0.f;
}

// Cosine + ScalarQuantizationI8: normalize_f32 (vector_similarity.rs:70-74) then quantize_f32_to_i8 (:1226-1232), done
// at index time for the corpus (vector.rs:585-640) and per query.  One warp per row.  The squared norm is accumulated
// strictly left to right with individually rounded multiplies / adds (the reference's scalar `.map(|x| x*x).sum()`), so
// the int8 codes — and with them every int32 dot product — are bit-identical to the CPU's: the sequential chain runs
// redundantly in all lanes over shuffled products.
__global__ void quantize_rows_i8(const float* __restrict__ src, uint64_t src_stride, uint64_t n, uint64_t n_out, uint32_t dims,
                                 int8_t* __restrict__ dst, uint32_t dpad8) {
    const int lane = threadIdx.x & 31;
    const uint64_t row = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_out) return;
    int8_t* o = dst + row * dpad8;
    if (row >= n) { for (uint32_t i = lane; i < dpad8; i += 32) o[i] = 0; return; }
    const float* r = src + row * src_stride;
    float s = 0.0f;
    for (uint32_t base = 0; base < dims; base += 32) {
        const float v = base + lane < dims ? r[base + lane] : 0.0f;
        const float p = __fmul_rn(v, v);
#pragma unroll
        for (int l = 0; l < 32; l++) s = __fadd_rn(s, __shfl_sync(FULL, p, l));   // out-of-range products are +0: exact no-ops
    }
    const float f = __fdiv_rn(1.0f, __fsqrt_rn(s));
    for (uint32_t i = lane; i < dpad8; i += 32) {
        int8_t q = 0;
        if (i < dims) {
            float x = roundf(__fmul_rn(__fmul_rn(r[i], f), 127.0f));    // Rust f32::round: half away from zero
            x = fminf(fmaxf(x, -127.0f), 127.0f);
            q = x == x ? (int8_t)x : (int8_t)0;                          // NaN (all-zero vector) `as i8` = 0
        }
        o[i] = q;
    }
}

// Dot / Euclidean + ScalarQuantizationI8: QuantizedVector::new_scale / new_scale_norm (vector_similarity.rs:1340-1371).  One warp per row.
__global__ void quantize_rows_scale_i8(const float* __restrict__ src, uint64_t src_stride, uint64_t n, uint64_t n_out, uint32_t dims,
                                       int8_t* __restrict__ dst, uint32_t dpad8, float* __restrict__ scale_out, float* __restrict__ norm_out, int want_norm) {
    const int lane = threadIdx.x & 31;
    const uint64_t row = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_out) return;
    int8_t* o = dst + row * dpad8;
    if (row >= n) { for (uint32_t i = lane; i < dpad8; i += 32) o[i] = 0; if (lane == 0) { scale_out[row] = 0.f; if (norm_out) norm_out[row] = 0.f; } return; }
    const float* r = src + row * src_stride;
    float mx = 0.0f;                                            // values.iter().map(|x| x.abs()).fold(0.0, f32::max): NaN is ignored by f32::max
    for (uint32_t i = lane; i < dims; i += 32) mx = fmaxf(mx, fabsf(r[i]));
    for (int m = 16; m; m >>= 1) mx = fmaxf(mx, __shfl_xor_sync(FULL, mx, m));
    const float scale = __fdiv_rn(mx, 127.0f);
    int sum = 0;
    for (uint32_t i = lane; i < dpad8; i += 32) {
        int8_t q = 0;
        if (i < dims) {
            float x = roundf(__fdiv_rn(r[i], scale));         // Rust f32::round: half away from zero; `as i8` saturates, NaN -> 0
            x = fminf(fmaxf(x, -128.0f), 127.0f);
            q = x == x ? (int8_t)x : (int8_t)0;
        }
        o[i] = q;
        sum += (int)q * (int)q;
    }
    for (int m = 16; m; m >>= 1) sum += __shfl_xor_sync(FULL, sum, m);
    if (lane == 0) {
        scale_out[row] = scale;
        if (norm_out) norm_out[row] = want_norm ? __fmul_rn(__fmul_rn((float)sum, scale), scale) : 0.0f;
    }
}

// ---- affine Euclidean SQ (QuantizedVector::new_scale_norm_affine, vector_similarity.rs:1414-1463; raster_range :1465-1472) ----
// raster_range: a range above 1.0 is widened to 2^m - 1 ((range as i64 as u64 + 1).next_power_of_two() - 1), smaller ranges stay
__host__ __device__ inline float ssb_raster_range(float range) {
    if (!(range > 1.0f)) return range;
    unsigned long long v = (unsigned long long)(long long)range + 1ull, p = 1ull;   // `as i64` truncates towards zero
    while (p < v) p <<= 1;
    return (float)(p - 1ull);
}
// one step of the reference's running state: (min_val, max_val) of the vector -> the (min, max) it is quantised with; state updated in place
__host__ __device__ inline void ssb_affine_step(float& st_min, float& st_max, float& mn, float& mx) {
    if (mn < st_min) st_min = mn; else mn = st_min;
    if (mx > st_max) st_max = ssb_raster_range(mx - mn); else mx = st_max;
}
__global__ void rows_minmax(const float* __restrict__ src, uint64_t src_stride, uint64_t n, uint32_t dims, float2* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const uint64_t row = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n) return;
    const float* r = src + row * src_stride;
    float mn = INFINITY, mx = -INFINITY;                       // fold((INF, -INF), (min, max)): f32::min / max ignore NaN like fminf / fmaxf
    for (uint32_t i = lane; i < dims; i += 32) { mn = fminf(mn, r[i]); mx = fmaxf(mx, r[i]); }
    for (int m = 16; m; m >>= 1) { mn = fminf(mn, __shfl_xor_sync(FULL, mn, m)); mx = fmaxf(mx, __shfl_xor_sync(FULL, mx, m)); }
    if (lane == 0) out[row] = make_float2(mn, mx);
}
__global__ void quantize_rows_affine_i8(const float* __restrict__ src, uint64_t src_stride, uint64_t n, uint64_t n_out, uint32_t dims,
                                        const float* __restrict__ scale_in, const int* __restrict__ zp_in, float st_min, float st_max,
                                        int8_t* __restrict__ dst, uint32_t dpad8, float* __restrict__ scale_out, float* __restrict__ norm_out,
                                        int2* __restrict__ aff_out, int is_query) {
    const int lane = threadIdx.x & 31;
    const uint64_t row = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_out) return;
    int8_t* o = dst + row * dpad8;
    if (row >= n) {
        for (uint32_t i = lane; i < dpad8; i += 32) o[i] = 0;
        if (lane == 0) { scale_out[row] = 0.f; norm_out[row] = 0.f; aff_out[row] = make_int2(0, 0); }
        return;
    }
    const float* r = src + row * src_stride;
    float scale; int zp;
    if (scale_in) { scale = __ldg(&scale_in[row]); zp = __ldg(&zp_in[row]); }
    else {
        float mn = INFINITY, mx = -INFINITY;
        for (uint32_t i = lane; i < dims; i += 32) { mn = fminf(mn, r[i]); mx = fmaxf(mx, r[i]); }
        for (int m = 16; m; m >>= 1) { mn = fminf(mn, __shfl_xor_sync(FULL, mn, m)); mx = fmaxf(mx, __shfl_xor_sync(FULL, mx, m)); }
        float a = st_min, b = st_max;
        ssb_affine_step(a, b, mn, mx);
        scale = __fdiv_rn(ssb_raster_range(__fsub_rn(mx, mn)), 255.0f);
        float z = roundf(__fsub_rn(-128.0f, __fdiv_rn(mn, scale)));
        z = fminf(fmaxf(z, -128.0f), 127.0f);
        zp = z == z ? (int)z : 0;
    }
    int sq = 0, sum = 0;
    for (uint32_t i = lane; i < dpad8; i += 32) {
        int8_t q = 0;
        if (i < dims) {
            const float x = roundf(__fdiv_rn(r[i], scale));      // (x / scale).round() as i32: saturating, NaN -> 0
            int xi = x != x ? 0 : (x >= 2147483648.0f ? INT_MAX : (x <= -2147483648.0f ? INT_MIN : (int)x));
            long long s = (long long)xi + zp;
            q = (int8_t)(s < -128 ? -128 : (s > 127 ? 127 : s));
        }
        o[i] = q;
        sq += (int)q * (int)q; sum += (int)q;
    }
    for (int m = 16; m; m >>= 1) { sq += __shfl_xor_sync(FULL, sq, m); sum += __shfl_xor_sync(FULL, sum, m); }
    if (lane == 0) {
        const int norm_i = sq - 2 * zp * sum + (int)dims * zp * zp;
        scale_out[row] = scale;
        norm_out[row] = __fmul_rn(__fmul_rn((float)norm_i, scale), scale);
        aff_out[row] = is_query ? make_int2(zp, sum) : make_int2(zp, (int)dims * zp - sum);
    }
}

// TurboQuantI8 (TurboQuant::quantize_f32_i8, vector_similarity.rs:1929-1958): zero-pad the vector to tq_dim (a power of two), flip signs
// by the index's seed mask, rotate with the normalised fast Walsh-Hadamard transform (fwht :1861-1880: butterflies h = 1, 2, 4, ..., then
// every element / sqrt(n)), scale = max(sigma / 32, 1e-8) with sigma = ||x|| / sqrt(dim) (calculate_scale :2035-2039), codes =
// round(x / scale) clamped to [-127, 127], norm = (sum of code^2) * scale * scale.  Cosine indexes normalise first (normalize_f32, vector.rs:585-596).
// One CTA per row, the vector in shared memory.  Butterflies are element-wise (any schedule gives the same bits); the two sums of squares
// are left-to-right chains of individually rounded products like the scalar reference, run by one thread.  negate: store -scale
// (the reference's Dot / Cosine score is -(dot * s1 * s2): negating ONE scale gives exactly that through the scaled int8 epilogue).
__global__ void __launch_bounds__(256) quantize_rows_turbo_i8(const float* __restrict__ src, uint64_t src_stride, uint64_t n, uint32_t dims, uint32_t tq_dim,
                                                              const float* __restrict__ mask, int8_t* __restrict__ dst, uint32_t dpad8,
                                                              float* __restrict__ scale_out, float* __restrict__ norm_out, int normalize, int negate) {
    extern __shared__ float a[];                                  // [tq_dim]
    __shared__ float s_val; __shared__ int s_sq;
    const uint64_t row = blockIdx.x;
    int8_t* o = dst + row * dpad8;
    if (row >= n) { for (uint32_t i = threadIdx.x; i < dpad8; i += blockDim.x) o[i] = 0; if (threadIdx.x == 0) { scale_out[row] = 0.f; norm_out[row] = 0.f; } return; }
    const float* r = src + row * src_stride;
    for (uint32_t i = threadIdx.x; i < tq_dim; i += blockDim.x) a[i] = i < dims ? r[i] : 0.0f;
    if (threadIdx.x == 0) s_sq = 0;
    __syncthreads();
    if (normalize) {
        if (threadIdx.x == 0) { float s = 0.0f; for (uint32_t i = 0; i < dims; i++) s = __fadd_rn(s, __fmul_rn(a[i], a[i])); s_val = __fdiv_rn(1.0f, __fsqrt_rn(s)); }
        __syncthreads();
        const float f = s_val;
        for (uint32_t i = threadIdx.x; i < dims; i += blockDim.x) a[i] = __fmul_rn(a[i], f);
        __syncthreads();
    }
    for (uint32_t i = threadIdx.x; i < tq_dim; i += blockDim.x) a[i] = __fmul_rn(a[i], __ldg(&mask[i]));
    __syncthreads();
    for (uint32_t h = 1; h < tq_dim; h <<= 1) {
        for (uint32_t p = threadIdx.x; p < tq_dim / 2; p += blockDim.x) {
            const uint32_t j = (p / h) * 2u * h + (p % h);
            const float x = a[j], y = a[j + h];
            a[j] = __fadd_rn(x, y); a[j + h] = __fsub_rn(x, y);
        }
        __syncthreads();
    }
    const float nrm = __fsqrt_rn((float)tq_dim);
    for (uint32_t i = threadIdx.x; i < tq_dim; i += blockDim.x) a[i] = __fdiv_rn(a[i], nrm);
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.0f;
        for (uint32_t i = 0; i < tq_dim; i++) s = __fadd_rn(s, __fmul_rn(a[i], a[i]));
        s_val = fmaxf(__fdiv_rn(__fdiv_rn(__fsqrt_rn(s), nrm), 32.0f), 1e-8f);
    }
    __syncthreads();
    const float scale = s_val;
    int sq = 0;
    for (uint32_t i = threadIdx.x; i < dpad8; i += blockDim.x) {
        int8_t q = 0;
        if (i < tq_dim) {
            float x = roundf(__fdiv_rn(a[i], scale));             // Rust f32::round (half away from zero), clamp, `as i8` (NaN -> 0)
            x = fminf(fmaxf(x, -127.0f), 127.0f);
            q = x == x ? (int8_t)x : (int8_t)0;
        }
        o[i] = q;
        sq += (int)q * (int)q;
    }
    atomicAdd(&s_sq, sq);
    __syncthreads();
    if (threadIdx.x == 0) {
        scale_out[row] = negate ? -scale : scale;
        norm_out[row] = __fmul_rn(__fmul_rn((float)s_sq, scale), scale);
    }
}

__global__ void fill_doc_ids(uint32_t* out, const uint16_t* local_ids, uint32_t level_id, uint32_t n) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (level_id << 16) | (local_ids ? (uint32_t)local_ids[i] : i);
}

// ---------------------------------------------------------------- host side
static int32_t launch_scan_ffma_impl(const ScanArgs& a, cudaStream_t st) {
    CUtensorMap tmA, tmQ;
    uint32_t n_tiles = (uint32_t)((a.n_rows + TILE_ROWS - 1) / TILE_ROWS);
    uint32_t n_groups = a.nq_pad / QT;
    if (n_tiles == 0 || n_groups == 0) return SSB_OK;
    SSB_TRY(encode_tmap_2d_f32(&tmA, a.rows, a.dpad, a.n_rows, (uint64_t)a.dpad * 4, KC, BOX_ROWS, 1));
    SSB_TRY(encode_tmap_2d_f32(&tmQ, a.queries_padded, a.dpad, a.nq_pad, (uint64_t)a.dpad * 4, KC, QT, 0));
    uint32_t gx = n_tiles < (uint32_t)a.n_sms ? n_tiles : (uint32_t)a.n_sms;
    dim3 grid(gx, n_groups);
    uint32_t n_lists = gx * (CWARPS / 2);
    if ((size_t)n_groups * n_lists * QT * LIST * 8 > a.scratch_bytes) {
        set_error("vector scan scratch too small"); return SSB_E_STATE;
    }
    auto kern = a.similarity == SSB_SIM_EUCLIDEAN ? scan_ffma<SSB_SIM_EUCLIDEAN> : scan_ffma<SSB_SIM_DOT>;
    // per launch: the attribute belongs to the current device's context (several devices per process are allowed)
    SSB_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    if (a.ev0) cudaEventRecord(a.ev0, st);
    kern<<<grid, THREADS, SMEM_BYTES, st>>>(tmA, tmQ, (uint32_t)a.n_rows, a.dpad / KC, n_tiles, a.k, a.doc_ids,
                                            a.scratch, a.thr_init, a.nq_valid ? a.nq_valid : a.nq_pad, a.ceil_keys, a.del_slot, a.del_words, a.ivf_sel, a.ivf_words, a.row_cluster,
                                            a.sample_groupmax ? 1u : 0u);
    if (a.sample_groupmax) {
        SSB_CUDA_TRY(cudaGetLastError());
        launch_kth_from_groupmax(a.scratch, n_tiles * 16, a.nq_pad, a.k, a.thr_buf, 0, st);
        if (a.launches) *a.launches += 2;   // scan + kth
        return SSB_OK;
    }
    if (a.ev1) cudaEventRecord(a.ev1, st);
    SSB_CUDA_TRY(cudaGetLastError());
    merge_lists<<<a.nq_pad, 256, 0, st>>>(a.scratch, n_lists, QT, a.keys_out);
    SSB_CUDA_TRY(cudaGetLastError());
    if (a.launches) *a.launches += 2;   // scan + merge
    return SSB_OK;
}

int32_t launch_scan_ffma(const ScanArgs& a, cudaStream_t st) {
    // sample rows: with S of them the full scan sees ~k*N/S threshold passes per query in total, while in the sample pass itself every
    // row passes at first.  Measured on 1M x 768: best at ~N/32, 4K..32K (94-95 % of HBM peak vs 89 % at N/128; inserts stall the FFMA warps)
    const uint64_t s = a.n_rows / 32 < 4096 ? 4096 : (a.n_rows / 32 > 32768 ? 32768 : a.n_rows / 32);
    return with_threshold_seed(a, s / 512 * 512, [st](const ScanArgs& x) { return launch_scan_ffma_impl(x, st); });
}

void merge_lists_generic(const uint64_t* in, uint32_t n_lists, uint32_t qt, uint32_t nq, uint64_t* out, cudaStream_t st) {
    merge_lists<<<nq, 256, 0, st>>>(in, n_lists, qt, out);
}

size_t scan_scratch_bytes(int n_sms, uint32_t nq_pad) {
    return (size_t)(nq_pad / QT) * (size_t)n_sms * (CWARPS / 2) * QT * LIST * 8;
}

int32_t launch_prep_queries(const float* q, uint32_t nq, uint32_t dims, uint64_t qstride, float* out,
                            uint32_t nq_pad, uint32_t dpad, int normalize, cudaStream_t st) {
    if (nq_pad == 0) return SSB_OK;
    prep_queries<<<(nq_pad + 7) / 8, 256, 0, st>>>(q, nq, dims, qstride, out, nq_pad, dpad, normalize);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

int32_t launch_quantize_rows_i8(const float* src, uint64_t src_stride, uint64_t n, uint64_t n_out, uint32_t dims, int8_t* dst,
                                uint32_t dpad8, cudaStream_t st) {
    if (n_out == 0) return SSB_OK;
    quantize_rows_i8<<<(unsigned)((n_out + 7) / 8), 256, 0, st>>>(src, src_stride, n, n_out, dims, dst, dpad8);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

int32_t launch_quantize_rows_scale_i8(const float* src, uint64_t src_stride, uint64_t n, uint64_t n_out, uint32_t dims, int8_t* dst,
                                      uint32_t dpad8, float* scale_out, float* norm_out, int want_norm, cudaStream_t st) {
    if (n_out == 0) return SSB_OK;
    quantize_rows_scale_i8<<<(unsigned)((n_out + 7) / 8), 256, 0, st>>>(src, src_stride, n, n_out, dims, dst, dpad8, scale_out, norm_out, want_norm);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

int32_t launch_rows_minmax(const float* src, uint64_t src_stride, uint64_t n, uint32_t dims, float* minmax_out, cudaStream_t st) {
    if (n == 0) return SSB_OK;
    rows_minmax<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(src, src_stride, n, dims, (float2*)minmax_out);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}
int32_t launch_quantize_rows_affine_i8(const float* src, uint64_t src_stride, uint64_t n, uint64_t n_out, uint32_t dims, const float* scale_in, const int* zp_in,
                                       float st_min, float st_max, int8_t* dst, uint32_t dpad8, float* scale_out, float* norm_out, int* aff_out, int is_query,
                                       cudaStream_t st) {
    if (n_out == 0) return SSB_OK;
    quantize_rows_affine_i8<<<(unsigned)((n_out + 7) / 8), 256, 0, st>>>(src, src_stride, n, n_out, dims, scale_in, zp_in, st_min, st_max, dst, dpad8,
                                                                       scale_out, norm_out, (int2*)aff_out, is_query);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}
// the reference's running (min, max) state walked over the rows of one level on the host: per row the scale and zero point it is quantised
// with (new_scale_norm_affine, vector_similarity.rs:1414-1446); st_min / st_max are updated in place
void affine_walk_rows(const float* minmax /*[n][2]*/, uint64_t n, float* st_min, float* st_max, float* scale_out, int* zp_out) {
    for (uint64_t r = 0; r < n; r++) {
        float mn = minmax[2 * r], mx = minmax[2 * r + 1];
        ssb_affine_step(*st_min, *st_max, mn, mx);
        volatile float range = ssb_raster_range(mx - mn);
        volatile float scale = range / 255.0f;
        volatile float q = mn / scale;
        volatile float zf = -128.0f - q;
        float z = roundf(zf);
        z = z < -128.0f ? -128.0f : (z > 127.0f ? 127.0f : z);
        scale_out[r] = scale; zp_out[r] = z == z ? (int)z : 0;
    }
}

int32_t launch_quantize_rows_turbo_i8(const float* src, uint64_t src_stride, uint64_t n, uint64_t n_out, uint32_t dims, uint32_t tq_dim, const float* mask,
                                      int8_t* dst, uint32_t dpad8, float* scale_out, float* norm_out, int normalize, int negate, cudaStream_t st) {
    if (n_out == 0) return SSB_OK;
    const size_t smem = (size_t)tq_dim * 4;
    if (smem > 48 * 1024) SSB_CUDA_TRY(cudaFuncSetAttribute(quantize_rows_turbo_i8, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    quantize_rows_turbo_i8<<<(unsigned)n_out, 256, smem, st>>>(src, src_stride, n, dims, tq_dim, mask, dst, dpad8, scale_out, norm_out, normalize, negate);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

int32_t launch_normalize_rows(float* rows, uint64_t n, uint32_t dims, uint32_t dpad, int normalize, cudaStream_t st) {
    if (n == 0) return SSB_OK;
    normalize_rows<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(rows, n, dims, dpad, normalize);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

int32_t launch_fill_doc_ids(uint32_t* out, const uint16_t* local_ids, uint32_t level_id, uint32_t n, cudaStream_t st) {
    if (n == 0) return SSB_OK;
    fill_doc_ids<<<(n + 255) / 256, 256, 0, st>>>(out, local_ids, level_id, n);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

int32_t launch_merge_lists(const uint64_t* in, uint32_t n_lists, uint32_t nq, uint64_t* out, cudaStream_t st) {
    if (nq == 0) return SSB_OK;
    // in: [n_lists][nq][32]  == generic form with qt = nq (single group)
    merge_lists<<<nq, 256, 0, st>>>(in, n_lists, nq, out);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

}  // namespace vec
}  // namespace ssb
