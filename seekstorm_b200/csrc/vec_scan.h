// vec_scan.h — host-visible launchers of the vector kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "scan_plan.h"

namespace ssb {
namespace vec {

struct ScanArgs {
    const float* rows;            // [n_rows][dpad]
    const void* rows_hi = nullptr; const void* rows_lo = nullptr;   // bf16 planes [n_rows][dpad] of the same rows (tensor-core bf16 scan)
    const void* rows_h16 = nullptr;   // scaled fp16 plane [n_rows][dpad] (filter scan)
    const uint32_t* doc_ids;      // [n_rows] or nullptr
    uint64_t n_rows;
    uint32_t dpad;                // multiple of 32
    const float* queries_padded;  // [nq_pad][dpad], nq_pad a multiple of the scan's queries_per_pass
    uint32_t nq_pad;
    uint32_t nq_valid = 0;         // real queries; rows >= nq_valid are zero padding and must never collect candidates
    uint32_t k;
    uint32_t similarity;
    int n_sms;
    uint64_t* scratch;
    size_t scratch_bytes;
    uint64_t* keys_out;           // [nq_pad][32]
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;   // recorded around the scan kernel when set
    float* q_hi = nullptr; float* q_lo = nullptr;  // [nq_pad][dpad] tf32 split of the queries (tensor-core kernel)
    uint32_t* thr_buf = nullptr;                   // [nq_pad] scratch for the pre-sampled per-query thresholds
    const uint32_t* thr_init = nullptr;            // internal: initial thresholds (ordered-uint scores) or null
    const uint64_t* ceil_keys = nullptr;           // [nq_pad] exclusive key ceilings for paging beyond 32 results, or null
    uint64_t* launches = nullptr;                  // incremented once per kernel launched (ssb_stats.kernel_launches)
    const int8_t* rows_i8 = nullptr;               // int8 path: [n_rows][dpad8] quantised corpus
    const int8_t* queries_i8 = nullptr;            //            [nq_pad][dpad8] quantised queries
    uint32_t dpad8 = 0;                            //            multiple of 128
    int i8_scaled = 0;                             // int8 path: 0 = Cosine SQ (plain int32 dot), 1 = Dot SQ (per-vector scales), 2 = Euclidean SQ non-affine (+ norms), 3 = Euclidean SQ affine (+ zero points / code sums)
    const float* row_scale = nullptr; const float* row_norm = nullptr;   // [n_rows]
    const float* q_scale = nullptr; const float* q_norm = nullptr;       // [nq_pad]
    const int* row_aff = nullptr; const int* q_aff = nullptr;            // i8_scaled 3 (affine Euclidean SQ): int2 per row (zp, dims*zp - sum_q) / per query (zp, sum_q)
    const uint32_t* del_slot = nullptr; const uint64_t* del_words = nullptr;   // delete set (null = none): deleted docs never enter a list
    bool sample_groupmax = false;                  // internal (int8): threshold-seeding pass, writes thr_buf instead of lists
    // IVF probe (vec_ivf.cu): selection mask [nq_pad][ivf_words] (bit per (query, cluster)) and each row's cluster id; null = AnnMode::All.
    // A field mask of a field-tagged index arrives the same way (launch_field_sel: row_cluster = cluster * 32 + field), on the int8 scans
    // too.  Like the delete set it disables the threshold-seeding sample pass (an unselected row must never seed a threshold).
    const uint32_t* ivf_sel = nullptr; uint32_t ivf_words = 0; const uint32_t* row_cluster = nullptr;
    // filter scan: receives the number of lists per query the scan left unmerged in `scratch` ([nq_pad / NQ][n][NQ][32]) for the refine
    // step to merge (the seeded 256-query pass, one list per query per CTA), or 0 when keys_out holds the merged lists.  Null: always merge.
    uint32_t* unmerged_lists = nullptr;
};

// Threshold seeding: `launch` first scans the first `sample_rows` rows keeping only each 32-row group's best score per query (no
// lists, no merge); the k-th largest of those group maxima (kth_from_groupmax) is a valid lower bound of the final k-th best score —
// k different groups each hold a row at least that good — and, written to thr_buf, seeds the threshold of the full scan: results are
// unchanged, but the expected number of list insertions per query drops from ~k*ln(rows/k) PER LIST to ~k*N/S in total.  Skipped
// below 64 K rows, and with a delete set or an IVF mask: a deleted or unselected row must never seed a threshold.
template <class F>
int32_t with_threshold_seed(const ScanArgs& a, uint64_t sample_rows, F launch) {
    if (a.thr_init || !a.thr_buf || a.del_slot || a.ivf_sel || a.n_rows < 65536) return launch(a);
    ScanArgs pre = a;
    pre.n_rows = sample_rows; pre.ev0 = nullptr; pre.ev1 = nullptr;
    pre.sample_groupmax = true;   // the sample launch writes the thresholds (thr_buf) itself
    SSB_TRY(launch(pre));
    ScanArgs full = a;
    full.thr_init = a.thr_buf;
    return launch(full);
}

int32_t launch_scan_ffma(const ScanArgs& a, cudaStream_t st);
size_t scan_scratch_bytes(int n_sms, uint32_t nq_pad);
int32_t launch_scan_tc(const ScanArgs& a, Scan s /*any but Scan::Ffma*/, cudaStream_t st);
size_t scan_tc_scratch_bytes(int n_sms, uint32_t nq_pad);
// fused query preparation of the bf16 tensor-core scan: pad + (Cosine) normalise + hi/lo split in one launch
int32_t launch_prep_split_queries_bf16(const float* q, uint32_t nq, uint32_t dims, uint64_t qstride, void* hi, void* lo, uint32_t nq_pad,
                                       uint32_t dpad, int normalize, cudaStream_t st, float* f32_out = nullptr, float* margin_out = nullptr,
                                       const uint32_t* row_err = nullptr);
// filter scan (vec_refine.cu / DESIGN.md §3.2c).  launch_rows_f16_err: load time, h16 = half_rn(rows * scale), err[0] = max_r |a_r*scale - h_r|,
// err[1] = max_r |h_r| (f32 bits, atomicMax).  launch_max_abs_f32: *out_bits = max(*out_bits, max|x|) over finite elements.
int32_t launch_rows_f16_err(const float* rows, void* h16, uint64_t n, uint32_t dpad, float scale, uint32_t* err, cudaStream_t st);
int32_t launch_max_abs_f32(const float* x, size_t n, uint32_t* out_bits, cudaStream_t st);
struct RefineArgs {
    const float* rows; const uint32_t* doc_ids; uint64_t n_rows; uint32_t dpad;
    const float* queries_padded;      // [nq_pad][dpad] f32 (normalised for Cosine)
    const float* margin;              // [nq_pad] 2 eps_q
    const uint64_t* keys;             // in: merged approximate keys [nq_pad][32] (low word = 0xFFFFFFFF - row), unless `lists` is set
    const uint64_t* lists = nullptr;  // in: the scan's unmerged lists [nq_pad / qt][n_lists][qt][32] (ScanArgs::unmerged_lists), or null
    uint32_t n_lists = 0, qt = 0;
    uint64_t* keys_out;               // out: exact keys [nq][32] (low word = 0xFFFFFFFF - doc id); may alias `keys`
    uint32_t nq, nq_pad, k;
    uint32_t* fb_state;               // [1 + nq_pad]: count of flagged queries + their indices (zeroed by the refine launch)
    uint64_t* fb_lists;               // [nq_pad][n_sms][32] fallback scratch
    const uint32_t* del_slot; const uint64_t* del_words;
    const uint32_t* ivf_sel; uint32_t ivf_words; const uint32_t* row_cluster;   // IVF selection mask (null = all clusters)
    int n_sms;
    uint64_t* launches;
};
// best row of each returned (query, doc) of a field-tagged index (vb field_id / chunk_id, TopK::push vector.rs:436-470): re-score the doc's
// rows that pass the query's field mask and keep the argmax, the earliest row on equal scores (push replaces only on a strictly better score)
struct BestRowArgs {
    uint32_t n_hits;
    const uint4* hits;                // [n_hits] (query, first CSR entry, row count, -)
    const uint32_t* doc_rows;         // CSR: the rows of every doc, grouped by doc, ascending (= record order) inside a doc
    const uint32_t* field_mask; const uint8_t* row_field;   // [nq] masks (0 = none), [n_rows] field ids
    const float* rows; const float* queries; uint32_t dpad; int euclid;   // f32 index: rows / padded queries (normalised for Cosine)
    const int8_t* rows_i8 = nullptr; const int8_t* queries_i8 = nullptr; uint32_t dpad8 = 0; int i8_scaled = 0;   // int8 index (ScanArgs)
    const float* row_scale = nullptr; const float* row_norm = nullptr; const float* q_scale = nullptr; const float* q_norm = nullptr;
    const int* row_aff = nullptr; const int* q_aff = nullptr;
    uint32_t* best_row;               // out [n_hits]: the winning row, 0xFFFFFFFF when no row passes
};
int32_t launch_best_rows(const BestRowArgs& a, cudaStream_t st);
// IVF probe: medoid scores + per-(query, level) cluster selection -> sel bits, observed vector counts (vec_ivf.cu)
struct IvfArgs {
    const float* medoids;             // [n_clusters][dpad] f32 copies of each cluster's first row
    const uint32_t* lvl_begin;        // [n_levels + 1] first cluster id of every level (arena order)
    const uint32_t* cl_count;         // [n_clusters] vectors per cluster
    uint32_t n_clusters, n_levels, max_level_clusters;
    const float* queries_padded;      // [nq_pad][dpad] f32 (normalised for Cosine)
    uint32_t nq, nq_pad, dpad, similarity;
    uint32_t ann_mode, n_probe; float cluster_threshold;   // SSB_ANN_*; threshold already pre-mapped (vector.rs:388-399)
    float* scores;                    // [nq][n_clusters] scratch
    uint32_t* sel; uint32_t words;    // [nq_pad][words]
    uint64_t* observed;               // [nq]
    uint64_t* launches;
};
int32_t launch_ivf_select(const IvfArgs& a, cudaStream_t st);
// field filter of a field-tagged index, folded into the scans' IVF test: a row's class is cluster * 32 + field (row_cluster of the
// scans), and out[q][c] holds the fields of cluster c that query q scans — its mask (all 32 bits for mask 0) where the probe selected
// the cluster (sel = [nq_pad][sel_words] bits, or null = every cluster), else 0.  out: [nq_pad][n_cl]
int32_t launch_field_sel(const uint32_t* sel, uint32_t sel_words, const uint32_t* fmask, uint32_t nq_pad, uint32_t n_cl, uint32_t* out, cudaStream_t st);
int32_t launch_gather_rows(const float* src, const uint32_t* idx_dev, uint32_t n, uint32_t dpad, float* dst, cudaStream_t st);
// re-score the candidates in f32, sort, flag candidate-set overflows; then the exact fallback scan for flagged queries (exits at once when none)
int32_t launch_refine(const RefineArgs& a, cudaStream_t st);
size_t refine_scratch_words(int n_sms, uint32_t nq_pad);   // u64 words behind fb_lists + fb_state
// load time: f32 rows (already normalised) -> bf16 hi / lo planes
int32_t launch_split_rows_bf16(const float* rows, void* hi, void* lo, size_t n_elems, cudaStream_t st);
// lists laid out [group][n_lists][qt][32] -> out [nq][32]
// thr[q] = ordered-uint score of the k-th entry of keys[q][32] (0 if the list is shorter)
// thr[q] = k-th largest group maximum (sample mode of the scans; is_int: int32 dot products instead of ordered-uint scores)
void launch_kth_from_groupmax(const void* gmax, uint32_t n_groups, uint32_t nq, uint32_t k, uint32_t* thr, int is_int, cudaStream_t st);
void merge_lists_generic(const uint64_t* in, uint32_t n_lists, uint32_t qt, uint32_t nq, uint64_t* out, cudaStream_t st);
int32_t launch_prep_queries(const float* q, uint32_t nq, uint32_t dims, uint64_t qstride, float* out,
                            uint32_t nq_pad, uint32_t dpad, int normalize, cudaStream_t st);
// f32 rows -> normalize_f32 + quantize_f32_to_i8 (bit-identical to the reference's scalar arithmetic); rows >= n are zero
int32_t launch_quantize_rows_i8(const float* src, uint64_t src_stride, uint64_t n, uint64_t n_out, uint32_t dims, int8_t* dst,
                                uint32_t dpad8, cudaStream_t st);
// QuantizedVector::new_scale / new_scale_norm (vector_similarity.rs:1340-1371): scale = max|x| / 127, codes = round(x / scale) as i8,
// norm = sum(code^2) as f32 * scale * scale (want_norm).  Every step is order-independent (max, exact integer sum): bit-identical to the CPU.
int32_t launch_quantize_rows_scale_i8(const float* src, uint64_t src_stride, uint64_t n, uint64_t n_out, uint32_t dims, int8_t* dst,
                                      uint32_t dpad8, float* scale_out, float* norm_out, int want_norm, cudaStream_t st);
// QuantizedVector::new_scale_norm_affine (vector_similarity.rs:1414-1463), integer-valued 0..255 data: codes = round(x / scale) + zero_point.
// rows: scale_in / zp_in hold each row's scale and zero point (the host walked the reference's running min / max state over the rows);
// queries (scale_in == null): every query derives them itself from the index's state (st_min, st_max), as search.rs:1514-1530 does with a copy.
// aff_out: int2 per row — rows (zero_point, dims * zero_point - sum_q), queries (zero_point, sum_q).  minmax_out (pass 1 for rows): float2 per row.
int32_t launch_rows_minmax(const float* src, uint64_t src_stride, uint64_t n, uint32_t dims, float* minmax_out, cudaStream_t st);
int32_t launch_quantize_rows_affine_i8(const float* src, uint64_t src_stride, uint64_t n, uint64_t n_out, uint32_t dims, const float* scale_in, const int* zp_in,
                                       float st_min, float st_max, int8_t* dst, uint32_t dpad8, float* scale_out, float* norm_out, int* aff_out, int is_query,
                                       cudaStream_t st);
void affine_walk_rows(const float* minmax, uint64_t n, float* st_min, float* st_max, float* scale_out, int* zp_out);
// TurboQuantI8 (vector_similarity.rs:1929-1958): pad to tq_dim, sign mask, FWHT, scale = max(sigma / 32, 1e-8); rows >= n are zero rows
int32_t launch_quantize_rows_turbo_i8(const float* src, uint64_t src_stride, uint64_t n, uint64_t n_out, uint32_t dims, uint32_t tq_dim, const float* mask,
                                      int8_t* dst, uint32_t dpad8, float* scale_out, float* norm_out, int normalize, int negate, cudaStream_t st);
int32_t launch_normalize_rows(float* rows, uint64_t n, uint32_t dims, uint32_t dpad, int normalize, cudaStream_t st);
int32_t launch_fill_doc_ids(uint32_t* out, const uint16_t* local_ids, uint32_t level_id, uint32_t n, cudaStream_t st);
// in: [n_lists][nq][32] descending lists -> out [nq][32]
int32_t launch_merge_lists(const uint64_t* in, uint32_t n_lists, uint32_t nq, uint64_t* out, cudaStream_t st);

}  // namespace vec
}  // namespace ssb
