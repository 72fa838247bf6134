// vec_index.h — vector index in HBM (rows, quantiser state, IVF and field tables) + batched query execution (host code).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>

#include "bm25.h"
#include "vec_scan.h"

namespace ssb {

struct IvfQuery { uint32_t mode, n_probe; float thr; };   // AnnMode of one call (thr pre-mapped, vector.rs:388-399)

// Per-call vector scratch of one search context (api.cu keeps a pool of them: concurrent searches on one index do not share any).
struct VecWorkspace {
    DevBuf<float> qpad, qstage, qhi, qlo, q_scale, q_norm; DevBuf<int8_t> q_i8; DevBuf<int> q_aff;
    DevBuf<uint64_t> scratch;
    DevBuf<float> ivf_scores; DevBuf<uint32_t> ivf_sel; DevBuf<uint64_t> ivf_obs; std::vector<uint64_t> h_obs;   // IVF probe (vec_ivf.cu)
    DevBuf<uint32_t> fmask, fsel, best; std::vector<uint32_t> h_best;   // field filter: per-query masks, per (query, cluster) fields; best-row step
    const uint32_t* fb_state = nullptr;   // filter scan of the current call: device count of queries that took the exact fallback
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;   // recorded around the scan kernel
};

class VecIndex {
public:
    // cfg: vector_dims / similarity / kernel / quantization of ssb_create (validated there); st: the load-time stream
    void init(const ssb_config& cfg, int n_sms, cudaStream_t st);
    void set_deleted(const DeleteSet* d) { del_ = d; }
    void set_kernel(uint32_t kernel) { kernel_ = kernel; }
    uint32_t dims() const { return dims_; }
    bool quant_i8() const { return quant_i8_; }
    bool euclid() const { return sim_ == SSB_SIM_EUCLIDEAN; }
    uint64_t n_rows() const { return n_rows_; }
    bool dup_docs() const { return dup_docs_; }   // some doc id occurs on more than one row: results are de-duplicated per doc
    bool tagged() const { return tagged_ == 1; }

    // capacity hint (ssb_vector_reserve): every per-row plane for n rows, allocated once at exactly that size
    int32_t reserve(uint64_t n);
    // one level (= one add call); arguments checked by the caller.  cluster_counts: the level's IVF cluster table or null (one cluster);
    // field_ids / chunk_ids: both or neither (ssb_vector_add_level_fields)
    int32_t add_level(uint32_t level_id, const float* rows, uint64_t row_stride, const uint16_t* local_ids, uint32_t n,
                      const uint32_t* cluster_counts, uint32_t n_clusters, const uint8_t* field_ids, const uint32_t* chunk_ids);
    int32_t set_turboquant_mask(const float* seed_mask, uint32_t dim);
    // keys of nq queries (host or device, f32 or int8 codes) -> keys_out_dev [nq][32].  Asynchronous on st; thread-safe for concurrent
    // calls with distinct workspaces.  ceil_dev: [>= nq_pad] exclusive paging ceilings or null; ivf: null = AnnMode::All; fmask_host: [nq]
    // field masks of a field-tagged index, or null: no query has one.  *timed is set when ws.ev0 / ev1 were recorded around the scan.
    int32_t search_keys(VecWorkspace& ws, cudaStream_t st, ssb_stats& stats, bool* timed, const void* queries, bool queries_i8, uint32_t nq,
                        uint32_t k, uint64_t* keys_out_dev, const uint64_t* ceil_dev = nullptr, const IvfQuery* ivf = nullptr,
                        const uint32_t* fmask_host = nullptr) const;
    // field masks of a vector search (HOST array [nq], bit f = indexed field f, 0 = no filter; the bits of ssb_lex_batch.field_masks).
    // *use = the array when some query has a mask, else null: an unmasked batch runs exactly the unfiltered path.  A mask on an index
    // whose rows carry no field ids is refused rather than ignored.
    int32_t field_masks(const uint32_t* masks, uint32_t nq, const char* who, const uint32_t** use) const;
    // vb field_id / chunk_id of every returned hit of a field-tagged index: the doc's best row among those passing the query's mask
    // (launch_best_rows).  Runs after search_keys, on the queries it left in ws (f32: prepared again, int8: its quantised codes).
    int32_t best_rows(VecWorkspace& ws, cudaStream_t st, ssb_stats& stats, const void* queries, uint32_t nq, uint32_t k, const ssb_hit* hits,
                      const uint32_t* nh, const uint32_t* fmask_host, ssb_hit_ext* ext) const;
    // observed_vector_count of a masked query: the rows in scope whose field passes the mask — every row (AnnMode::All) or the rows of the
    // clusters the probe selected (its selection bits are still in ws)
    int32_t masked_observed(VecWorkspace& ws, cudaStream_t st, uint32_t nq, const uint32_t* fmask_host, bool use_ivf, uint64_t* observed) const;

private:
    // every per-row plane this config writes, for n rows (growth, or exactly n)
    int32_t reserve_rows(uint64_t n, bool exact);
    // the int8 scan's epilogue operands (ScanArgs / BestRowArgs): codes, and the per-vector scales / norms / zero points of the scaled variants
    template <class A> void i8_operands(A& a, const VecWorkspace& ws) const;

    cudaStream_t st_ = nullptr;
    int n_sms_ = 0;
    uint32_t sim_ = 0, kernel_ = 0;
    const DeleteSet* del_ = nullptr;
    uint32_t dims_ = 0, dpad_ = 0, dpad8_ = 0;
    bool quant_i8_ = false;           // ScalarQuantizationI8 / TurboQuantI8: int8 corpus, exact int32 dot products
    bool turbo_ = false;              // TurboQuantI8: rows and queries are sign-flipped, FWHT-rotated and quantised at tq_dim = next_pow2(dims)
    uint32_t tq_dim_ = 0; DevBuf<float> tq_mask_;   // the index's seed mask (+-1), ssb_vector_set_turboquant_mask
    bool dup_docs_ = false;
    DevBuf<float> rows_;
    DevBuf<uint16_t> rows_hi_, rows_lo_;   // bf16 planes of `rows` (hi = bf16_rn(x), lo = bf16_rn(x - hi)): what the tensor-core bf16 scan streams
    DevBuf<int8_t> rows_i8_;
    DevBuf<float> row_scale_, row_norm_;   // Dot / Euclidean + ScalarQuantizationI8: per-vector scale (and norm), QuantizedVector vector_similarity.rs:1340-1371
    // Euclidean + ScalarQuantizationI8 over integer-valued 0..255 data: the AFFINE quantiser (new_scale_norm_affine, vector_similarity.rs:1414-1463)
    bool affine_ = false; float aff_min_ = 3.402823466e+38f /* f32::MAX */, aff_max_ = -3.402823466e+38f /* f32::MIN */;   // shard.min / max_vector_value
    DevBuf<int> row_aff_;                 // int2 per row: (zero_point, dims * zero_point - sum_q)
    DevBuf<uint32_t> doc_ids_;
    DevBuf<uint16_t> rows_h16_;       // filter scan: fp16 plane half_rn(rows * vec_scale)
    DevBuf<uint32_t> vec_err_;        // filter scan: {max_r |a_r*scale - h_r|, max_r |h_r|, scratch} as f32 bits (launch_rows_f16_err)
    float vec_scale_ = 0.f;           // power of two; 0 = not chosen yet (first add_level)
    // IVF cluster tables (vector.rs:1066-1094; f32 indexes): one entry per add call ("level"), clusters numbered across levels
    DevBuf<float> medoids_; DevBuf<uint32_t> row_cluster_, cl_count_, lvl_begin_;
    std::vector<uint32_t> h_lvl_begin_; uint32_t n_clusters_ = 0, max_level_clusters_ = 0;
    // multi-vector documents (ssb_vector_add_level_fields; VectorHeader.field_id / chunk_id, vector.rs:62-73): every level carries them or
    // none does.  row_field: the byte the best-row step tests; row_class: cluster * 32 + field, what the scans' IVF test reads under a field
    // mask (int8 indexes: one cluster); h_field / h_chunk: what the best-row step reports; field_rows / cl_field_rows: rows per field, and
    // per (cluster, field) on f32 indexes, for observed_vector_count under a mask.  doc_rows (device) lists every doc's rows in record
    // order, grouped by doc; doc_key / doc_off (host) index it.
    int tagged_ = -1;                 // -1: no vector level yet, 0: untagged, 1: field-tagged
    DevBuf<uint8_t> row_field_; DevBuf<uint32_t> row_class_; std::vector<uint8_t> h_field_; std::vector<uint32_t> h_chunk_;
    uint64_t field_rows_[32] = {}; std::vector<uint32_t> cl_field_rows_;   // [n_clusters][32]
    DevBuf<uint32_t> doc_rows_; std::vector<uint64_t> doc_pairs_ /*(doc << 32) | row, sorted*/; std::vector<uint32_t> doc_key_, doc_off_;
    uint64_t n_rows_ = 0;
};

}  // namespace ssb
