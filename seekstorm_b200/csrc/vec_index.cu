// vec_index.cu — VecIndex: vector rows and their planes, quantiser state, IVF and field tables; the host side of a vector search.
// No kernels: the launchers are in vec_scan.cu, vec_scan_tc.cu, vec_refine.cu and vec_ivf.cu.
#include <string.h>
#include <algorithm>
#include <vector>

#include "vec_index.h"

namespace ssb {

void VecIndex::init(const ssb_config& cfg, int n_sms, cudaStream_t st) {
    st_ = st; n_sms_ = n_sms;
    sim_ = cfg.vector_similarity; kernel_ = cfg.vector_kernel;
    dims_ = cfg.vector_dims;
    dpad_ = (cfg.vector_dims + 31) / 32 * 32;
    dpad8_ = (cfg.vector_dims + 127) / 128 * 128;
    quant_i8_ = cfg.vector_quantization == SSB_QUANT_SCALAR_I8 || cfg.vector_quantization == SSB_QUANT_TURBO_I8;
    turbo_ = cfg.vector_quantization == SSB_QUANT_TURBO_I8;
    if (turbo_) {
        // TurboQuant::new: dim = next power of two >= vector_dims (vector_similarity.rs:1836-1859); the codes of a row span tq_dim bytes
        uint32_t d = 1; while (d < cfg.vector_dims) d <<= 1;
        tq_dim_ = d;
        dpad8_ = (d + 127) / 128 * 128;
    }
}

int32_t VecIndex::reserve_rows(uint64_t n, bool exact) {
    const uint64_t m = n_rows_;
    SSB_TRY(doc_ids_.reserve(n, m, st_, exact));
    if (quant_i8_) {
        SSB_TRY(rows_i8_.reserve(n * dpad8_, m * dpad8_, st_, exact));
        if (turbo_ || sim_ != SSB_SIM_COSINE) { SSB_TRY(row_scale_.reserve(n, m, st_, exact)); SSB_TRY(row_norm_.reserve(n, m, st_, exact)); }
        if (affine_) SSB_TRY(row_aff_.reserve(n * 2, m * 2, st_, exact));
    } else {
        SSB_TRY(rows_.reserve(n * dpad_, m * dpad_, st_, exact));
        if (sim_ != SSB_SIM_EUCLIDEAN) {
            // the tensor-core scan reads the corpus as two bf16 planes (same 4 bytes per element as the f32 rows, which stay for
            // the FP32 scan); the filter scan reads the scaled fp16 plane
            SSB_TRY(rows_hi_.reserve(n * dpad_, m * dpad_, st_, exact));
            SSB_TRY(rows_lo_.reserve(n * dpad_, m * dpad_, st_, exact));
            SSB_TRY(rows_h16_.reserve(n * dpad_, m * dpad_, st_, exact));
        }
    }
    return SSB_OK;
}

int32_t VecIndex::reserve(uint64_t n) { return n <= n_rows_ ? SSB_OK : reserve_rows(n, true); }

int32_t VecIndex::add_level(uint32_t level_id, const float* rows, uint64_t row_stride, const uint16_t* local_ids, uint32_t n,
                            const uint32_t* cluster_counts, uint32_t n_clusters, const uint8_t* field_ids, const uint32_t* chunk_ids) {
    if (n == 0) return SSB_OK;   // an empty level (a block whose docs carry no vectors, vector.rs:1056-1073) is neither tagged nor untagged
    const int tag = field_ids ? 1 : 0;
    if (tagged_ >= 0 && tagged_ != tag) {
        set_error("vector levels %s field ids, this one %s: every level carries them or none does", tagged_ ? "carry" : "carry no", tag ? "does" : "does not");
        return SSB_E_STATE;
    }
    std::vector<uint8_t> h_fld; std::vector<uint32_t> h_chk;
    if (tag) {   // validated before anything is written
        h_fld.resize(n); h_chk.resize(n);
        SSB_CUDA_TRY(cudaMemcpy(h_fld.data(), field_ids, n, cudaMemcpyDefault));
        SSB_CUDA_TRY(cudaMemcpy(h_chk.data(), chunk_ids, (size_t)n * 4, cudaMemcpyDefault));
        for (uint32_t i = 0; i < n; i++) if (h_fld[i] >= 32) { set_error("field id %u of row %u: indexed field ids must be < 32", h_fld[i], i); return SSB_E_INVALID; }
    }
    cudaStream_t st = st_;
    const uint32_t dims = dims_;
    // device-resident inputs may still be in flight on the caller's stream (the load stream is non-blocking): load time is not
    // hot, wait for the device once
    if (is_device_ptr(rows) || (local_ids && is_device_ptr(local_ids))) SSB_CUDA_TRY(cudaDeviceSynchronize());
    // multi-chunk documents: several rows may share a local id (one vector per chunk, vector.rs:62-73); the reference's TopK keeps
    // the best chunk per doc id (vector.rs:436-470) — remember that this index needs the de-duplicating result path
    std::vector<uint16_t> h_ids;
    if (local_ids) {
        h_ids.resize(n);
        SSB_CUDA_TRY(cudaMemcpy(h_ids.data(), local_ids, (size_t)n * 2, cudaMemcpyDefault));
        std::vector<bool> seen(65536, false);
        for (uint32_t i = 0; i < n; i++) { if (seen[h_ids[i]]) dup_docs_ = true; seen[h_ids[i]] = true; }
    }
    if (turbo_ && !tq_mask_.p) { set_error("TurboQuantI8: call ssb_vector_set_turboquant_mask before adding vectors"); return SSB_E_STATE; }
    DevTmp<float> stage;
    if (quant_i8_) {
        // index-time normalise + quantise (vector.rs:585-640); the f32 rows are only staged
        SSB_CUDA_TRY(stage.alloc((size_t)n * dims));
        SSB_CUDA_TRY(cudaMemcpy2DAsync(stage.p, (size_t)dims * 4, rows, row_stride * 4, (size_t)dims * 4, n, cudaMemcpyDefault, st));
        if (!turbo_ && sim_ == SSB_SIM_EUCLIDEAN && n_rows_ == 0) {
            // Euclidean: new_scale_norm_affine when the FIRST vector of the shard is all integers in 0..255, else new_scale_norm
            // (vector.rs:651-664), decided for the shard's whole life
            std::vector<float> first(dims);
            SSB_CUDA_TRY(cudaMemcpyAsync(first.data(), stage.p, (size_t)dims * 4, cudaMemcpyDeviceToHost, st));
            SSB_CUDA_TRY(cudaStreamSynchronize(st));
            bool non_affine = false;
            for (float x : first) non_affine = non_affine || x != floorf(x) || x < 0.0f || x > 255.0f;
            affine_ = !non_affine;
        }
    }
    SSB_TRY(reserve_rows(n_rows_ + n, false));
    if (turbo_) {
        // TurboQuant::quantize_f32_i8 for every similarity (vector.rs:684-695, 729-740), after normalize_f32 for Cosine (:585-596)
        SSB_TRY(vec::launch_quantize_rows_turbo_i8(stage.p, dims, n, n, dims, tq_dim_, tq_mask_.p, rows_i8_.p + n_rows_ * dpad8_, dpad8_,
                                                   row_scale_.p + n_rows_, row_norm_.p + n_rows_, sim_ == SSB_SIM_COSINE, 0, st));
    } else if (quant_i8_ && sim_ == SSB_SIM_COSINE) {
        SSB_TRY(vec::launch_quantize_rows_i8(stage.p, dims, n, n, dims, rows_i8_.p + n_rows_ * dpad8_, dpad8_, st));
    } else if (quant_i8_ && affine_) {
        // new_scale_norm_affine: every vector is quantised with the running (min, max) of everything indexed before it — the state is
        // walked on the host over the level's per-row (min, max) (64K rows), the codes are written by one more kernel
        DevTmp<float> mm, d_scale; DevTmp<int> d_zp;
        SSB_CUDA_TRY(mm.alloc((size_t)n * 2)); SSB_CUDA_TRY(d_scale.alloc(n)); SSB_CUDA_TRY(d_zp.alloc(n));
        SSB_TRY(vec::launch_rows_minmax(stage.p, dims, n, dims, mm.p, st));
        std::vector<float> h_mm((size_t)n * 2), h_scale(n); std::vector<int> h_zp(n);
        SSB_CUDA_TRY(cudaMemcpyAsync(h_mm.data(), mm.p, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
        SSB_CUDA_TRY(cudaStreamSynchronize(st));
        float smin = aff_min_, smax = aff_max_;
        vec::affine_walk_rows(h_mm.data(), n, &smin, &smax, h_scale.data(), h_zp.data());
        SSB_CUDA_TRY(cudaMemcpyAsync(d_scale.p, h_scale.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
        SSB_CUDA_TRY(cudaMemcpyAsync(d_zp.p, h_zp.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
        SSB_TRY(vec::launch_quantize_rows_affine_i8(stage.p, dims, n, n, dims, d_scale.p, d_zp.p, 0.f, 0.f, rows_i8_.p + n_rows_ * dpad8_, dpad8_,
                                                    row_scale_.p + n_rows_, row_norm_.p + n_rows_, row_aff_.p + n_rows_ * 2, 0, st));
        SSB_CUDA_TRY(cudaStreamSynchronize(st));
        aff_min_ = smin; aff_max_ = smax;
    } else if (quant_i8_) {
        // Dot: QuantizedVector::new_scale; Euclidean: new_scale_norm (the non-affine variant)
        SSB_TRY(vec::launch_quantize_rows_scale_i8(stage.p, dims, n, n, dims, rows_i8_.p + n_rows_ * dpad8_, dpad8_,
                                                   row_scale_.p + n_rows_, row_norm_.p + n_rows_, sim_ == SSB_SIM_EUCLIDEAN, st));
    } else {
        float* dst = rows_.p + n_rows_ * dpad_;
        SSB_CUDA_TRY(cudaMemcpy2DAsync(dst, (size_t)dpad_ * 4, rows, row_stride * 4, (size_t)dims * 4, n, cudaMemcpyDefault, st));
        SSB_TRY(vec::launch_normalize_rows(dst, n, dims, dpad_, sim_ == SSB_SIM_COSINE, st));
        if (sim_ != SSB_SIM_EUCLIDEAN) {
            // the bf16 planes are split once here instead of per stage in shared memory
            SSB_TRY(vec::launch_split_rows_bf16(dst, rows_hi_.p + n_rows_ * dpad_, rows_lo_.p + n_rows_ * dpad_, (size_t)n * dpad_, st));
            // filter scan: scaled fp16 plane + its index-wide error bounds.  The scale (a power of two, fixed for the life of the index)
            // puts Cosine's unit rows below 256 and a Dot index's first level into [128, 256): later rows may be 255x larger before fp16
            // overflows — an overflowing row makes the error bound infinite and every filter query takes the exact fallback.
            if (!vec_err_.p) { SSB_TRY(vec_err_.reserve(4, 0, st, true)); SSB_CUDA_TRY(cudaMemsetAsync(vec_err_.p, 0, 16, st)); }
            if (vec_scale_ == 0.f) {
                if (sim_ == SSB_SIM_COSINE) vec_scale_ = 256.f;
                else {
                    uint32_t bits = 0;
                    SSB_TRY(vec::launch_max_abs_f32(dst, (size_t)n * dpad_, vec_err_.p + 2, st));
                    SSB_CUDA_TRY(cudaMemcpyAsync(&bits, vec_err_.p + 2, 4, cudaMemcpyDeviceToHost, st));
                    SSB_CUDA_TRY(cudaStreamSynchronize(st));
                    float mx; memcpy(&mx, &bits, 4);
                    vec_scale_ = mx > 0.f ? exp2f((float)(7 - ilogbf(mx))) : 1.f;
                }
            }
            SSB_TRY(vec::launch_rows_f16_err(dst, rows_h16_.p + n_rows_ * dpad_, n, dpad_, vec_scale_, vec_err_.p, st));
        }
    }
    DevTmp<uint16_t> tmp;
    const uint16_t* lid = local_ids;
    if (local_ids && !is_device_ptr(local_ids)) {
        SSB_CUDA_TRY(tmp.alloc(n));
        SSB_CUDA_TRY(cudaMemcpyAsync(tmp.p, h_ids.data(), (size_t)n * 2, cudaMemcpyHostToDevice, st));
        lid = tmp.p;
    }
    SSB_TRY(vec::launch_fill_doc_ids(doc_ids_.p + n_rows_, lid, level_id, n, st));
    std::vector<uint32_t> row_cl;   // tagged f32 levels: each row's global cluster id
    if (!quant_i8_) {
        // IVF tables: clusters are numbered across levels; a cluster's medoid is its first row (vector.rs:1316-1320)
        const uint32_t one = n;
        if (!cluster_counts) { cluster_counts = &one; n_clusters = 1; }
        std::vector<uint32_t> rc(n), mrow(n_clusters);
        uint32_t r = 0;
        for (uint32_t c = 0; c < n_clusters; c++) {
            mrow[c] = (uint32_t)n_rows_ + r;
            for (uint32_t i = 0; i < cluster_counts[c]; i++) rc[r++] = n_clusters_ + c;
        }
        SSB_TRY(row_cluster_.reserve(n_rows_ + n, n_rows_, st));
        SSB_TRY(cl_count_.reserve(n_clusters_ + n_clusters, n_clusters_, st));
        SSB_TRY(medoids_.reserve((size_t)(n_clusters_ + n_clusters) * dpad_, (size_t)n_clusters_ * dpad_, st));
        SSB_TRY(lvl_begin_.reserve(h_lvl_begin_.size() + 2, 0, st));
        DevTmp<uint32_t> midx; SSB_CUDA_TRY(midx.alloc(n_clusters));
        SSB_CUDA_TRY(cudaMemcpyAsync(row_cluster_.p + n_rows_, rc.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
        SSB_CUDA_TRY(cudaMemcpyAsync(cl_count_.p + n_clusters_, cluster_counts, (size_t)n_clusters * 4, cudaMemcpyHostToDevice, st));
        SSB_CUDA_TRY(cudaMemcpyAsync(midx.p, mrow.data(), (size_t)n_clusters * 4, cudaMemcpyHostToDevice, st));
        SSB_TRY(vec::launch_gather_rows(rows_.p, midx.p, n_clusters, dpad_, medoids_.p + (size_t)n_clusters_ * dpad_, st));
        if (tag) {
            cl_field_rows_.resize((size_t)(n_clusters_ + n_clusters) * 32, 0u);
            for (uint32_t i = 0; i < n; i++) cl_field_rows_[(size_t)rc[i] * 32 + h_fld[i]]++;
            row_cl = std::move(rc);
        }
        std::vector<uint32_t> lb = h_lvl_begin_; lb.push_back(n_clusters_); lb.push_back(n_clusters_ + n_clusters);
        SSB_CUDA_TRY(cudaMemcpyAsync(lvl_begin_.p, lb.data(), lb.size() * 4, cudaMemcpyHostToDevice, st));
        SSB_CUDA_TRY(cudaStreamSynchronize(st));
        h_lvl_begin_.push_back(n_clusters_);
        n_clusters_ += n_clusters;
        if (n_clusters > max_level_clusters_) max_level_clusters_ = n_clusters;
    }
    if (tag) {
        // row fields for the scans; the doc -> rows table of the best-row step: the level's (doc, row) pairs merged into the sorted list
        SSB_TRY(row_field_.reserve(n_rows_ + n, n_rows_, st));
        SSB_CUDA_TRY(cudaMemcpyAsync(row_field_.p + n_rows_, h_fld.data(), n, cudaMemcpyHostToDevice, st));
        std::vector<uint32_t> cls(n);
        for (uint32_t i = 0; i < n; i++) cls[i] = (quant_i8_ ? 0u : row_cl[i]) * 32u + h_fld[i];
        SSB_TRY(row_class_.reserve(n_rows_ + n, n_rows_, st));
        SSB_CUDA_TRY(cudaMemcpyAsync(row_class_.p + n_rows_, cls.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
        for (uint32_t i = 0; i < n; i++) field_rows_[h_fld[i]]++;
        const size_t old = doc_pairs_.size();
        for (uint32_t i = 0; i < n; i++) {
            const uint32_t doc = (level_id << 16) | (local_ids ? (uint32_t)h_ids[i] : i);
            doc_pairs_.push_back(((uint64_t)doc << 32) | (n_rows_ + i));
        }
        std::sort(doc_pairs_.begin() + old, doc_pairs_.end());
        // levels usually arrive in level order: every new doc sorts after the table's last one, and the level's entries are appended (host
        // index and device rows).  Otherwise the pairs are merged and the table is rebuilt.
        const bool append = old == 0 || (uint32_t)(doc_pairs_[old] >> 32) > doc_key_.back();
        size_t from = old;
        if (append) { if (!doc_off_.empty()) doc_off_.pop_back(); }
        else {
            std::inplace_merge(doc_pairs_.begin(), doc_pairs_.begin() + old, doc_pairs_.end());
            doc_key_.clear(); doc_off_.clear(); from = 0;
        }
        std::vector<uint32_t> rows_of(doc_pairs_.size() - from);
        for (size_t i = from; i < doc_pairs_.size(); i++) {
            const uint32_t doc = (uint32_t)(doc_pairs_[i] >> 32);
            if (doc_key_.empty() || doc_key_.back() != doc) { doc_key_.push_back(doc); doc_off_.push_back((uint32_t)i); }
            rows_of[i - from] = (uint32_t)doc_pairs_[i];
        }
        doc_off_.push_back((uint32_t)doc_pairs_.size());
        SSB_TRY(doc_rows_.reserve(doc_pairs_.size(), from, st));
        SSB_CUDA_TRY(cudaMemcpyAsync(doc_rows_.p + from, rows_of.data(), rows_of.size() * 4, cudaMemcpyHostToDevice, st));
        h_field_.insert(h_field_.end(), h_fld.begin(), h_fld.end());
        h_chunk_.insert(h_chunk_.end(), h_chk.begin(), h_chk.end());
    }
    SSB_CUDA_TRY(cudaStreamSynchronize(st));
    tagged_ = tag;
    n_rows_ += n;
    return SSB_OK;
}

// TurboQuant.seed_mask (vector_similarity.rs:1845-1859): the reference draws the +-1 mask once per index from ChaCha8Rng::seed_from_u64(1234)
// (index.rs:2215-2216) — a third-party generator this library does not restate; the host hands over the mask it holds.
int32_t VecIndex::set_turboquant_mask(const float* seed_mask, uint32_t dim) {
    if (!turbo_) { set_error("ssb_vector_set_turboquant_mask: the index was not created with SSB_QUANT_TURBO_I8"); return SSB_E_STATE; }
    if (n_rows_) { set_error("ssb_vector_set_turboquant_mask: call it before the first vector level"); return SSB_E_STATE; }
    if (dim != tq_dim_) { set_error("ssb_vector_set_turboquant_mask: dim %u, expected next_power_of_two(vector_dims) = %u", dim, tq_dim_); return SSB_E_INVALID; }
    std::vector<float> m(dim);
    SSB_CUDA_TRY(cudaMemcpy(m.data(), seed_mask, (size_t)dim * 4, cudaMemcpyDefault));
    for (float x : m) if (x != 1.0f && x != -1.0f) { set_error("ssb_vector_set_turboquant_mask: the mask must hold +1 / -1"); return SSB_E_INVALID; }
    SSB_TRY(tq_mask_.reserve(dim, 0, st_, true));
    SSB_CUDA_TRY(cudaMemcpy(tq_mask_.p, m.data(), (size_t)dim * 4, cudaMemcpyHostToDevice));
    return SSB_OK;
}

template <class A>
void VecIndex::i8_operands(A& a, const VecWorkspace& ws) const {
    a.rows_i8 = rows_i8_.p; a.queries_i8 = ws.q_i8.p; a.dpad8 = dpad8_;
    if (turbo_ || sim_ != SSB_SIM_COSINE) {
        a.i8_scaled = sim_ == SSB_SIM_EUCLIDEAN ? (affine_ ? 3 : 2) : 1;
        a.row_scale = row_scale_.p; a.row_norm = row_norm_.p; a.q_scale = ws.q_scale.p; a.q_norm = ws.q_norm.p;
        a.row_aff = row_aff_.p; a.q_aff = ws.q_aff.p;
    }
}

int32_t VecIndex::search_keys(VecWorkspace& ws, cudaStream_t st, ssb_stats& stats, bool* timed, const void* queries, bool queries_i8, uint32_t nq,
                              uint32_t k, uint64_t* keys_out_dev, const uint64_t* ceil_dev, const IvfQuery* ivf, const uint32_t* fmask_host) const {
    if (ivf && (quant_i8_ || !medoids_.p)) { set_error("AnnMode other than All needs an f32 vector index"); return SSB_E_UNSUPPORTED; }
    if (dims_ == 0) { set_error("no vector index configured (vector_dims = 0)"); return SSB_E_STATE; }
    if (k == 0 || k > SSB_K_MAX) { set_error("k must be in 1..%u", SSB_K_MAX); return SSB_E_UNSUPPORTED; }
    if (queries_i8 && !quant_i8_) { set_error("int8 queries need a ScalarQuantizationI8 index"); return SSB_E_INVALID; }
    if (nq == 0) return SSB_OK;
    const vec::Scan scan = vec::plan_scan(kernel_, sim_, quant_i8_, rows_h16_.p && vec_err_.p, nq, k, ceil_dev != nullptr);
    const bool filter = vec::is_filter(scan);
    const uint32_t passes = (nq + vec::queries_per_pass(scan) - 1) / vec::queries_per_pass(scan);   // corpus passes of the scan
    const uint32_t nq_pad = passes * vec::queries_per_pass(scan);
    const bool cosine = sim_ == SSB_SIM_COSINE;
    if (scan != vec::Scan::I8_128) SSB_TRY(ws.qpad.reserve((size_t)nq_pad * dpad_, 0, st));
    const size_t qbytes = (size_t)nq * dims_ * (queries_i8 ? 1 : 4);
    const void* qsrc = queries;
    if (!is_device_ptr(queries)) {
        SSB_TRY(ws.qstage.reserve(((size_t)nq * dims_ + 3) / (queries_i8 ? 4 : 1) + 1, 0, st));
        SSB_CUDA_TRY(cudaMemcpyAsync(ws.qstage.p, queries, qbytes, cudaMemcpyHostToDevice, st));
        stats.h2d_bytes += qbytes;
        qsrc = ws.qstage.p;
    }
    if (scan == vec::Scan::I8_128) {
        SSB_TRY(ws.q_i8.reserve((size_t)nq_pad * dpad8_, 0, st));
        if (queries_i8 && (turbo_ || !cosine)) { set_error("int8 query codes are accepted for Cosine + ScalarQuantizationI8 only (the other quantisers need the query scale)"); return SSB_E_UNSUPPORTED; }
        if (turbo_ || !cosine) { SSB_TRY(ws.q_scale.reserve(nq_pad, 0, st)); SSB_TRY(ws.q_norm.reserve(nq_pad, 0, st)); }   // scaled epilogues (i8_operands)
        if (turbo_) {
            // the query goes through the same TurboQuant as the rows (search.rs:1545-1556, 1592-1602).  Dot / Cosine: the reference's score is
            // -(dot * query_scale * row_scale) (vector_similarity.rs:161-176): the NEGATED query scale through the scaled epilogue is exactly that
            SSB_TRY(vec::launch_quantize_rows_turbo_i8((const float*)qsrc, dims_, nq, nq_pad, dims_, tq_dim_, tq_mask_.p, ws.q_i8.p, dpad8_, ws.q_scale.p,
                                                       ws.q_norm.p, cosine, sim_ != SSB_SIM_EUCLIDEAN, st));
        } else if (affine_) {
            // affine Euclidean: the query is quantised with a COPY of the shard's (min, max) state (search.rs:1514-1530, 1562-1580)
            SSB_TRY(ws.q_aff.reserve((size_t)nq_pad * 2, 0, st));
            SSB_TRY(vec::launch_quantize_rows_affine_i8((const float*)qsrc, dims_, nq, nq_pad, dims_, nullptr, nullptr, aff_min_, aff_max_, ws.q_i8.p, dpad8_,
                                                        ws.q_scale.p, ws.q_norm.p, ws.q_aff.p, 1, st));
        } else if (!cosine) {
            // Dot / Euclidean: the query goes through the same QuantizedVector::new_scale[_norm] as the rows (search.rs:1499-1530)
            SSB_TRY(vec::launch_quantize_rows_scale_i8((const float*)qsrc, dims_, nq, nq_pad, dims_, ws.q_i8.p, dpad8_, ws.q_scale.p, ws.q_norm.p,
                                                       sim_ == SSB_SIM_EUCLIDEAN, st));
        } else if (queries_i8) {
            // the caller already ran normalize + quantize_f32_to_i8 (what the reference's server holds after search.rs:1477-1490): pad only
            SSB_CUDA_TRY(cudaMemsetAsync(ws.q_i8.p, 0, (size_t)nq_pad * dpad8_, st));
            SSB_CUDA_TRY(cudaMemcpy2DAsync(ws.q_i8.p, dpad8_, qsrc, dims_, dims_, nq, cudaMemcpyDeviceToDevice, st));
        } else {
            // the query is normalised and quantised exactly like the corpus (search.rs:1464-1475, vector_similarity.rs:1226-1232)
            SSB_TRY(vec::launch_quantize_rows_i8((const float*)qsrc, dims_, nq, nq_pad, dims_, ws.q_i8.p, dpad8_, st));
        }
    } else if (filter || scan == vec::Scan::Bf16_64 || scan == vec::Scan::Bf16_128 || scan == vec::Scan::Bf16_256) {
        // one launch: pad + normalise + bf16 hi/lo split (the scan reads only the split parts)
        SSB_TRY(ws.qhi.reserve((size_t)nq_pad * dpad_, 0, st));
        SSB_TRY(ws.qlo.reserve((size_t)nq_pad * dpad_, 0, st));
        if (filter) SSB_TRY(ws.q_scale.reserve(nq_pad, 0, st));   // per-query margins 2 eps_q
        SSB_TRY(vec::launch_prep_split_queries_bf16((const float*)qsrc, nq, dims_, dims_, ws.qhi.p, ws.qlo.p, nq_pad, dpad_, cosine, st,
                                                    (filter || ivf) ? ws.qpad.p : nullptr, filter ? ws.q_scale.p : nullptr, filter ? vec_err_.p : nullptr));
    } else
    SSB_TRY(vec::launch_prep_queries((const float*)qsrc, nq, dims_, dims_, ws.qpad.p, nq_pad, dpad_, cosine, st));
    stats.kernel_launches += 1;
    if (n_rows_ == 0) { SSB_CUDA_TRY(cudaMemsetAsync(keys_out_dev, 0, (size_t)nq * LIST * 8, st)); return SSB_OK; }
    size_t sb = vec::is_tensor_core(scan) ? vec::scan_tc_scratch_bytes(n_sms_, nq_pad) : vec::scan_scratch_bytes(n_sms_, nq_pad);
    const size_t head_words = sb / 8 + (size_t)nq_pad * LIST + (nq_pad + 1) / 2;
    SSB_TRY(ws.scratch.reserve(head_words + (filter ? vec::refine_scratch_words(n_sms_, nq_pad) : 0), 0, st));
    vec::ScanArgs a{};
    a.rows = rows_.p; a.rows_hi = rows_hi_.p; a.rows_lo = rows_lo_.p; a.rows_h16 = rows_h16_.p; a.doc_ids = doc_ids_.p; a.n_rows = n_rows_; a.dpad = dpad_; a.queries_padded = ws.qpad.p;
    a.nq_pad = nq_pad; a.nq_valid = nq; a.k = k; a.similarity = sim_; a.n_sms = n_sms_;
    a.scratch = ws.scratch.p; a.scratch_bytes = sb;
    uint64_t* merged = ws.scratch.p + sb / 8;   // [nq_pad][32]
    a.keys_out = merged; a.ev0 = ws.ev0; a.ev1 = ws.ev1; *timed = true;
    a.thr_buf = reinterpret_cast<uint32_t*>(merged + (size_t)nq_pad * LIST);
    a.ceil_keys = ceil_dev;
    if (del_->n) { a.del_slot = del_->d_slot; a.del_words = del_->d_words; }
    a.launches = &stats.kernel_launches;
    uint32_t unmerged = 0;
    if (filter) a.unmerged_lists = &unmerged;
    if (ivf) {
        // cluster probe: medoid scores, per-(query, level) selection -> one bit per (query, cluster); the scans test it per candidate
        vec::IvfArgs v{};
        v.medoids = medoids_.p; v.lvl_begin = lvl_begin_.p; v.cl_count = cl_count_.p;
        v.n_clusters = n_clusters_; v.n_levels = (uint32_t)h_lvl_begin_.size(); v.max_level_clusters = max_level_clusters_;
        v.queries_padded = ws.qpad.p; v.nq = nq; v.nq_pad = nq_pad; v.dpad = dpad_; v.similarity = sim_;
        v.ann_mode = ivf->mode; v.n_probe = ivf->n_probe; v.cluster_threshold = ivf->thr;
        v.words = (n_clusters_ + 31) / 32;
        SSB_TRY(ws.ivf_scores.reserve((size_t)nq * n_clusters_, 0, st));
        SSB_TRY(ws.ivf_sel.reserve((size_t)nq_pad * v.words, 0, st));
        SSB_TRY(ws.ivf_obs.reserve(nq, 0, st));
        v.scores = ws.ivf_scores.p; v.sel = ws.ivf_sel.p; v.observed = ws.ivf_obs.p; v.launches = &stats.kernel_launches;
        SSB_TRY(vec::launch_ivf_select(v, st));
        a.ivf_sel = ws.ivf_sel.p; a.ivf_words = v.words; a.row_cluster = row_cluster_.p;
    }
    if (fmask_host) {
        // field filter (vector.rs:1226-1238): folded into the scans' per-candidate IVF test — a row's class is cluster * 32 + field and
        // the selection holds, per (query, cluster), the fields the query scans.  Like the IVF mask it turns the threshold seed off.
        const uint32_t n_cl = quant_i8_ ? 1u : n_clusters_;
        SSB_TRY(ws.fmask.reserve(nq_pad, 0, st));
        SSB_TRY(ws.fsel.reserve((size_t)nq_pad * n_cl, 0, st));
        SSB_CUDA_TRY(cudaMemsetAsync(ws.fmask.p, 0, (size_t)nq_pad * 4, st));   // padding queries: no filter (they collect nothing anyway)
        SSB_CUDA_TRY(cudaMemcpyAsync(ws.fmask.p, fmask_host, (size_t)nq * 4, cudaMemcpyHostToDevice, st));
        stats.h2d_bytes += (uint64_t)nq * 4;
        SSB_TRY(vec::launch_field_sel(a.ivf_sel, a.ivf_words, ws.fmask.p, nq_pad, n_cl, ws.fsel.p, st));
        stats.kernel_launches += 1;
        a.ivf_sel = ws.fsel.p; a.ivf_words = n_cl; a.row_cluster = row_class_.p;
    }
    if (scan == vec::Scan::I8_128) {
        i8_operands(a, ws);
    } else if (vec::is_tensor_core(scan)) {
        SSB_TRY(ws.qhi.reserve((size_t)nq_pad * dpad_, 0, st));
        SSB_TRY(ws.qlo.reserve((size_t)nq_pad * dpad_, 0, st));
        a.q_hi = ws.qhi.p; a.q_lo = ws.qlo.p;
        if (filter) a.q_scale = ws.q_scale.p;
    }
    SSB_TRY(vec::is_tensor_core(scan) ? vec::launch_scan_tc(a, scan, st) : vec::launch_scan_ffma(a, st));
    if (filter) {
        vec::RefineArgs r{};
        r.rows = rows_.p; r.doc_ids = doc_ids_.p; r.n_rows = n_rows_; r.dpad = dpad_; r.queries_padded = ws.qpad.p; r.margin = ws.q_scale.p;
        r.keys = merged; r.keys_out = keys_out_dev;   // the refine step writes the caller's buffer directly
        if (unmerged) { r.lists = a.scratch; r.n_lists = unmerged; r.qt = vec::queries_per_pass(scan); }   // seeded 256-query pass: merged in the refine step
        r.nq = nq; r.nq_pad = nq_pad; r.k = k;
        r.fb_lists = ws.scratch.p + head_words;
        r.fb_state = reinterpret_cast<uint32_t*>(r.fb_lists + (size_t)nq_pad * n_sms_ * LIST);
        r.del_slot = a.del_slot; r.del_words = a.del_words; r.ivf_sel = a.ivf_sel; r.ivf_words = a.ivf_words; r.row_cluster = a.row_cluster; r.n_sms = n_sms_; r.launches = &stats.kernel_launches;
        SSB_TRY(vec::launch_refine(r, st));
        ws.fb_state = r.fb_state;
    } else {
        SSB_CUDA_TRY(cudaMemcpyAsync(keys_out_dev, merged, (size_t)nq * LIST * 8, cudaMemcpyDeviceToDevice, st));
    }
    const uint64_t pass_bytes = n_rows_ * dims_ * (scan == vec::Scan::I8_128 ? 1 : 4);   // algorithmic bytes of one corpus pass
    stats.algorithmic_bytes += passes * pass_bytes;
    // bytes the scan kernel actually streams per call: the filter scan reads the 2-byte fp16 plane (half the f32 bytes), the refine step
    // <= 32 f32 rows per query
    stats.scan_bytes_read += filter ? passes * pass_bytes / 2 + (uint64_t)nq * LIST * dims_ * 4 : passes * pass_bytes;
    return SSB_OK;
}

int32_t VecIndex::field_masks(const uint32_t* masks, uint32_t nq, const char* who, const uint32_t** use) const {
    *use = nullptr;
    if (!masks) return SSB_OK;
    if (is_device_ptr(masks)) { set_error("%s: field_masks must be a host array", who); return SSB_E_INVALID; }
    bool any = false;
    for (uint32_t q = 0; q < nq; q++) any = any || masks[q] != 0u;
    if (!any) return SSB_OK;
    if (tagged_ != 1) { set_error("%s: a field mask needs vector rows with field ids (ssb_vector_add_level_fields)", who); return SSB_E_STATE; }
    *use = masks;
    return SSB_OK;
}

int32_t VecIndex::best_rows(VecWorkspace& ws, cudaStream_t st, ssb_stats& stats, const void* queries, uint32_t nq, uint32_t k, const ssb_hit* hits,
                            const uint32_t* nh, const uint32_t* fmask_host, ssb_hit_ext* ext) const {
    std::vector<uint32_t> hq;   // per hit: (query, first CSR entry, row count, 0)
    std::vector<uint32_t> slot;  // ext index of each hit
    for (uint32_t q = 0; q < nq; q++)
        for (uint32_t j = 0; j < nh[q]; j++) {
            const uint32_t doc = (uint32_t)hits[(size_t)q * k + j].doc_id;
            const auto it = std::lower_bound(doc_key_.begin(), doc_key_.end(), doc);
            if (it == doc_key_.end() || *it != doc) continue;
            const size_t d = (size_t)(it - doc_key_.begin());
            hq.insert(hq.end(), {q, doc_off_[d], doc_off_[d + 1] - doc_off_[d], 0u});
            slot.push_back(q * k + j);
        }
    const uint32_t n = (uint32_t)slot.size();
    if (n == 0) return SSB_OK;
    SSB_TRY(ws.best.reserve((size_t)n * 5, 0, st));
    SSB_TRY(ws.fmask.reserve(nq, 0, st));
    if (fmask_host) SSB_CUDA_TRY(cudaMemcpyAsync(ws.fmask.p, fmask_host, (size_t)nq * 4, cudaMemcpyHostToDevice, st));
    else SSB_CUDA_TRY(cudaMemsetAsync(ws.fmask.p, 0, (size_t)nq * 4, st));
    SSB_CUDA_TRY(cudaMemcpyAsync(ws.best.p, hq.data(), (size_t)n * 16, cudaMemcpyHostToDevice, st));
    vec::BestRowArgs b{};
    b.n_hits = n; b.hits = reinterpret_cast<const uint4*>(ws.best.p); b.doc_rows = doc_rows_.p; b.best_row = ws.best.p + (size_t)n * 4;
    b.field_mask = ws.fmask.p; b.row_field = row_field_.p;
    if (quant_i8_) {
        i8_operands(b, ws);   // the int8 codes (and scales) of the queries are still in the workspace from the search's last page
    } else {
        const void* qsrc = is_device_ptr(queries) ? queries : ws.qstage.p;   // host queries were staged by the search
        SSB_TRY(ws.qpad.reserve((size_t)nq * dpad_, 0, st));
        SSB_TRY(vec::launch_prep_queries((const float*)qsrc, nq, dims_, dims_, ws.qpad.p, nq, dpad_, sim_ == SSB_SIM_COSINE, st));
        stats.kernel_launches += 1;
        b.rows = rows_.p; b.queries = ws.qpad.p; b.dpad = dpad_; b.euclid = sim_ == SSB_SIM_EUCLIDEAN;
    }
    SSB_TRY(vec::launch_best_rows(b, st));
    stats.kernel_launches += 1;
    ws.h_best.resize(n);
    SSB_CUDA_TRY(cudaMemcpyAsync(ws.h_best.data(), b.best_row, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    SSB_CUDA_TRY(cudaStreamSynchronize(st));
    stats.h2d_bytes += (uint64_t)n * 16; stats.d2h_bytes += (uint64_t)n * 4;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t row = ws.h_best[i];
        if (row == 0xFFFFFFFFu) continue;
        ext[slot[i]].field_id = h_field_[row];
        ext[slot[i]].chunk_id = h_chunk_[row];
    }
    return SSB_OK;
}

int32_t VecIndex::masked_observed(VecWorkspace& ws, cudaStream_t st, uint32_t nq, const uint32_t* fmask_host, bool use_ivf, uint64_t* observed) const {
    std::vector<uint32_t> sel;
    const uint32_t words = (n_clusters_ + 31) / 32;
    if (use_ivf) {
        sel.resize((size_t)nq * words);
        SSB_CUDA_TRY(cudaMemcpyAsync(sel.data(), ws.ivf_sel.p, sel.size() * 4, cudaMemcpyDeviceToHost, st));
        SSB_CUDA_TRY(cudaStreamSynchronize(st));
    }
    for (uint32_t q = 0; q < nq; q++) {
        const uint32_t m = fmask_host[q];
        if (!m) continue;
        uint64_t n = 0;
        if (!use_ivf) { for (uint32_t f = 0; f < 32; f++) if ((m >> f) & 1u) n += field_rows_[f]; }
        else
            for (uint32_t cl = 0; cl < n_clusters_; cl++)
                if ((sel[(size_t)q * words + cl / 32] >> (cl % 32)) & 1u)
                    for (uint32_t f = 0; f < 32; f++) if ((m >> f) & 1u) n += cl_field_rows_[(size_t)cl * 32 + f];
        observed[q] = n;
    }
    return SSB_OK;
}

}  // namespace ssb
