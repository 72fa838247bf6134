// facets.cu — FacetSet: the device-resident facet columns of an index (ssb_set_facets), their per-block zones and the value orders of
// String facets (ssb_set_facet_value_order); and the reduction of a sorted search's criteria against them.
#include <algorithm>

#include "common.cuh"
#include "facets.h"

namespace ssb {

// one CTA per zone block: min / max of the block's column keys (or ranks) -> zone[2 * block]
__global__ void __launch_bounds__(256) facet_zone_minmax(const uint64_t* __restrict__ col, uint64_t rows, uint32_t first_doc, uint32_t block0,
                                                         const uint32_t* __restrict__ rank, uint32_t n_rank, uint64_t* __restrict__ zone) {
    __shared__ uint64_t smin[8], smax[8];
    const uint64_t d0 = (uint64_t)(block0 + blockIdx.x) << 16;
    const uint64_t lo = d0 > first_doc ? d0 - first_doc : 0, hi = (d0 + 65536 - first_doc) < rows ? d0 + 65536 - first_doc : rows;
    uint64_t mn = ~0ull, mx = 0;
    for (uint64_t r = lo + threadIdx.x; r < hi; r += blockDim.x) {
        uint64_t x = col[r];
        if (rank) x = x < n_rank ? rank[x] : ~0ull;
        mn = x < mn ? x : mn; mx = x > mx ? x : mx;
    }
    for (int s = 16; s; s >>= 1) {
        const uint64_t a = shfl64_xor(mn, s), b = shfl64_xor(mx, s);
        mn = a < mn ? a : mn; mx = b > mx ? b : mx;
    }
    if ((threadIdx.x & 31) == 0) { smin[threadIdx.x >> 5] = mn; smax[threadIdx.x >> 5] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < 8; i++) { mn = smin[i] < mn ? smin[i] : mn; mx = smax[i] > mx ? smax[i] : mx; }
        zone[2 * blockIdx.x] = mn; zone[2 * blockIdx.x + 1] = mx;
    }
}
// the member occurrences of every row of a StringSet column: sum over rows of the size of the row's combination -> *out
__global__ void __launch_bounds__(256) facet_member_rows(const uint64_t* __restrict__ col, uint64_t rows, const uint64_t* __restrict__ set_off,
                                                         unsigned long long* out) {
    unsigned long long s = 0;
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t c = col[r];
        s += set_off[c + 1] - set_off[c];
    }
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(out, s);
}
// per-block min / max of facet f's column (through its value order when it has one) -> d_zones; asynchronous on st
static int32_t facet_zones(FacetSet& fs, uint32_t f, cudaStream_t st) {
    if (!fs.n_facets || !fs.n_rows) return SSB_OK;
    if (!fs.d_zones) {
        fs.zone_block0 = fs.first_doc >> 16;
        fs.n_zone_blocks = (uint32_t)(((uint64_t)fs.first_doc + fs.n_rows - 1) >> 16) - fs.zone_block0 + 1;
        SSB_CUDA_TRY(cudaMalloc(&fs.d_zones, (size_t)fs.n_facets * fs.n_zone_blocks * 16));
    }
    facet_zone_minmax<<<fs.n_zone_blocks, 256, 0, st>>>(fs.d_keys + (size_t)f * fs.n_rows, fs.n_rows, fs.first_doc, fs.zone_block0, fs.d_rank[f], fs.n_rank[f],
                                                        fs.d_zones + (size_t)f * fs.n_zone_blocks * 2);
    SSB_CUDA_TRY(cudaGetLastError());
    return SSB_OK;
}

// facets_file_mmap (is_facet_filter, add_result.rs:340-478, reads `facets_size_sum * docid + facet.offset`): every value becomes an
// order-preserving 64-bit key, one column per facet, so the kernels test any FilterSparse range with two unsigned compares.
int32_t FacetSet::set_columns(const void* rows, uint64_t first_doc_id, uint64_t n_docs, uint32_t row_bytes, const ssb_facet_field* fields,
                              uint32_t n_fields, cudaStream_t st) {
    release();
    if (n_docs == 0 || n_fields == 0) return SSB_OK;
    if (!rows || !fields) { set_error("ssb_set_facets: null argument"); return SSB_E_INVALID; }
    if (n_fields > SSB_MAX_FACETS) { set_error("ssb_set_facets: more than %u facets", SSB_MAX_FACETS); return SSB_E_UNSUPPORTED; }
    if (first_doc_id + n_docs > (1ull << 32)) { set_error("ssb_set_facets: doc ids must be < 2^32"); return SSB_E_INVALID; }
    for (uint32_t f = 0; f < n_fields; f++) {
        const uint32_t w = facet_type_bytes(fields[f].type);
        if (!w) { set_error("ssb_set_facets: field %u has unsupported type %u", f, fields[f].type); return SSB_E_UNSUPPORTED; }
        if ((uint64_t)fields[f].offset + w > row_bytes) { set_error("ssb_set_facets: field %u does not fit a %u-byte row", f, row_bytes); return SSB_E_INVALID; }
    }
    std::vector<uint64_t> keys((size_t)n_fields * n_docs);
    const uint8_t* base = (const uint8_t*)rows;
    for (uint32_t f = 0; f < n_fields; f++) {
        uint64_t* col = keys.data() + (size_t)f * n_docs;
        const uint32_t type = fields[f].type, off = fields[f].offset;
        for (uint64_t d = 0; d < n_docs; d++) col[d] = facet_value_key(type, base + d * row_bytes + off);
    }
    SSB_CUDA_TRY(cudaMalloc(&d_keys, keys.size() * 8));
    SSB_CUDA_TRY(cudaMemcpy(d_keys, keys.data(), keys.size() * 8, cudaMemcpyHostToDevice));
    n_rows = n_docs; first_doc = (uint32_t)first_doc_id; n_facets = n_fields;
    for (uint32_t f = 0; f < n_fields; f++) {
        types[f] = (uint8_t)fields[f].type;
        const uint64_t* col = keys.data() + (size_t)f * n_docs;
        max_key[f] = *std::max_element(col, col + n_docs);
        SSB_TRY(facet_zones(*this, f, st));                          // per-level bounds of sorted searches
    }
    SSB_CUDA_TRY(cudaStreamSynchronize(st));
    return SSB_OK;
}

int32_t FacetSet::set_value_order(uint32_t facet, const uint32_t* rank_of_id, uint32_t n_ids, cudaStream_t st) {
    cudaFree(d_rank[facet]); d_rank[facet] = nullptr; n_rank[facet] = 0;
    SSB_CUDA_TRY(cudaMalloc(&d_rank[facet], (size_t)n_ids * 4));
    SSB_CUDA_TRY(cudaMemcpy(d_rank[facet], rank_of_id, (size_t)n_ids * 4, cudaMemcpyHostToDevice));
    n_rank[facet] = n_ids;
    SSB_TRY(facet_zones(*this, facet, st));                          // the level bounds of this facet are ranks from now on
    SSB_CUDA_TRY(cudaStreamSynchronize(st));
    return SSB_OK;
}

int32_t FacetSet::set_string_sets(uint32_t facet, const uint64_t* set_offsets, const uint32_t* members, uint32_t ns, uint32_t nv, cudaStream_t st) {
    cudaFree(d_set_off[facet]); d_set_off[facet] = nullptr; cudaFree(d_set_mem[facet]); d_set_mem[facet] = nullptr;
    cudaFree(d_rank[facet]); d_rank[facet] = nullptr; n_rank[facet] = 0; n_sets[facet] = 0; n_values[facet] = 0; member_rows[facet] = 0;
    const uint64_t n_mem = set_offsets[ns];
    const std::vector<uint32_t> rank = string_set_sort_ranks(set_offsets, members, ns);
    SSB_CUDA_TRY(cudaMalloc(&d_set_off[facet], ((size_t)ns + 1) * 8));
    SSB_CUDA_TRY(cudaMemcpy(d_set_off[facet], set_offsets, ((size_t)ns + 1) * 8, cudaMemcpyHostToDevice));
    // member occurrences over every row: the members a pass over all rows reads (ssb_last_stats of the empty query's counts)
    unsigned long long* d_occ = nullptr;
    SSB_CUDA_TRY(cudaMalloc(&d_occ, 8));
    cudaMemsetAsync(d_occ, 0, 8, st);
    facet_member_rows<<<(uint32_t)std::min<uint64_t>((n_rows + 255) / 256, 4096), 256, 0, st>>>(d_keys + (size_t)facet * n_rows, n_rows, d_set_off[facet], d_occ);
    unsigned long long occ = 0;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(&occ, d_occ, 8, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(d_occ);
    if (e != cudaSuccess) { set_error("ssb_set_facet_string_sets: %s", cudaGetErrorString(e)); return SSB_E_CUDA; }
    SSB_CUDA_TRY(cudaMalloc(&d_set_mem[facet], (size_t)std::max<uint64_t>(n_mem, 1) * 4));
    if (n_mem) SSB_CUDA_TRY(cudaMemcpy(d_set_mem[facet], members, (size_t)n_mem * 4, cudaMemcpyHostToDevice));
    SSB_CUDA_TRY(cudaMalloc(&d_rank[facet], (size_t)ns * 4));
    SSB_CUDA_TRY(cudaMemcpy(d_rank[facet], rank.data(), (size_t)ns * 4, cudaMemcpyHostToDevice));
    n_rank[facet] = ns; n_sets[facet] = ns; n_values[facet] = nv; member_rows[facet] = occ;
    SSB_TRY(facet_zones(*this, facet, st));                          // the level bounds of this facet are first-member ranks from now on
    SSB_CUDA_TRY(cudaStreamSynchronize(st));
    return SSB_OK;
}

int32_t sort_of_criteria(const FacetSet* fs, const ssb_sort_criterion* crit, uint32_t n, bool has_bases, SortDev* out, bool* sorted) {
    if (n && !crit) { set_error("search_lexical_sorted: null criteria"); return SSB_E_INVALID; }
    if (n > SSB_MAX_SORT_CRITERIA) { set_error("search_lexical_sorted: more than %u criteria", SSB_MAX_SORT_CRITERIA); return SSB_E_UNSUPPORTED; }
    const uint32_t nf = fs ? fs->n_facets : 0;
    for (uint32_t i = 0; i < n; i++) {
        if (crit[i].source > SSB_SORT_SCORE || crit[i].order > SSB_SORT_DESCENDING) { set_error("sort criterion %u: bad source / order", i); return SSB_E_INVALID; }
        if (crit[i].source == SSB_SORT_FACET && nf && crit[i].facet >= nf) { set_error("sort criterion %u: facet %u of %u", i, crit[i].facet, nf); return SSB_E_INVALID; }
    }
    SortDev s{};
    uint32_t bits = 0;
    bool any_facet = false, ended = false;
    for (uint32_t i = 0; i < n && !ended; i++) {                   // _id / _score end the comparison (min_heap.rs:580-604)
        const ssb_sort_criterion& c = crit[i];
        if (c.source == SSB_SORT_SCORE) { s.score_asc = c.order == SSB_SORT_ASCENDING; ended = true; continue; }
        // a Point facet without a FacetValue::Point base is skipped (min_heap.rs:510-529: `if let FacetValue::Point(base)`)
        if (c.source == SSB_SORT_FACET && nf && fs->types[c.facet] == SSB_FACET_POINT && !has_bases) continue;
        ended = c.source == SSB_SORT_ID;
        const uint32_t j = s.n++;
        s.src[j] = c.source == SSB_SORT_ID ? SORT_SRC_ID : SORT_SRC_FACET; s.desc[j] = c.order == SSB_SORT_DESCENDING;
        if (s.src[j] == SORT_SRC_FACET) { s.facet[j] = c.facet; any_facet = true; }
        s.type[j] = s.src[j] == SORT_SRC_FACET && nf ? fs->types[c.facet] : 0u;
        bits += sort_width(s.src[j], s.type[j]);
    }
    *sorted = s.n > 0 || s.score_asc;
    if (!*sorted) return SSB_OK;
    if (any_facet && !nf) { set_error("search_lexical_sorted: sorting by a facet needs ssb_set_facets"); return SSB_E_STATE; }
    if (bits > 64) { set_error("search_lexical_sorted: the criteria take %u bits (at most 64)", bits); return SSB_E_UNSUPPORTED; }
    if (any_facet) {
        for (uint32_t j = 0; j < s.n; j++) {
            if (s.src[j] != SORT_SRC_FACET) continue;
            const uint32_t f = s.facet[j];
            if (facet_is_string(s.type[j])) {
                if (!fs->d_rank[f] || fs->max_key[f] >= fs->n_rank[f]) {
                    set_error("search_lexical_sorted: String facet %u needs a value order covering its ids (ssb_set_facet_value_order)", f); return SSB_E_STATE;
                }
                s.rank[j] = fs->d_rank[f];
            } else if (facet_is_stringset(s.type[j])) {
                if (!fs->n_sets[f]) { set_error("search_lexical_sorted: StringSet facet %u needs its string sets (ssb_set_facet_string_sets)", f); return SSB_E_STATE; }
                s.rank[j] = fs->d_rank[f];                           // the first-member ranks of set_string_sets
            }
        }
        s.zones = fs->d_zones; s.zone_block0 = fs->zone_block0; s.n_zone_blocks = fs->n_zone_blocks;
    }
    *out = s;
    return SSB_OK;
}

}  // namespace ssb
