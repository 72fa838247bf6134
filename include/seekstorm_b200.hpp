// seekstorm_b200.hpp — header-only C++17 host mirror of the reference's search interface, on top of the C-ABI
// (include/seekstorm_b200.h).  The reference is a Rust crate; no Rust toolchain exists in this build environment, so the
// compiled-language host side a SeekStorm maintainer would write in Rust (INTEGRATION.md) is mirrored here in C++ with
// the same names, argument meaning and error behaviour:
//
//   ssb::Index::search(...)            <- Search::search              seekstorm/src/search.rs:1134-1150 (impl 1153-2131)
//   ssb::QueryType / ResultType        <- search.rs `QueryType`, `ResultType` (:150-175)
//   ssb::SearchMode / AnnMode          <- search.rs `SearchMode::{Lexical,Vector,Hybrid}`, vector_similarity.rs:43-67
//   ssb::Result / ResultObject         <- min_heap.rs:17-40, search.rs:186-213
//
// Like the reference, `search` is infallible by type for data-dependent failures (unknown terms, empty index -> empty
// ResultObject, search.rs:1630-1631); programming errors (k too large, no GPU, unsupported arguments) throw ssb::Error.
// Facet counting / sort / uncommitted search / query rewriting are outside the GPU hot path and throw; facet filters, field filter and
// phrase queries go through the C-ABI (ssb_facet_filter / field_masks / SSB_QUERY_PHRASE).
#pragma once
#include <cstdint>
#include <cstring>
#include <functional>
#include <optional>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "seekstorm_b200.h"

namespace ssb {

struct Error : std::runtime_error {
    int32_t code;
    Error(int32_t c, const std::string& m) : std::runtime_error(m), code(c) {}
};
inline void check(int32_t rc) {
    if (rc != SSB_OK) throw Error(rc, std::string("libseekstorm_b200 error ") + std::to_string(rc) + ": " + ssb_last_error());
}

enum class QueryType : uint32_t { Union = SSB_QUERY_UNION, Intersection = SSB_QUERY_INTERSECTION, Phrase = SSB_QUERY_PHRASE };
enum class ResultType : uint32_t { Count = SSB_RESULT_COUNT, Topk = SSB_RESULT_TOPK, TopkCount = SSB_RESULT_TOPKCOUNT };
enum class VectorSimilarity : uint32_t { Dot = SSB_SIM_DOT, Cosine = SSB_SIM_COSINE, Euclidean = SSB_SIM_EUCLIDEAN };
enum class Quantization : uint32_t { None = SSB_QUANT_NONE, ScalarQuantizationI8 = SSB_QUANT_SCALAR_I8, TurboQuantI8 = SSB_QUANT_TURBO_I8 };   // vector.rs:230-240
// AnnMode (vector_similarity.rs:43-66): which IVF clusters of each level are searched (vector.rs:1300-1392)
struct AnnMode {
    uint32_t kind = SSB_ANN_ALL; uint32_t n_probe = 0; float threshold = 0.f;
    static AnnMode All() { return {}; }
    static AnnMode Nprobe(uint32_t n) { return {SSB_ANN_NPROBE, n, 0.f}; }
    static AnnMode Similaritythreshold(float t) { return {SSB_ANN_SIMILARITY_THRESHOLD, 0, t}; }
    static AnnMode NprobeSimilaritythreshold(uint32_t n, float t) { return {SSB_ANN_NPROBE_SIMILARITY_THRESHOLD, n, t}; }
};

struct SearchMode {
    enum Kind { Lexical, Vector, Hybrid } kind = Lexical;
    std::optional<float> similarity_threshold;
    AnnMode ann_mode = AnnMode::All();
    static SearchMode lexical() { return {Lexical, std::nullopt, AnnMode::All()}; }
    static SearchMode vector(std::optional<float> t = std::nullopt, AnnMode a = AnnMode::All()) { return {Vector, t, a}; }
    static SearchMode hybrid(std::optional<float> t = std::nullopt) { return {Hybrid, t, AnnMode::All()}; }
};

struct Result { uint64_t doc_id; float score; };

struct ResultObject {
    std::string original_query, query;
    std::vector<std::string> query_terms;
    size_t result_count = 0, result_count_total = 0;
    std::vector<Result> results;
    size_t observed_vector_count = 0;
};

// 64-bit FNV-1a with the low 3 bits cleared (the reference reserves them for the n-gram type, index.rs:4165-4225; its
// real key is an ahash of the term string — any stable 64-bit key function works as long as index and queries agree)
inline uint64_t fnv1a64(const std::string& term) {
    uint64_t h = 0xCBF29CE484222325ull;
    for (unsigned char c : term) h = (h ^ c) * 0x100000001B3ull;
    return h & ~7ull;
}

// `FacetFilter` (search.rs:735-860) resolved against the schema: facet = index of the facet field (order of set_facets), a Rust
// `Range<T>` as start <= value < end with the bounds widened to 8 bytes (u64 / i64 two's complement / f64 bits — see ssb_facet_filter),
// or the value ids of a String16 / String32 filter, or a geo distance range on a Point facet (`FacetFilter::Point`: base (lat, lon),
// start <= distance < end in unit — SSB_FILTER_POINT), or a StringSet16 / StringSet32 filter (string_set: the member ids of the filter
// strings and the combination ids whose joined key equals a filter string without holding it, search.rs:2643-2710; an empty list passes
// no doc)
struct FacetFilter {
    uint32_t facet = 0;
    uint64_t start = 0, end = 0;
    std::vector<uint64_t> values;
    bool point = false; double lat = 0.0, lon = 0.0; uint32_t unit = SSB_UNIT_KILOMETERS;
    bool is_set = false;              // SSB_FILTER_SET even with no values (a StringSet filter none of whose strings resolved)
    static FacetFilter range_u(uint32_t facet, uint64_t a, uint64_t b) { FacetFilter f; f.facet = facet; f.start = a; f.end = b; return f; }
    static FacetFilter range_i(uint32_t facet, int64_t a, int64_t b) { return range_u(facet, static_cast<uint64_t>(a), static_cast<uint64_t>(b)); }
    static FacetFilter range_f(uint32_t facet, double a, double b) { uint64_t x, y; std::memcpy(&x, &a, 8); std::memcpy(&y, &b, 8); return range_u(facet, x, y); }
    static FacetFilter set(uint32_t facet, std::vector<uint64_t> ids) { FacetFilter f; f.facet = facet; f.values = std::move(ids); return f; }
    static FacetFilter string_set(uint32_t facet, const std::vector<uint32_t>& member_ids, const std::vector<uint32_t>& combination_ids = {}) {
        FacetFilter f; f.facet = facet; f.is_set = true;
        f.values.assign(member_ids.begin(), member_ids.end());
        for (uint32_t c : combination_ids) f.values.push_back(SSB_SET_COMBINATION | c);
        return f;
    }
    static FacetFilter geo(uint32_t facet, double lat, double lon, double start, double end, uint32_t unit = SSB_UNIT_KILOMETERS) {
        FacetFilter f = range_f(facet, start, end); f.point = true; f.lat = lat; f.lon = lon; f.unit = unit; return f;
    }
};

// `ResultSort` (search.rs:893-901) resolved against the schema (ResultSortIndex, search.rs:2497-2525): a facet field (index in the order
// of set_facets; a String16 / String32 facet needs set_facet_value_order), the doc id ("_id") or the score ("_score").  A Point facet
// sorts by the distance to its base (FacetValue::Point: has_base, lat, lon; ascending = nearest first); without a base it is skipped.
enum class SortOrder : uint32_t { Ascending = SSB_SORT_ASCENDING, Descending = SSB_SORT_DESCENDING };   // search.rs:885-890
struct ResultSort {
    uint32_t source = SSB_SORT_FACET, facet = 0;
    SortOrder order = SortOrder::Descending;
    bool has_base = false; double lat = 0.0, lon = 0.0;
    static ResultSort facet_field(uint32_t facet, SortOrder o) { ResultSort r; r.facet = facet; r.order = o; return r; }
    static ResultSort geo(uint32_t facet, SortOrder o, double lat, double lon) {
        ResultSort r = facet_field(facet, o); r.has_base = true; r.lat = lat; r.lon = lon; return r;
    }
    static ResultSort id(SortOrder o) { ResultSort r; r.source = SSB_SORT_ID; r.order = o; return r; }
    static ResultSort score(SortOrder o) { ResultSort r; r.source = SSB_SORT_SCORE; r.order = o; return r; }
};

class Index {
public:
    using TermKeyFn = std::function<uint64_t(const std::string&)>;

    explicit Index(int device = 0, uint32_t vector_dims = 0, VectorSimilarity sim = VectorSimilarity::Cosine,
                   uint32_t max_batch = 4096, TermKeyFn key_fn = fnv1a64, Quantization quantization = Quantization::None)
        : key_fn_(std::move(key_fn)), sim_(sim) {
        ssb_config cfg{};
        cfg.device = device; cfg.max_batch = max_batch; cfg.vector_dims = vector_dims;
        cfg.vector_similarity = static_cast<uint32_t>(sim); cfg.vector_kernel = SSB_VEC_KERNEL_AUTO;
        cfg.vector_quantization = static_cast<uint32_t>(quantization);
        check(ssb_create(&cfg, &h_));
    }
    ~Index() { if (h_) ssb_destroy(h_); }
    Index(const Index&) = delete;
    Index& operator=(const Index&) = delete;

    ssb_index* handle() const { return h_; }

    // ---- load (what the Rust level loader of INTEGRATION.md §2 would call) ----
    void add_lexical_level(const ssb_level_desc& level) { check(ssb_lexical_add_level(h_, &level)); }
    void commit(uint64_t indexed_doc_count, uint64_t positions_sum_normalized) {
        check(ssb_lexical_commit(h_, indexed_doc_count, positions_sum_normalized));
        indexed_doc_count_ = indexed_doc_count;
    }
    void add_vector_level(uint32_t level_id, const float* rows, uint32_t n, uint32_t dims, uint64_t row_stride = 0,
                          const uint16_t* local_ids = nullptr) {
        check(ssb_vector_add_level(h_, level_id, rows, row_stride, local_ids, n, dims));
    }
    // multi-vector documents: each row's indexed field (< 32) and chunk (VectorHeader.field_id / chunk_id, vector.rs:62-73); every level of
    // an index carries them or none does.  search()'s field_filter then applies to the vector half as well (vector.rs:1226-1238).
    void add_vector_level_fields(uint32_t level_id, const float* rows, uint32_t n, uint32_t dims, const uint8_t* field_ids, const uint32_t* chunk_ids,
                                 uint64_t row_stride = 0, const uint16_t* local_ids = nullptr, const uint32_t* cluster_counts = nullptr,
                                 uint32_t n_clusters = 0) {
        check(ssb_vector_add_level_fields(h_, level_id, rows, row_stride, local_ids, n, dims, cluster_counts, n_clusters, field_ids, chunk_ids));
        if (n) vector_fields_ = true;
    }
    // a shard's vector.bin with every record's field / chunk id kept (ssb_load_vector_bin_fields); returns the number of vectors
    uint64_t load_vector_bin_fields(const void* bytes, uint64_t len) {
        uint64_t n = 0;
        check(ssb_load_vector_bin_fields(h_, bytes, len, &n));
        if (n) vector_fields_ = true;
        return n;
    }
    // the shard's facet file (facets_file_mmap): one row of row_bytes per doc id, typed fields at their offsets
    void set_facets(const void* rows, uint64_t first_doc_id, uint64_t n_docs, uint32_t row_bytes, const std::vector<ssb_facet_field>& fields) {
        check(ssb_set_facets(h_, rows, first_doc_id, n_docs, row_bytes, fields.data(), static_cast<uint32_t>(fields.size())));
    }
    // String16 / String32 facet: rank_of_id[id] = position of the id's string in byte-wise order (what sorting by the facet compares)
    void set_facet_value_order(uint32_t facet, const std::vector<uint32_t>& rank_of_id) {
        check(ssb_set_facet_value_order(h_, facet, rank_of_id.data(), static_cast<uint32_t>(rank_of_id.size())));
    }
    // StringSet16 / StringSet32 facet: the member ids of every combination as CSR (set_offsets [n_sets + 1]), n_values distinct members
    void set_facet_string_sets(uint32_t facet, const std::vector<uint64_t>& set_offsets, const std::vector<uint32_t>& members, uint32_t n_values) {
        check(ssb_set_facet_string_sets(h_, facet, set_offsets.data(), members.data(), set_offsets.empty() ? 0u : static_cast<uint32_t>(set_offsets.size() - 1), n_values));
    }
    // several indexed fields: boosts (before the first level) and the fields' names in schema order (for field_filter)
    void set_field_boosts(const std::vector<float>& boosts) { check(ssb_lexical_set_field_boosts(h_, static_cast<uint32_t>(boosts.size()), boosts.data())); }
    void set_field_names(std::vector<std::string> names) { field_names_ = std::move(names); }
    // n-gram lists: the similarity (SSB_LEXSIM_*) and df-level rule (SSB_NGRAM_DF_*) before the first level, then levels with their
    // component tfs [n_postings][3] and key-head df bytes [n_terms][3]
    void set_ngram_config(uint32_t similarity, uint32_t df_rule) { check(ssb_lexical_set_ngram_config(h_, similarity, df_rule)); }
    void add_level_ngrams(const ssb_level_desc& level, const uint16_t* component_tfs, const uint8_t* component_df_bytes) {
        const ssb_level_ngrams ng{component_tfs, component_df_bytes};
        check(ssb_lexical_add_level_ngrams(h_, &level, &ng));
    }
    // the key of an n-gram: the hash of its words joined by one space, low 3 bits replaced by its NgramType (SSB_NGRAM_*)
    static uint64_t ngram_key(uint64_t phrase_hash, uint32_t ngram_type) { return (phrase_hash & ~7ull) | (ngram_type & 7u); }
    // TurboQuantI8 indexes: the index's +-1 sign mask (TurboQuant.seed_mask)
    void set_turboquant_mask(const std::vector<float>& seed_mask) { check(ssb_vector_set_turboquant_mask(h_, seed_mask.data(), static_cast<uint32_t>(seed_mask.size()))); }
    // facet counts of a lexical batch (query_facets; ssb_search_lexical_facets), to run next to the batch's search: per query and request,
    // in request order, the (value, count) entries the call wrote.  bases: [n_queries][number of POINT requests][2] (lat, lon), or empty.
    std::vector<std::vector<std::vector<ssb_facet_count>>> facet_counts(const ssb_lex_batch& batch, const std::vector<ssb_facet_request>& req,
                                                                        const std::vector<double>& bases = {}) const {
        std::vector<size_t> cap(req.size());
        size_t stride = 0;
        for (size_t r = 0; r < req.size(); r++) stride += cap[r] = req[r].kind == SSB_FACET_COUNT_VALUES ? req[r].length : req[r].n_ranges;
        const size_t nq = batch.n_queries;
        std::vector<ssb_facet_count> out(nq * stride + 1);
        std::vector<uint32_t> n_out(nq * req.size() + 1);
        check(ssb_search_lexical_facets(h_, &batch, req.data(), static_cast<uint32_t>(req.size()), bases.empty() ? nullptr : bases.data(),
                                        out.data(), n_out.data()));
        std::vector<std::vector<std::vector<ssb_facet_count>>> res(nq, std::vector<std::vector<ssb_facet_count>>(req.size()));
        for (size_t q = 0; q < nq; q++) {
            const ssb_facet_count* p = out.data() + q * stride;
            for (size_t r = 0; r < req.size(); r++) { res[q][r].assign(p, p + n_out[q * req.size() + r]); p += cap[r]; }
        }
        return res;
    }
    uint64_t indexed_doc_count() const { return indexed_doc_count_; }
    uint64_t vector_count() const { uint64_t n = 0; check(ssb_vector_count(h_, &n)); return n; }

    // ---- Search::search (search.rs:1134-1150), 1-shard semantics, committed data ----
    ResultObject search(const std::string& query_string, const std::optional<std::vector<float>>& query_vector,
                        QueryType query_type_default, const SearchMode& search_mode, bool enable_empty_query, size_t offset,
                        size_t length, ResultType result_type, bool include_uncommitted = false,
                        const std::vector<std::string>& field_filter = {}, size_t n_query_facets = 0,
                        const std::vector<FacetFilter>& facet_filter = {}, const std::vector<ResultSort>& result_sort = {}) const {
        if (include_uncommitted || n_query_facets)
            throw Error(SSB_E_UNSUPPORTED, "facet counts / uncommitted search are outside the GPU hot path");
        if (!result_sort.empty() && search_mode.kind != SearchMode::Lexical)
            throw Error(SSB_E_UNSUPPORTED, "result_sort on vector / hybrid search is not built");
        if (enable_empty_query && query_string.empty() && !query_vector && search_mode.kind == SearchMode::Lexical)
            return search_empty(offset, length, result_type, facet_filter, result_sort);
        // field_filter: names of indexed fields (set_field_names, schema order) -> field_filter_set as a bitmask
        uint32_t field_mask = 0;
        for (auto& name : field_filter) {
            size_t f = 0;
            while (f < field_names_.size() && field_names_[f] != name) f++;
            if (f == field_names_.size()) throw Error(SSB_E_INVALID, "field_filter: unknown indexed field " + name);
            field_mask |= 1u << f;
        }
        ResultObject ro;
        ro.original_query = ro.query = query_string;
        const size_t heap = offset + length;                                   // search.rs:1708: per-shard length = offset+length
        // tokenizer stand-in (tokenizer.rs is out of scope): whitespace split, leading '+' = mandatory, unique terms
        QueryType qt = query_type_default;
        std::vector<std::string> terms, not_terms;
        {
            // "..." (or QueryType::Phrase as the default type) = a phrase: its terms in order, repeats kept (non_unique_query_list)
            std::string qs = query_string;
            bool phrase = query_type_default == QueryType::Phrase;
            if (qs.size() >= 2 && qs.front() == '"' && qs.back() == '"') { phrase = true; qs = qs.substr(1, qs.size() - 2); }
            std::istringstream is(qs);
            std::string tok; bool all_plus = true, any = false;
            while (is >> tok) {
                if (tok[0] == '"') throw Error(SSB_E_UNSUPPORTED, "a phrase mixed with other terms is outside the GPU hot path");
                if (phrase) { if (tok[0] == '+') tok.erase(0, 1); if (!tok.empty()) terms.push_back(tok); continue; }
                if (tok[0] == '-') {                                            // '-' operator: not_query_list (add_result.rs:3440-3496)
                    tok.erase(0, 1);
                    bool dup = tok.empty();
                    for (auto& t : not_terms) dup = dup || t == tok;
                    if (!dup) not_terms.push_back(tok);
                    continue;
                }
                any = true;
                if (tok[0] == '+') tok.erase(0, 1); else all_plus = false;
                if (tok.empty()) continue;
                bool dup = false;
                for (auto& t : terms) dup = dup || t == tok;
                if (!dup) terms.push_back(tok);
            }
            if (any && all_plus) qt = QueryType::Intersection;
            if (phrase) qt = terms.size() >= 2 ? QueryType::Phrase : QueryType::Intersection;
        }
        for (auto& t : terms) { bool dup = false; for (auto& u : ro.query_terms) dup = dup || u == t; if (!dup) ro.query_terms.push_back(t); }
        ResultType rt = result_type;
        if (length == 0 && rt == ResultType::TopkCount) rt = ResultType::Count;   // search.rs:2472-2478
        std::vector<ssb_hit> lex, vec;
        uint64_t total = 0;
        const bool want_lex = (search_mode.kind != SearchMode::Vector) && !terms.empty();
        const bool want_vec = (search_mode.kind != SearchMode::Lexical) && query_vector.has_value();
        if (want_lex) {
            std::vector<uint64_t> keys; std::vector<uint8_t> flags;
            for (auto& t : terms) { keys.push_back(key_fn_(t)); flags.push_back(0); }
            for (auto& t : not_terms) { keys.push_back(key_fn_(t)); flags.push_back(SSB_TERM_NOT); }
            uint32_t offs[2] = {0, static_cast<uint32_t>(keys.size())};
            ssb_lex_batch b{1, static_cast<uint32_t>(qt), offs, keys.data(), not_terms.empty() ? nullptr : flags.data(), nullptr, nullptr, nullptr, nullptr};
            // facet_filter (search.rs:735-860 -> FilterSparse per facet): applied to every candidate of the lexical search
            Filters fs(facet_filter);
            fs.apply(b);
            if (field_mask) b.field_masks = &field_mask;
            const uint32_t k = rt == ResultType::Count ? 0u : static_cast<uint32_t>(heap);
            lex.resize(k ? k : 1);
            uint32_t n = 0;
            Sort so(result_sort);
            const std::vector<ssb_sort_criterion>& sc = so.sc;
            const double* base = so.base; const bool has_base = so.has_base;
            if (sc.empty()) check(ssb_search_lexical(h_, &b, k, static_cast<uint32_t>(rt), lex.data(), &n, &total));
            else check(ssb_search_lexical_sorted_ex(h_, &b, sc.data(), static_cast<uint32_t>(sc.size()), has_base ? base : nullptr, k,
                                                    static_cast<uint32_t>(rt), lex.data(), &n, &total));
            lex.resize(n);
        }
        if (want_vec) {
            const uint32_t k = static_cast<uint32_t>(heap ? heap : 1);
            vec.resize(k);
            uint32_t n = 0;
            // search_vector_shard with all of its arguments (vector.rs:1105-1115): threshold pre-map, AnnMode, observed count behind the ABI
            ssb_vec_query vq{};
            vq.queries = query_vector->data(); vq.n_queries = 1; vq.k = k; vq.query_format = SSB_QFMT_F32;
            vq.has_threshold = search_mode.similarity_threshold ? 1u : 0u;
            vq.similarity_threshold = search_mode.similarity_threshold ? *search_mode.similarity_threshold : 0.f;
            vq.ann_mode = search_mode.ann_mode.kind; vq.n_probe = search_mode.ann_mode.n_probe; vq.cluster_threshold = search_mode.ann_mode.threshold;
            uint64_t observed = 0;
            // the field filter reaches the vector rows when they carry field ids (the reference tests every record, vector.rs:1226-1238)
            const uint32_t* vmask = field_mask && vector_fields_ ? &field_mask : nullptr;
            check(ssb_search_vector_fields(h_, &vq, vmask, vec.data(), &n, nullptr, &observed));
            vec.resize(n < heap ? n : heap);
            ro.observed_vector_count = static_cast<size_t>(observed);
        }
        std::vector<ssb_hit> fused;
        if (search_mode.kind == SearchMode::Lexical) { fused = lex; ro.result_count_total = total; }
        else if (search_mode.kind == SearchMode::Vector) { fused = vec; ro.result_count_total = vec.size(); }
        else {
            fused.resize(lex.size() + vec.size() + 1);
            uint32_t n = 0;
            check(ssb_rrf_fuse(lex.data(), static_cast<uint32_t>(lex.size()), vec.data(), static_cast<uint32_t>(vec.size()), fused.data(), &n));
            fused.resize(n);
            ro.result_count_total = total;
        }
        // search.rs:2108-2121: drop `offset`, truncate to `length`
        for (size_t i = offset; i < fused.size() && ro.results.size() < length; i++) ro.results.push_back({fused[i].doc_id, fused[i].score});
        ro.result_count = ro.results.size();
        return ro;
    }

private:
    // one query's facet filters in ABI form (ssb_facet_filter + filter_set_values), kept alive next to the batch that points at them
    struct Filters {
        std::vector<ssb_facet_filter> ff; std::vector<uint64_t> set_values; uint32_t foffs[2] = {0, 0};
        explicit Filters(const std::vector<FacetFilter>& facet_filter) {
            for (auto& f : facet_filter) {
                ssb_facet_filter c{};
                c.facet = f.facet; c.kind = f.point ? SSB_FILTER_POINT : (f.values.empty() && !f.is_set) ? SSB_FILTER_RANGE : SSB_FILTER_SET; c.start = f.start; c.end = f.end;
                c.set_first = static_cast<uint32_t>(set_values.size());
                if (f.point) {                // payload: base lat / lon as f64 bits, the unit
                    uint64_t la, lo; std::memcpy(&la, &f.lat, 8); std::memcpy(&lo, &f.lon, 8);
                    set_values.insert(set_values.end(), {la, lo, static_cast<uint64_t>(f.unit)});
                    c.set_count = 3;
                } else {
                    c.set_count = static_cast<uint32_t>(f.values.size());
                    set_values.insert(set_values.end(), f.values.begin(), f.values.end());
                }
                ff.push_back(c);
            }
            foffs[1] = static_cast<uint32_t>(ff.size());
        }
        void apply(ssb_lex_batch& b) { if (!ff.empty()) { b.filter_offsets = foffs; b.filters = ff.data(); b.filter_set_values = set_values.data(); } }
    };
    // result_sort in ABI form and the Point criterion's FacetValue::Point base (one query: one base)
    struct Sort {
        std::vector<ssb_sort_criterion> sc; double base[2] = {0.0, 0.0}; bool has_base = false;
        explicit Sort(const std::vector<ResultSort>& result_sort) {
            for (auto& r : result_sort) {
                sc.push_back(ssb_sort_criterion{r.source, r.facet, static_cast<uint32_t>(r.order), 0});
                if (r.has_base && !has_base) { base[0] = r.lat; base[1] = r.lon; has_base = true; }
            }
        }
    };
    // Search::search("", enable_empty_query = true, ..): the index route (search.rs:1413-1432, iterator.rs:360-413) without facet filter and
    // with at most one _id / _score criterion — the live doc ids from the largest (ascending when that criterion is Ascending), total = the
    // live docs for every result type; else the shard route (iterator.rs:316-358) — the filters and the sort through ssb_search_empty,
    // counted under Count / TopkCount, total 0 under Topk.
    ResultObject search_empty(size_t offset, size_t length, ResultType result_type, const std::vector<FacetFilter>& facet_filter,
                              const std::vector<ResultSort>& result_sort) const {
        ResultObject ro;
        ResultType rt = result_type;
        const bool index_route = facet_filter.empty() &&
                                 (result_sort.empty() || (result_sort.size() == 1 && result_sort[0].source != SSB_SORT_FACET));
        uint32_t offs[2] = {0, 0};
        ssb_lex_batch b{1, SSB_QUERY_UNION, offs, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
        std::vector<ssb_hit> hits;
        uint32_t n = 0;
        uint64_t total = 0;
        if (index_route) {
            check(ssb_search_empty(h_, &b, nullptr, 0, nullptr, 0, SSB_RESULT_COUNT, nullptr, &n, &total));
            ro.result_count_total = total;
            if (rt != ResultType::Count && length) {
                const ssb_sort_criterion asc{SSB_SORT_ID, 0, SSB_SORT_ASCENDING, 0};
                const bool up = !result_sort.empty() && result_sort[0].order == SortOrder::Ascending;
                hits.resize(offset + length);
                check(ssb_search_empty(h_, &b, up ? &asc : nullptr, up ? 1u : 0u, nullptr, static_cast<uint32_t>(offset + length), SSB_RESULT_TOPK,
                                       hits.data(), &n, &total));
            }
        } else {
            if (length == 0 && rt != ResultType::Count) {              // search.rs:2472-2478
                if (rt == ResultType::Topk) return ro;
                rt = ResultType::Count;
            }
            Filters fs(facet_filter);
            fs.apply(b);
            Sort so(rt == ResultType::Count ? std::vector<ResultSort>{} : result_sort);
            const uint32_t k = rt == ResultType::Count ? 0u : static_cast<uint32_t>(offset + length);
            hits.resize(k ? k : 1);
            check(ssb_search_empty(h_, &b, so.sc.data(), static_cast<uint32_t>(so.sc.size()), so.has_base ? so.base : nullptr, k,
                                   static_cast<uint32_t>(rt), hits.data(), &n, &total));
            ro.result_count_total = rt == ResultType::Topk ? 0 : total;
        }
        for (size_t i = offset; i < n && ro.results.size() < length; i++) ro.results.push_back({hits[i].doc_id, hits[i].score});
        ro.result_count = ro.results.size();
        return ro;
    }

    ssb_index* h_ = nullptr;
    TermKeyFn key_fn_;
    VectorSimilarity sim_;
    uint64_t indexed_doc_count_ = 0;
    std::vector<std::string> field_names_;
    bool vector_fields_ = false;   // vector rows carry field ids (add_vector_level_fields / load_vector_bin_fields)
};

}  // namespace ssb
