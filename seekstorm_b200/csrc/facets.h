// facets.h — the facet key format: one order-preserving 64-bit key per facet value, the filters and sort criteria of a batch in that key
// space, and the host encoders that produce them.  Compiles with plain g++ (tests/test_facets_cpu.py); helpers the kernels call too are
// SSB_HD, __host__ __device__ under nvcc.  facets.cuh holds the device side, facets.cu the device-resident columns (FacetSet).
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include <vector>

#include "../../include/seekstorm_b200.h"

#ifdef __CUDACC__
#define SSB_HD __host__ __device__ __forceinline__
#else
#define SSB_HD inline
#endif

namespace ssb {

void set_error(const char* fmt, ...);   // api.cu: the calling thread's last error

// One facet filter of one query, bounds already in key space (FilterSparse, search.rs:863-881): RANGE lo <= key < hi;
// SET key in filt_sets[set_first .. +set_n); NEVER rejects every doc (a NaN bound: Range::contains is false for every value);
// POINT: lo <= Morton code < hi, then the distance test with the staged geo payload filt_sets[set_first .. +GEO_WORDS);
// MEMBERS (SET on a StringSet facet): the key is a combination id, lo / hi the device addresses of the facet's CSR (set offsets, member
// ids), the staged payload filt_sets[set_first .. +set_n) = {F, F flagged combination ids ascending, the member ids ascending, unique}
enum { FILT_RANGE = 0, FILT_SET = 1, FILT_NEVER = 2, FILT_POINT = 3, FILT_MEMBERS = 4 };
// payload of a POINT filter in filt_sets, as f64 bits: base lat, base lon, distance start, distance end, earth radius of the unit
enum { GEO_LAT = 0, GEO_LON = 1, GEO_START = 2, GEO_END = 3, GEO_RADIUS = 4, GEO_WORDS = 5 };
struct FiltDev { uint32_t facet, kind; uint64_t lo, hi; uint32_t set_first, set_n; };

// The sort of one sorted batch (ssb_search_lexical_sorted), validated and reduced by sort_of_criteria (facets.cu).  Criteria 0..n-1 are the
// facet / _id criteria that make up the packed key `hi` (sort_pack_hi in facets.cuh); a `_score` criterion ends the list and only sets score_asc.
enum { SORT_SRC_FACET = 0, SORT_SRC_ID = 1 };
struct SortDev {
    uint32_t n; uint32_t score_asc;                    // score_asc: `_score` ascending — the score half of the 128-bit top-k key is inverted
    uint32_t src[4], facet[4], type[4], desc[4];      // per criterion (type: SSB_FACET_* of a facet criterion)
    const uint32_t* rank[4];                           // String facets: rank_of_id (ssb_set_facet_value_order), else null
    const uint64_t* zones; uint32_t zone_block0, n_zone_blocks;   // FacetSet zones (level bounds)
    const double* bases;                               // a POINT criterion: [n_queries][2] per-query base (lat, lon), staged by stage_sort_bases
};

// ---- keys: FilterSparse bounds and facet values -> the key space of the facet columns ----
// Keys: unsigned types as they are; signed types and Timestamp with the sign bit flipped; F32 / F64 through the f64 value's bits
// (negative: all bits flipped, else sign bit set; -0.0 counts as +0.0, PartialOrd) — NaN has no key: a NaN VALUE gets ~0, which
// no range contains (every finite / infinite bound maps below it), a NaN BOUND makes the filter reject everything.
// The order key of an f64: the F32 / F64 column key, the float filter bounds and the distance key of a Point sort criterion.
SSB_HD uint64_t f64_order_key(double x) {
    if (x != x) return ~0ull;
    if (x == 0.0) x = 0.0;                                           // -0.0 == +0.0
#ifdef __CUDA_ARCH__
    const uint64_t b = (uint64_t)__double_as_longlong(x);
#else
    uint64_t b; memcpy(&b, &x, 8);
#endif
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
// the f64 of a key f64_order_key made, other than NaN's (-0.0 comes back as +0.0)
SSB_HD double f64_of_order_key(uint64_t k) {
    const uint64_t b = (k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k;
#ifdef __CUDA_ARCH__
    return __longlong_as_double((long long)b);
#else
    double x; memcpy(&x, &b, 8); return x;
#endif
}
inline bool facet_is_signed(uint32_t t) { return t == SSB_FACET_I8 || t == SSB_FACET_I16 || t == SSB_FACET_I32 || t == SSB_FACET_I64 || t == SSB_FACET_TIMESTAMP; }
inline bool facet_is_float(uint32_t t) { return t == SSB_FACET_F32 || t == SSB_FACET_F64; }
inline bool facet_is_string(uint32_t t) { return t == SSB_FACET_STRING16 || t == SSB_FACET_STRING32; }
inline bool facet_is_stringset(uint32_t t) { return t == SSB_FACET_STRINGSET16 || t == SSB_FACET_STRINGSET32; }
// facet value (as stored in the reference's facet file) -> order-preserving key
inline uint64_t facet_value_key(uint32_t type, const uint8_t* p) {
    switch (type) {
        case SSB_FACET_U8: return p[0];
        case SSB_FACET_U16: case SSB_FACET_STRING16: case SSB_FACET_STRINGSET16: { uint16_t x; memcpy(&x, p, 2); return x; }
        case SSB_FACET_U32: case SSB_FACET_STRING32: case SSB_FACET_STRINGSET32: { uint32_t x; memcpy(&x, p, 4); return x; }
        case SSB_FACET_U64: case SSB_FACET_POINT: { uint64_t x; memcpy(&x, p, 8); return x; }   // Point: the Morton code itself
        case SSB_FACET_I8: { int8_t x; memcpy(&x, p, 1); return (uint64_t)(int64_t)x ^ 0x8000000000000000ull; }
        case SSB_FACET_I16: { int16_t x; memcpy(&x, p, 2); return (uint64_t)(int64_t)x ^ 0x8000000000000000ull; }
        case SSB_FACET_I32: { int32_t x; memcpy(&x, p, 4); return (uint64_t)(int64_t)x ^ 0x8000000000000000ull; }
        case SSB_FACET_I64: case SSB_FACET_TIMESTAMP: { int64_t x; memcpy(&x, p, 8); return (uint64_t)x ^ 0x8000000000000000ull; }
        case SSB_FACET_F32: { float x; memcpy(&x, p, 4); return f64_order_key((double)x); }
        case SSB_FACET_F64: { double x; memcpy(&x, p, 8); return f64_order_key(x); }
    }
    return ~0ull;
}
// byte width of a facet type (0 = unknown type)
inline uint32_t facet_type_bytes(uint32_t type) {
    switch (type) {
        case SSB_FACET_U8: case SSB_FACET_I8: return 1;
        case SSB_FACET_U16: case SSB_FACET_I16: case SSB_FACET_STRING16: case SSB_FACET_STRINGSET16: return 2;
        case SSB_FACET_U32: case SSB_FACET_I32: case SSB_FACET_F32: case SSB_FACET_STRING32: case SSB_FACET_STRINGSET32: return 4;
        case SSB_FACET_U64: case SSB_FACET_I64: case SSB_FACET_TIMESTAMP: case SSB_FACET_F64: case SSB_FACET_POINT: return 8;
    }
    return 0;
}

// ---- sort keys (ssb_search_lexical_sorted; result_ordering_shard, min_heap.rs:574-1051) ----
// The width a criterion takes in the packed key `hi` (sort_pack_hi): its natural width, 64 for the 64-bit types and Point distances.  A
// table of its own rather than 8 * facet_type_bytes: written that way, sort_pack_hi (once per criterion) costs lex_plan<true> 224 and
// every sorted lex_generic 152 more SASS instructions (CUDA 12.9, sm_90a).
SSB_HD uint32_t sort_width(uint32_t src, uint32_t type) {
    if (src == SORT_SRC_ID) return 32;
    switch (type) {
        case SSB_FACET_U8: case SSB_FACET_I8: return 8;
        case SSB_FACET_U16: case SSB_FACET_I16: case SSB_FACET_STRING16: case SSB_FACET_STRINGSET16: return 16;
        case SSB_FACET_U32: case SSB_FACET_I32: case SSB_FACET_F32: case SSB_FACET_STRING32: case SSB_FACET_STRINGSET32: return 32;
    }
    return 64;
}
// The sort rank of every combination of a StringSet facet (CSR set_offsets [n_sets + 1] / members): the reference sorts by the FIRST
// member string of the doc's combination (min_heap.rs:393-420, 900-925), member ids are in string order, so the rank is the dense rank
// of the first member id among the combinations' first members, + 1, and 0 for the empty combination (the reference panics on it; here
// it sorts below every string).  Dense, so that the ranks of a StringSet16 facet (at most 65,535 combinations) fit its 16 bits.
inline std::vector<uint32_t> string_set_sort_ranks(const uint64_t* set_offsets, const uint32_t* members, uint32_t n_sets) {
    std::vector<uint32_t> first;
    for (uint32_t c = 0; c < n_sets; c++) if (set_offsets[c + 1] > set_offsets[c]) first.push_back(members[set_offsets[c]]);
    std::sort(first.begin(), first.end()); first.erase(std::unique(first.begin(), first.end()), first.end());
    std::vector<uint32_t> rank(n_sets);
    for (uint32_t c = 0; c < n_sets; c++)
        rank[c] = set_offsets[c + 1] > set_offsets[c] ? (uint32_t)(std::lower_bound(first.begin(), first.end(), members[set_offsets[c]]) - first.begin()) + 1u : 0u;
    return rank;
}
// a sort with a POINT criterion: it needs the per-query bases and the GEO instantiation of the kernels
inline bool sort_has_point(const SortDev& s) {
    for (uint32_t j = 0; j < s.n; j++) if (s.src[j] == SORT_SRC_FACET && s.type[j] == SSB_FACET_POINT) return true;
    return false;
}

// ---- geo on the host: encode_morton_2_d and point_distance_to_morton_range (geo_search.rs:27-42, 109-144) for the filter interval.  The
// host code is compiled without FMA contraction (-ffp-contract=off); the expressions hold no multiply-add anyway.
#define SSB_DEG2RAD 0.017453292519943295
inline int32_t rust_as_i32(double v) {                             // Rust `f64 as i32`: truncation, saturating, NaN -> 0
    if (v != v) return 0;
    if (v >= 2147483648.0) return INT32_MAX;
    if (v <= -2147483648.0) return INT32_MIN;
    return (int32_t)v;
}
inline uint64_t morton_spread(uint32_t v) {                         // encode_morton_64_bit (geo_search.rs:11-20)
    uint64_t x = v;
    x = (x | (x << 16)) & 0x0000FFFF0000FFFFull;
    x = (x | (x << 8)) & 0x00FF00FF00FF00FFull;
    x = (x | (x << 4)) & 0x0F0F0F0F0F0F0F0Full;
    x = (x | (x << 2)) & 0x3333333333333333ull;
    x = (x | (x << 1)) & 0x5555555555555555ull;
    return x;
}
inline uint64_t encode_morton_2d(double lat, double lon) {
    return morton_spread((uint32_t)rust_as_i32(lat * 10000000.0)) | (morton_spread((uint32_t)rust_as_i32(lon * 10000000.0)) << 1);
}
inline double earth_radius(uint64_t unit) { return unit == SSB_UNIT_MILES ? 3958.761315801475 : 6371.0087714; }

// Facet filter i of a batch, on a facet of type `type` -> *out in key space.  set_values: the batch's filter_set_values.  A SET filter keeps
// its values where they are (out->set_first = f.set_first); a POINT filter appends its payload (GEO_WORDS f64 words) to geo and
// out->set_first is its index there — the caller rebases it once it knows where the payloads go.  A SET filter on a StringSet facet
// (n_sets / n_values: its string sets, n_sets = 0: none given) appends its MEMBERS payload to geo the same way; the caller sets lo / hi.
// Returns SSB_OK or an SSB_E_* code with set_error called.
inline int32_t encode_filter(const ssb_facet_filter& f, uint32_t i, uint32_t type, const uint64_t* set_values, FiltDev* out,
                             std::vector<uint64_t>& geo, uint32_t n_sets = 0, uint32_t n_values = 0) {
    FiltDev d{}; d.facet = f.facet;
    if ((f.kind == SSB_FILTER_POINT) != (type == SSB_FACET_POINT)) { set_error("facet filter %u: a Point facet takes SSB_FILTER_POINT and only it", i); return SSB_E_INVALID; }
    if (f.kind == SSB_FILTER_POINT) {
        // FilterSparse::Point(base, start..end, unit, point_distance_to_morton_range(base, end, unit)) (search.rs:2712-2723)
        if (f.set_count != 3) { set_error("facet filter %u: SSB_FILTER_POINT takes 3 filter_set_values (lat, lon, unit), not %u", i, f.set_count); return SSB_E_INVALID; }
        if (!set_values) { set_error("facet filter %u: null filter_set_values", i); return SSB_E_INVALID; }
        const uint64_t* p = set_values + f.set_first;
        if (p[2] > SSB_UNIT_MILES) { set_error("facet filter %u: bad distance unit %llu", i, (unsigned long long)p[2]); return SSB_E_INVALID; }
        double lat, lon, start, end; memcpy(&lat, &p[0], 8); memcpy(&lon, &p[1], 8); memcpy(&start, &f.start, 8); memcpy(&end, &f.end, 8);
        const double r = earth_radius(p[2]);
        const double lat_delta = end / (SSB_DEG2RAD * r);
        const double lon_delta = end / (SSB_DEG2RAD * r * cos(SSB_DEG2RAD * lat));
        d.lo = encode_morton_2d(lat - lat_delta, lon - lon_delta);
        d.hi = encode_morton_2d(lat + lat_delta, lon + lon_delta);
        // an empty interval (a box across latitude / longitude 0, a NaN anywhere) or a NaN start: no doc passes
        d.kind = d.lo < d.hi && start == start ? FILT_POINT : FILT_NEVER;
        d.set_first = (uint32_t)geo.size();
        uint64_t rb; memcpy(&rb, &r, 8);
        for (uint64_t w : {p[0], p[1], f.start, f.end, rb}) geo.push_back(w);
    } else if (f.kind == SSB_FILTER_RANGE) {
        if (facet_is_string(type) || facet_is_stringset(type)) { set_error("facet filter %u: a String facet takes SSB_FILTER_SET", i); return SSB_E_INVALID; }
        d.kind = FILT_RANGE;
        if (facet_is_float(type)) {
            double a, b; memcpy(&a, &f.start, 8); memcpy(&b, &f.end, 8);
            if (a != a || b != b) d.kind = FILT_NEVER; else { d.lo = f64_order_key(a); d.hi = f64_order_key(b); }
        } else if (facet_is_signed(type)) { d.lo = f.start ^ 0x8000000000000000ull; d.hi = f.end ^ 0x8000000000000000ull; }
        else { d.lo = f.start; d.hi = f.end; }
    } else if (f.kind == SSB_FILTER_SET && facet_is_stringset(type)) {
        // FilterSparse::String16 / 32 of combination ids (search.rs:2643-2710), kept as the member ids and flagged combination ids the
        // host resolved the strings to: sorted and unique, so that the device test is one binary search per member of the doc
        if (f.set_count && !set_values) { set_error("facet filter %u: null filter_set_values", i); return SSB_E_INVALID; }
        if (!n_sets) { set_error("facet filter %u: a StringSet facet needs its string sets (ssb_set_facet_string_sets)", i); return SSB_E_STATE; }
        std::vector<uint64_t> flagged, members;
        for (uint32_t j = 0; j < f.set_count; j++) {
            const uint64_t x = set_values[f.set_first + j];
            if (x & SSB_SET_COMBINATION) {
                if ((x & ~SSB_SET_COMBINATION) >= n_sets) { set_error("facet filter %u: combination id %llu of %u", i, (unsigned long long)(x & ~SSB_SET_COMBINATION), n_sets); return SSB_E_INVALID; }
                flagged.push_back(x & ~SSB_SET_COMBINATION);
            } else {
                if (x >= n_values) { set_error("facet filter %u: member id %llu of %u", i, (unsigned long long)x, n_values); return SSB_E_INVALID; }
                members.push_back(x);
            }
        }
        for (auto* v : {&flagged, &members}) { std::sort(v->begin(), v->end()); v->erase(std::unique(v->begin(), v->end()), v->end()); }
        d.kind = FILT_MEMBERS;
        d.set_first = (uint32_t)geo.size(); d.set_n = (uint32_t)(1 + flagged.size() + members.size());
        geo.push_back(flagged.size());
        geo.insert(geo.end(), flagged.begin(), flagged.end());
        geo.insert(geo.end(), members.begin(), members.end());
    } else if (f.kind == SSB_FILTER_SET) {
        if (!facet_is_string(type)) { set_error("facet filter %u: SSB_FILTER_SET needs a String16 / String32 facet", i); return SSB_E_INVALID; }
        if (f.set_count && !set_values) { set_error("facet filter %u: null filter_set_values", i); return SSB_E_INVALID; }
        d.kind = FILT_SET; d.set_first = f.set_first; d.set_n = f.set_count;
    } else { set_error("facet filter %u: bad kind %u", i, f.kind); return SSB_E_INVALID; }
    *out = d;
    return SSB_OK;
}

// ---- facet counts (ssb_search_lexical_facets; facet_count, add_result.rs:487-640) ----
// One request of a facet count call in key space.  VALUES: n_bins = the facet's largest id + 1, one histogram bin per id.  RANGES: n_bins =
// n_ranges; the starts' keys are staged at start_first of the call's start array, a doc's bin is the last start <= its key.  POINT: a RANGES
// request on a POINT facet, binned by f64_order_key of the distance to base point_idx of the query (radius: earth_radius(unit)).
// is_float: F32 / F64 (a NaN value, key ~0, is not counted).  hist_off / out_off / point_idx are set by the caller once it knows the layout.
enum { FREQ_VALUES = 0, FREQ_RANGES = 1, FREQ_POINT = 2 };
// A VALUES request on a StringSet facet bins under member ids: n_bins = n_values, and the prefix interval is one of member ids; a doc adds
// one to the bin of every member occurrence of its combination (the kernels take the facet's CSR next to the request).
struct FacetReqDev {
    uint32_t facet, kind, n_bins, is_float;
    uint32_t start_first, point_idx, hist_off, out_off;
    uint32_t length, has_prefix, rank_lo, rank_hi;
    double radius;
};
// Request i of a call on a facet of type `type` -> *out, its starts' keys appended to `starts`.  has_order: the facet has a value order
// (ssb_set_facet_value_order; a StringSet facet: its string sets); max_key: its largest column key (a StringSet facet: n_values - 1, the
// largest member id); has_bases: the call carries POINT bases.  Returns SSB_OK or an SSB_E_* code
// with set_error called.
inline int32_t encode_facet_request(const ssb_facet_request& r, uint32_t i, uint32_t type, bool has_order, uint64_t max_key, bool has_bases,
                                    FacetReqDev* out, std::vector<uint64_t>& starts) {
    FacetReqDev d{}; d.facet = r.facet;
    if (facet_is_stringset(type)) {
        if (r.kind == SSB_FACET_COUNT_RANGES) { set_error("facet request %u: a StringSet facet takes SSB_FACET_COUNT_VALUES", i); return SSB_E_INVALID; }
        if (r.kind == SSB_FACET_COUNT_VALUES && !has_order) { set_error("facet request %u: a StringSet facet needs its string sets (ssb_set_facet_string_sets)", i); return SSB_E_STATE; }
    }
    if (r.kind == SSB_FACET_COUNT_VALUES) {
        if (!facet_is_string(type) && !facet_is_stringset(type)) { set_error("facet request %u: SSB_FACET_COUNT_VALUES needs a String16 / String32 facet", i); return SSB_E_INVALID; }
        if (r.length > SSB_MAX_FACET_LENGTH) { set_error("facet request %u: length %u above %u", i, r.length, SSB_MAX_FACET_LENGTH); return SSB_E_UNSUPPORTED; }
        if (r.has_prefix && !has_order) { set_error("facet request %u: a prefix needs the facet's value order (ssb_set_facet_value_order)", i); return SSB_E_STATE; }
        if (r.has_prefix && r.rank_lo > r.rank_hi) { set_error("facet request %u: rank_lo %u above rank_hi %u", i, r.rank_lo, r.rank_hi); return SSB_E_INVALID; }
        d.kind = FREQ_VALUES; d.n_bins = (uint32_t)(max_key + 1); d.length = r.length;
        d.has_prefix = r.has_prefix ? 1u : 0u; d.rank_lo = r.rank_lo; d.rank_hi = r.rank_hi;
    } else if (r.kind == SSB_FACET_COUNT_RANGES) {
        if (facet_is_string(type)) { set_error("facet request %u: a String facet takes SSB_FACET_COUNT_VALUES", i); return SSB_E_INVALID; }
        if (r.n_ranges == 0) { set_error("facet request %u: no ranges", i); return SSB_E_INVALID; }
        if (r.n_ranges > SSB_MAX_FACET_RANGES) { set_error("facet request %u: %u ranges, at most %u", i, r.n_ranges, SSB_MAX_FACET_RANGES); return SSB_E_UNSUPPORTED; }
        if (!r.range_starts) { set_error("facet request %u: null range_starts", i); return SSB_E_INVALID; }
        const bool point = type == SSB_FACET_POINT;
        if (point) {
            if (r.unit > SSB_UNIT_MILES) { set_error("facet request %u: bad distance unit %u", i, r.unit); return SSB_E_INVALID; }
            if (!has_bases) { set_error("facet request %u: a Point facet needs the queries' bases", i); return SSB_E_INVALID; }
            d.radius = earth_radius(r.unit);
        }
        d.kind = point ? FREQ_POINT : FREQ_RANGES; d.n_bins = r.n_ranges; d.is_float = facet_is_float(type) ? 1u : 0u;
        d.start_first = (uint32_t)starts.size();
        for (uint32_t j = 0; j < r.n_ranges; j++) {
            uint64_t key = r.range_starts[j];
            if (point || facet_is_float(type)) {
                double x; memcpy(&x, &key, 8);
                if (x != x) { set_error("facet request %u: range start %u is NaN", i, j); return SSB_E_INVALID; }
                key = f64_order_key(x);
            } else if (facet_is_signed(type)) key ^= 0x8000000000000000ull;
            if (j && key <= starts.back()) { set_error("facet request %u: range starts must ascend strictly (start %u)", i, j); return SSB_E_INVALID; }
            starts.push_back(key);
        }
    } else { set_error("facet request %u: bad kind %u", i, r.kind); return SSB_E_INVALID; }
    *out = d;
    return SSB_OK;
}

}  // namespace ssb

// The rest owns device memory: nvcc translation units only.
#ifdef __CUDACC__
#include <cuda_runtime.h>

namespace ssb {

// device-resident facet columns of an index (api.cu owns it, the lexical view borrows it; facets.cu)
// zones: per facet and 65536-doc block of doc ids (block b = doc ids (zone_block0 + b) << 16 ..), the min and the max key of the block's rows
// — the column key, or for a String facet with a value order the rank of the id; sorted searches bound a level's sort key with them.
// rank / n_rank: the value order of a String facet (ssb_set_facet_value_order); max_key: the largest column key (host copy)
struct FacetSet {
    uint64_t* d_keys = nullptr; uint64_t n_rows = 0; uint32_t first_doc = 0; uint32_t n_facets = 0; uint8_t types[16] = {0};
    uint64_t* d_zones = nullptr; uint32_t zone_block0 = 0, n_zone_blocks = 0;   // [n_facets][n_zone_blocks][2] {min, max}
    uint32_t* d_rank[16] = {}; uint32_t n_rank[16] = {}; uint64_t max_key[16] = {};
    // StringSet facets (ssb_set_facet_string_sets): the CSR of the combinations' member ids, n_sets / n_values (0: not given), and the
    // member occurrences over every row (the members a pass over all rows reads); d_rank holds the combinations' first-member ranks
    uint64_t* d_set_off[16] = {}; uint32_t* d_set_mem[16] = {}; uint32_t n_sets[16] = {}, n_values[16] = {}; uint64_t member_rows[16] = {};
    // ssb_set_facets after the caller's synchronisation: drops the old columns, validates and keys the rows, computes max_key and the zones
    int32_t set_columns(const void* rows, uint64_t first_doc_id, uint64_t n_docs, uint32_t row_bytes, const ssb_facet_field* fields,
                        uint32_t n_fields, cudaStream_t st);
    // ssb_set_facet_value_order after its checks: the rank of every id of String facet `facet`, and that facet's zones in ranks
    int32_t set_value_order(uint32_t facet, const uint32_t* rank_of_id, uint32_t n_ids, cudaStream_t st);
    // ssb_set_facet_string_sets after its argument checks: validates the ids, uploads the CSR, derives the sort ranks and the zones
    int32_t set_string_sets(uint32_t facet, const uint64_t* set_offsets, const uint32_t* members, uint32_t n_sets, uint32_t n_values, cudaStream_t st);
    void release() {
        cudaFree(d_keys); d_keys = nullptr; n_rows = 0; n_facets = 0;
        cudaFree(d_zones); d_zones = nullptr; n_zone_blocks = 0;
        for (int f = 0; f < 16; f++) {
            cudaFree(d_rank[f]); d_rank[f] = nullptr; n_rank[f] = 0;
            cudaFree(d_set_off[f]); d_set_off[f] = nullptr; cudaFree(d_set_mem[f]); d_set_mem[f] = nullptr;
            n_sets[f] = 0; n_values[f] = 0; member_rows[f] = 0;
        }
    }
};

// ssb_search_lexical_sorted's criteria against the facets (fs: null = none set) -> *out; *sorted = false: they reduce to "_score desc".
// has_bases: the call carries POINT bases (else a POINT criterion is dropped).  The caller checks that the facet rows cover its levels.
int32_t sort_of_criteria(const FacetSet* fs, const ssb_sort_criterion* crit, uint32_t n, bool has_bases, SortDev* out, bool* sorted);

}  // namespace ssb
#endif  // __CUDACC__
