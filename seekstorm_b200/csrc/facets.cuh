// facets.cuh — the device side of the facet key format (facets.h): the facet filter test, the geo distance test and the packed sort key
// of sorted batches.  Included by bm25.cu and empty_query.cu, after the lexical view (LexView) it reads.
#pragma once
#include "facets.h"

namespace ssb {

// ---- geo (Point facets, geo_search.rs): Morton decode and the two distances, every f64 operation individually rounded in the reference's
// order (Rust does not contract into FMA); cos is CUDA's double cos (documented within 2 ulp of the exact value, not bit-equal to glibc's)
// decode_morton_64_bit (geo_search.rs:44-52): the even bits of code, compacted
__device__ __forceinline__ uint32_t morton_even_bits(uint64_t code) {
    uint64_t x = code & 0x5555555555555555ull;
    x = (x ^ (x >> 1)) & 0x3333333333333333ull;
    x = (x ^ (x >> 2)) & 0x0F0F0F0F0F0F0F0Full;
    x = (x ^ (x >> 4)) & 0x00FF00FF00FF00FFull;
    x = (x ^ (x >> 8)) & 0x0000FFFF0000FFFFull;
    x = (x ^ (x >> 16)) & 0x00000000FFFFFFFFull;
    return (uint32_t)x;
}
// decode_morton_2_d (geo_search.rs:58-79): (x_u32 as i32) as f64 / 1e7 — lat from the even bits, lon from the odd bits
__device__ __forceinline__ double morton_lat(uint64_t code) { return __ddiv_rn((double)(int32_t)morton_even_bits(code), 10000000.0); }
__device__ __forceinline__ double morton_lon(uint64_t code) { return __ddiv_rn((double)(int32_t)morton_even_bits(code >> 1), 10000000.0); }
// euclidian_distance(base, decode(code), unit) (geo_search.rs:95-107): the equirectangular distance of the doc at Morton code `code` from
// (blat, blon); radius() returns the unit's earth radius.  The distance filter and the Point facet counts share it.  radius is read where
// the product needs it: the filter loads it from its payload there, and with it geo_rejects_impl keeps the code it had as one expression.
template <class Radius>
__device__ __forceinline__ double geo_distance(uint64_t code, double blat, double blon, Radius radius) {
    const double plat = morton_lat(code), plon = morton_lon(code);
    const double c = cos(__ddiv_rn(__dmul_rn(SSB_DEG2RAD, __dadd_rn(blat, plat)), 2.0));
    const double x = __dmul_rn(__dmul_rn(SSB_DEG2RAD, __dsub_rn(plon, blon)), c);
    const double y = __dmul_rn(SSB_DEG2RAD, __dsub_rn(plat, blat));
    return __dmul_rn(radius(), __dsqrt_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y))));
}
// FilterSparse::Point (add_result.rs:462-478): true = the doc is filtered OUT.  range.contains(code) on the Morton interval staged in
// [lo, hi), then distance_range.contains(euclidian_distance(base, decode(code), unit)) (geo_search.rs:95-107).  g: the staged payload
// (GEO_* words, f64 bits).  Out of line: only POINT filters reach it.
static __device__ __noinline__ bool geo_rejects_impl(uint64_t code, uint64_t lo, uint64_t hi, const uint64_t* g) {
    if (!(code >= lo && code < hi)) return true;
    const double blat = __longlong_as_double((long long)__ldg(&g[GEO_LAT])), blon = __longlong_as_double((long long)__ldg(&g[GEO_LON]));
    const double d = geo_distance(code, blat, blon, [&] { return __longlong_as_double((long long)__ldg(&g[GEO_RADIUS])); });
    const double start = __longlong_as_double((long long)__ldg(&g[GEO_START])), end = __longlong_as_double((long long)__ldg(&g[GEO_END]));
    return !(start <= d && d < end);
}
// the sort key of a POINT criterion (morton_ordering, geo_search.rs:82-93): the order key of simplified_distance(decode(code), base) — the
// F64 column key (f64_order_key: NaN = all ones, above +inf).  base: the query's (lat, lon).  Out of line: only POINT criteria reach it.
static __device__ __noinline__ uint64_t point_sort_key(uint64_t code, const double* base) {
    const double blat = __ldg(&base[0]), blon = __ldg(&base[1]);
    const double plat = morton_lat(code), plon = morton_lon(code);
    const double x = __dmul_rn(__dsub_rn(blon, plon), cos(__ddiv_rn(__dmul_rn(SSB_DEG2RAD, __dadd_rn(plat, blat)), 2.0)));
    const double y = __dsub_rn(blat, plat);
    return f64_order_key(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)));
}

// FilterSparse::String16 / 32 on a StringSet facet (add_result.rs:340-478 over the combination ids search.rs:2643-2710 resolves): true =
// the doc is filtered OUT.  key: the doc's combination id; p: the MEMBERS payload (FILT_MEMBERS); set_off / set_mem: the facet's CSR.  The
// doc passes on a flagged id equal to its combination or on one of its combination's members found in the sorted member list.  Out of
// line: only MEMBERS filters reach it.
static __device__ __noinline__ bool members_rejects_impl(uint64_t key, const uint64_t* p, uint32_t n, const uint64_t* set_off, const uint32_t* set_mem) {
    const uint32_t nflag = (uint32_t)__ldg(&p[0]);
    for (uint32_t i = 0; i < nflag; i++) if (__ldg(&p[1 + i]) == key) return false;
    const uint64_t* m = p + 1 + nflag;
    const uint32_t nm = n - 1 - nflag;
    if (nm == 0) return true;
    const uint64_t e = __ldg(&set_off[key + 1]);
    for (uint64_t j = __ldg(&set_off[key]); j < e; j++) {
        const uint64_t x = __ldg(&set_mem[j]);
        uint32_t lo = 0, hi = nm;                                      // the first listed member >= x
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(&m[mid]) < x) lo = mid + 1; else hi = mid; }
        if (lo < nm && __ldg(&m[lo]) == x) return false;
    }
    return true;
}

// is_facet_filter (add_result.rs:340-478): true = the doc is filtered OUT.  The typed range / set tests of the reference run on the
// order-preserving 64-bit keys ssb_set_facets stored per doc and facet (bounds converted the same way by the host), so one unsigned
// compare pair covers every FilterSparse range type.  filter_rejects_key is the test of one filter on one key: the column path below and
// the staged rows of the empty-query scan (empty_query.cu) share it.  sets: the batch's filter_sets.
// GEO: the batch holds a POINT or a MEMBERS filter (the out-of-line tests) — its own instantiation, so that the common one keeps its
// code and its callers their registers
template <bool GEO>
__device__ __forceinline__ bool filter_rejects_key(const FiltDev& f, uint64_t key, const uint64_t* sets) {
    if (f.kind == FILT_RANGE) return !(key >= f.lo && key < f.hi);
    if (f.kind == FILT_SET) {
        bool in = false;
        for (uint32_t s = 0; s < f.set_n; s++) in = in || __ldg(&sets[f.set_first + s]) == key;
        return !in;
    }
    if (GEO && f.kind == FILT_POINT) return geo_rejects_impl(key, f.lo, f.hi, sets + f.set_first);
    if (GEO && f.kind == FILT_MEMBERS)
        return members_rejects_impl(key, sets + f.set_first, f.set_n, reinterpret_cast<const uint64_t*>(f.lo), reinterpret_cast<const uint32_t*>(f.hi));
    return true;
}
// Out of line, by value, on the rare candidate / count path of lex_generic only.
struct FacetArgs { const uint64_t* keys; uint64_t rows; const FiltDev* filt; const uint64_t* sets; uint32_t first_doc; };
template <bool GEO>
__device__ __noinline__ bool facet_rejects_impl(FacetArgs a, uint32_t f0, uint32_t nf, uint32_t doc) {
    const uint64_t row = (uint64_t)doc - a.first_doc;
    if (doc < a.first_doc || row >= a.rows) return true;             // no facet row for this doc
    for (uint32_t i = 0; i < nf; i++) {
        const FiltDev f = a.filt[f0 + i];
        const uint64_t key = __ldg(&a.keys[(size_t)f.facet * a.rows + row]);
        if (filter_rejects_key<GEO>(f, key, a.sets)) return true;
    }
    return false;
}
template <bool GEO = false>
__device__ __forceinline__ bool facet_rejects(const LexView& v, uint32_t f0, uint32_t nf, uint32_t doc) {
    return facet_rejects_impl<GEO>(FacetArgs{v.facet_keys, v.facet_rows, v.filt, v.filt_sets, v.facet_first_doc}, f0, nf, doc);
}

// ---- sort keys (ssb_search_lexical_sorted; result_ordering_shard, min_heap.rs:574-1051) ----
// The packed sort key `hi` — the one place that knows its layout.  v[i] is criterion i's value: the facet's column key (facet_value_key;
// for a String facet already replaced by the rank of its id in the value order) or the doc id (_id).  Each is narrowed to its natural
// width (sort_width) keeping its order: unsigned values and ranks as they are, signed ones with the sign bit flipped within the width,
// F32 by the IEEE order trick on 32 bits (-0.0 already folded into +0.0, NaN = all ones: above +inf), 64-bit keys as they are; inverted
// within the width when ascending; concatenated with the first criterion most significant, left-aligned at bit 63.  Compared as one
// unsigned word, hi orders docs like the criteria compared left to right.  The 128-bit top-k key is (hi, lo), lo = pack_key(score, doc)
// with its score half inverted for `_score` ascending: ties on every criterion fall back to score desc (min_heap.rs:1043-1050), then
// doc id asc.  hi is monotone in every v[i]: packing per-criterion upper bounds bounds the key of every doc (level_sort_bound).
__device__ __forceinline__ uint64_t sort_pack_hi(const SortDev& s, const uint64_t* v) {
    uint64_t hi = 0; uint32_t used = 0;
#pragma unroll
    for (uint32_t i = 0; i < SSB_MAX_SORT_CRITERIA; i++) {
        if (i >= s.n) break;
        const uint32_t w = sort_width(s.src[i], s.type[i]);
        const uint64_t mask = w == 64 ? ~0ull : (1ull << w) - 1ull;
        uint64_t x = v[i];
        if (s.src[i] == SORT_SRC_FACET) {
            const uint32_t t = s.type[i];
            if (t == SSB_FACET_I8 || t == SSB_FACET_I16 || t == SSB_FACET_I32) x = (x & mask) ^ (1ull << (w - 1));
            else if (t == SSB_FACET_F32) {        // column key = the f64 order key of the value: back to the float, 32-bit order key
                if (x == ~0ull) x = 0xFFFFFFFFull;
                else x = ord_f32(__double2float_rn(f64_of_order_key(x)));
            }
        }
        x &= mask;
        if (!s.desc[i]) x ^= mask;
        used += w;
        hi |= x << (64 - used);
    }
    return hi;
}
// upper bound of hi over the docs of a level: per criterion the level's largest value (descending) or smallest (ascending, inverted by
// the packing) — the block's zone for a facet, level << 16 | 0xFFFF or level << 16 for _id.  A Point criterion takes the trivial bound
// (the largest key after packing): its zones hold Morton codes, not distances, and no level is skipped.  id_lo / id_hi: the smallest and
// largest doc id of the docs bounded when they are a part of the level (the empty-query scan bounds one tile of a level).
__device__ __forceinline__ uint64_t level_sort_bound(const SortDev& s, uint32_t level_id, uint32_t id_lo = 0u, uint32_t id_hi = 0xFFFFu) {
    uint64_t val[SSB_MAX_SORT_CRITERIA];
    const uint32_t b = level_id - s.zone_block0;                       // prepare_sort: the zones cover every level
#pragma unroll
    for (uint32_t i = 0; i < SSB_MAX_SORT_CRITERIA; i++) {
        val[i] = s.desc[i] ? ((uint64_t)level_id << 16 | id_hi) : ((uint64_t)level_id << 16 | id_lo);
        if (i < s.n && s.src[i] == SORT_SRC_FACET)
            val[i] = s.type[i] == SSB_FACET_POINT ? (s.desc[i] ? ~0ull : 0ull) : s.zones[((size_t)s.facet[i] * s.n_zone_blocks + b) * 2 + (s.desc[i] ? 1 : 0)];
    }
    return sort_pack_hi(s, val);
}
// doc's packed sort key for query q: the facet keys of its row (a String facet's id through its value order, a Point facet's code
// through its distance to the query's base), or its id.  key_of(i): criterion i's column key of the doc.
template <bool GEO, class KeyOf>
__device__ __forceinline__ uint64_t sort_hi_of(const SortDev& s, uint32_t doc, uint32_t q, KeyOf key_of) {
    uint64_t val[SSB_MAX_SORT_CRITERIA];
#pragma unroll
    for (uint32_t i = 0; i < SSB_MAX_SORT_CRITERIA; i++) {
        val[i] = doc;
        if (i < s.n && s.src[i] == SORT_SRC_FACET) {
            val[i] = key_of(i);
            if (s.rank[i]) val[i] = __ldg(&s.rank[i][val[i]]);          // sort_of_criteria: every id of the column has a rank
            else if (GEO && s.type[i] == SSB_FACET_POINT) val[i] = point_sort_key(val[i], s.bases + 2 * (size_t)q);
        }
    }
    return sort_pack_hi(s, val);
}
template <bool GEO>
__device__ __forceinline__ uint64_t doc_sort_hi(const LexView& v, const SortDev& s, uint32_t doc, uint32_t q) {
    const uint64_t row = (uint64_t)(doc - v.facet_first_doc);          // prepare_sort: the facet rows cover every doc of the levels
    return sort_hi_of<GEO>(s, doc, q, [&](uint32_t i) { return __ldg(&v.facet_keys[(size_t)s.facet[i] * v.facet_rows + row]); });
}

}  // namespace ssb
