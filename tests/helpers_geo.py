"""Geo search (Point facets) restated for the tests with Python floats and math.cos — the C library's cos, the one the library's host
code uses for the Morton interval (never numpy's vectorised cos): encode_morton_2_d / decode_morton_2_d (geo_search.rs:11-79),
point_distance_to_morton_range (:109-144), euclidian_distance (:95-107) and simplified_distance (:82-93), each f64 operation in the
reference's order.  The filter oracle hands the docs a Point filter rejects to the C oracle as deleted docs: is_facet_filter and the delete
set both drop a doc from the top-k and from the counts (add_result.rs:3435, 3498-3500)."""
import math

import numpy as np

DEG2RAD = 0.017453292519943295
RADIUS = {0: 6371.0087714, 1: 3958.761315801475}           # DistanceUnit::Kilometers / Miles


def _cos(x):
    return math.cos(x) if math.isfinite(x) else math.nan     # C cos(+-inf) is NaN; math.cos raises


def as_i32(v):
    """Rust `f64 as i32`: truncation toward zero, saturating, NaN -> 0"""
    if v != v:
        return 0
    if v >= 2147483648.0:
        return 2147483647
    if v <= -2147483648.0:
        return -2147483648
    return int(v)


def encode(lat, lon):
    x, y = as_i32(lat * 10000000.0) & 0xFFFFFFFF, as_i32(lon * 10000000.0) & 0xFFFFFFFF
    code = 0
    for b in range(32):
        code |= ((x >> b) & 1) << (2 * b) | ((y >> b) & 1) << (2 * b + 1)
    return code


def decode(code):
    x = y = 0
    for b in range(32):
        x |= ((code >> (2 * b)) & 1) << b
        y |= ((code >> (2 * b + 1)) & 1) << b
    sx, sy = x - (1 << 32) if x >> 31 else x, y - (1 << 32) if y >> 31 else y
    return sx / 10000000.0, sy / 10000000.0


def morton_range(base, distance, unit):
    r = RADIUS[unit]
    lat_delta = distance / (DEG2RAD * r)
    c = _cos(DEG2RAD * base[0])
    lon_delta = distance / (DEG2RAD * r * c) if c != 0.0 else math.copysign(math.inf, distance) if distance == distance else math.nan
    return encode(base[0] - lat_delta, base[1] - lon_delta), encode(base[0] + lat_delta, base[1] + lon_delta)


def euclidian_distance(p1, p2, unit):
    x = DEG2RAD * (p2[1] - p1[1]) * _cos(DEG2RAD * (p1[0] + p2[0]) / 2.0)
    y = DEG2RAD * (p2[0] - p1[0])
    return RADIUS[unit] * math.sqrt(x * x + y * y)


def simplified_distance(p1, p2):
    x = (p2[1] - p1[1]) * _cos(DEG2RAD * (p1[0] + p2[0]) / 2.0)
    y = p2[0] - p1[0]
    return x * x + y * y


def filter_rejects(codes, base, start, end, unit, rel=1e-12):
    """doc indices (into codes) a FacetFilter::Point rejects, and the distances of the docs inside the Morton interval; asserts that none
    of them lies within a relative `rel` of a bound (the precision contract's condition)"""
    lo, hi = morton_range(base, end, unit)
    inside = np.nonzero((codes >= np.uint64(lo)) & (codes < np.uint64(hi)))[0] if lo < hi else np.zeros(0, dtype=np.int64)
    keep = np.zeros(len(codes), dtype=bool)
    lat, lon = decode_np(codes[inside])
    for i, a, o in zip(inside.tolist(), lat.tolist(), lon.tolist()):
        d = euclidian_distance(base, (a, o), unit)
        for b in (start, end):
            assert not (math.isfinite(b) and d == d and abs(d - b) <= rel * abs(b)), ("a doc lies at a bound", d, b)
        keep[i] = start <= d < end
    return np.nonzero(~keep)[0]


def decode_np(codes):
    """decode_morton_2_d on an array of codes (integer bit compaction, then the f64 division by 1e7) -> (lat, lon) arrays"""
    def compact(c):
        x = c & np.uint64(0x5555555555555555)
        for sh, m in ((1, 0x3333333333333333), (2, 0x0F0F0F0F0F0F0F0F), (4, 0x00FF00FF00FF00FF), (8, 0x0000FFFF0000FFFF), (16, 0xFFFFFFFF)):
            x = (x ^ (x >> np.uint64(sh))) & np.uint64(m)
        return x.astype(np.uint32).view(np.int32).astype(np.float64) / 10000000.0
    c = np.asarray(codes, dtype=np.uint64)
    return compact(c), compact(c >> np.uint64(1))


def sort_distances(docs, codes, first_doc, base):
    """simplified_distance(decode(code), base) of each doc (NaN -> +inf: it orders above every distance), with math.cos"""
    lat, lon = decode_np(codes[np.asarray(docs, dtype=np.int64) - first_doc])
    out = []
    for a, b in zip(lat.tolist(), lon.tolist()):
        d = simplified_distance((a, b), base)
        out.append(math.inf if d != d else d)
    return out


def sort_by_distance(hits, dists, descending, score_asc=False, k=None):
    """hits [(doc, score)] with their distances (sort_distances) ordered by distance (NaN above +inf), ties by score desc (asc with a
    trailing `_score` ascending criterion), then doc id asc; asserts that distinct distances of neighbouring hits in that order differ by
    more than a relative 1e-12"""
    keyed = [(dd, np.float32(s), d) for (d, s), dd in zip(hits, dists)]
    keyed.sort(key=lambda t: ((-t[0] if descending else t[0]), (t[1] if score_asc else -t[1]), t[2]))
    keyed = keyed[:k + 1] if k is not None else keyed
    for a, b in zip(keyed, keyed[1:]):
        if a[0] != b[0] and math.isfinite(a[0]) and math.isfinite(b[0]):
            assert abs(a[0] - b[0]) > 1e-12 * max(abs(a[0]), abs(b[0])), ("two hits within 1e-12", a, b)
    return [(d, float(s)) for _, s, d in keyed[:k]]
