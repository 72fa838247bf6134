"""Geo search without a GPU: Morton encode / decode known answers (saturation, invalid coordinates), the test restatement (helpers_geo)
against an independent struct-level one, the reference's interval quirks, the Python mirror's encoder, and the C-ABI encoding of Point
filters and sort bases built by index.py."""
import math
import struct

import numpy as np

import helpers_geo as G
from seekstorm_b200 import DistanceUnit, FacetFilter, Index, ResultSort, SortOrder, _lib
from seekstorm_b200.index import encode_morton_2d, point_column


def _interleave(x, y):
    return sum(((x >> b) & 1) << (2 * b) | ((y >> b) & 1) << (2 * b + 1) for b in range(32))


def test_encode_decode_known_answers():
    assert G.encode(0.0, 0.0) == 0
    assert G.encode(0.5, 0.25) == _interleave(5000000, 2500000)
    assert G.decode(G.encode(0.5, 0.25)) == (0.5, 0.25)
    # negative coordinates: two's complement of the i32, decoded back through the sign
    assert G.encode(-1.0, -2.0) == _interleave((-10000000) & 0xFFFFFFFF, (-20000000) & 0xFFFFFFFF)
    assert G.decode(G.encode(-1.0, -2.0)) == (-1.0, -2.0)
    # saturation of `as i32` (lon +-250 and +-inf exceed the i32 range at 1e7 per degree) and NaN -> 0
    assert G.encode(0.0, 250.0) == _interleave(0, 0x7FFFFFFF) and G.encode(0.0, -250.0) == _interleave(0, 0x80000000)
    assert G.encode(0.0, math.inf) == _interleave(0, 0x7FFFFFFF)
    assert G.encode(0.0, -math.inf) == _interleave(0, 0x80000000)
    assert G.encode(math.nan, 1.0) == _interleave(0, 10000000)
    assert G.as_i32(250.0 * 1e7) == 2147483647 and G.as_i32(-250.0 * 1e7) == -2147483648 and G.as_i32(-1.9) == -1
    # the Python mirror (numpy) against the restatement
    r = np.random.default_rng(5)
    lat = np.concatenate([r.uniform(-90, 90, 500), [0.0, -0.0, 90.0, -90.0, math.inf, -math.inf, math.nan, 250.0, -250.0, 1e300]])
    lon = np.concatenate([r.uniform(-180, 180, 500), [0.0, 180.0, -180.0, 1.0, 2.0, 3.0, 4.0, -250.0, 250.0, -1e300]])
    got = encode_morton_2d(lat, lon)
    assert [int(c) for c in got] == [G.encode(float(a), float(b)) for a, b in zip(lat, lon)]
    # invalid coordinates are not written: the row stays 0
    col = point_column(np.stack([lat, lon], axis=1))
    ok = (lat >= -90) & (lat <= 90) & (lon >= -180) & (lon <= 180)
    assert [int(c) for c in col] == [G.encode(float(a), float(b)) if v else 0 for a, b, v in zip(lat, lon, ok)]
    assert int(point_column([[91.0, 0.0]])[0]) == 0 and int(point_column([[0.0, -180.5]])[0]) == 0


def _f(x):
    return struct.unpack("<d", struct.pack("<d", x))[0]


def test_distances_against_an_independent_restatement():
    r = np.random.default_rng(7)
    for _ in range(300):
        b = (float(r.uniform(-80, 80)), float(r.uniform(-170, 170)))
        p = (float(r.uniform(-80, 80)), float(r.uniform(-170, 170)))
        unit = int(r.integers(0, 2))
        R = 6371.0087714 if unit == 0 else 3958.761315801475
        d2r = 0.017453292519943295
        c = math.cos(_f(_f(d2r * _f(b[0] + p[0])) / 2.0))
        x = _f(_f(d2r * _f(p[1] - b[1])) * c)
        y = _f(d2r * _f(p[0] - b[0]))
        assert G.euclidian_distance(b, p, unit) == _f(R * math.sqrt(_f(_f(x * x) + _f(y * y))))
        xs = _f(_f(b[1] - p[1]) * c)
        ys = _f(b[0] - p[0])
        assert G.simplified_distance(p, b) == _f(_f(xs * xs) + _f(ys * ys))
        dist = float(r.uniform(1, 500))
        lat_d = dist / (d2r * R)
        lon_d = dist / (d2r * R * math.cos(d2r * b[0]))
        assert G.morton_range(b, dist, unit) == (G.encode(b[0] - lat_d, b[1] - lon_d), G.encode(b[0] + lat_d, b[1] + lon_d))


def test_interval_quirks():
    # London lies on longitude 0: the box of a 100 km disc crosses it, the u32-cast interval is empty (min > max) — no doc passes
    lo, hi = G.morton_range((51.5072, -0.1276), 100.0, 0)
    assert lo > hi
    # Berlin: a proper interval holding the base itself
    lo, hi = G.morton_range((52.52, 13.405), 25.0, 0)
    assert lo < G.encode(52.52, 13.405) < hi
    # a base at the pole: the longitude delta explodes and the encode saturates
    lo, hi = G.morton_range((90.0, 10.0), 50.0, 0)
    assert G.decode(hi)[1] == 2147483647 / 1e7 and G.decode(lo)[1] == -2147483648 / 1e7
    # end = inf and NaN bases: empty intervals
    lo, hi = G.morton_range((10.0, 10.0), math.inf, 0)
    assert lo >= hi
    lo, hi = G.morton_range((math.nan, 10.0), 10.0, 1)
    assert lo >= hi


def test_point_filter_and_bases_encoding():
    ix = Index.__new__(Index)
    ix._facet_schema = {"price": (0, _lib.FACET_U32), "loc": (1, _lib.FACET_POINT)}
    offs, arr, sv = ix._encode_filters([[FacetFilter("loc", 1.5, 25.0, base=(52.5, -13.25), unit=DistanceUnit.Miles)],
                                        [FacetFilter("price", 3, 9), FacetFilter("loc", 0.0, math.inf, base=(-1.0, 2.0))]])
    assert list(offs) == [0, 1, 3]
    f = arr[0]
    assert (f.facet, f.kind, f.set_first, f.set_count) == (1, _lib.FILTER_POINT, 0, 3)
    assert struct.unpack("<d", struct.pack("<Q", f.start))[0] == 1.5 and struct.unpack("<d", struct.pack("<Q", f.end))[0] == 25.0
    assert [struct.unpack("<d", struct.pack("<Q", int(x)))[0] for x in sv[:2]] == [52.5, -13.25] and int(sv[2]) == _lib.UNIT_MILES
    assert (arr[1].kind, arr[2].kind, arr[2].set_first, int(sv[5])) == (_lib.FILTER_RANGE, _lib.FILTER_POINT, 3, _lib.UNIT_KILOMETERS)
    # sort bases: the explicit per-query array, else the ResultSort base for every query, else none
    rs = [ResultSort("loc", SortOrder.Ascending, base=(1.0, 2.0))]
    assert ix._sort_bases(rs, 3).tolist() == [[1.0, 2.0]] * 3
    assert ix._sort_bases([ResultSort("loc")], 2) is None
    assert ix._sort_bases(rs, 2, [(3.0, 4.0), (5.0, 6.0)]).tolist() == [[3.0, 4.0], [5.0, 6.0]]
    crit, n = ix._sort_criteria(rs)
    assert n == 1 and (crit[0].source, crit[0].facet, crit[0].order) == (_lib.SORT_FACET, 1, _lib.SORT_ASCENDING)
