"""The facet key format's host encoders (seekstorm_b200/csrc/facets.h) compiled with g++ and compared with the suite's Python
restatements: facet_value_key on every type (NaN, +-0.0, +-inf, integer extremes) against the typed order of the values, range and set
filter bounds against is_facet_filter on the typed columns (helpers_facets.numpy_pass), the Point interval and payload against
helpers_geo (NaN bases, boxes across 0, pole saturation), the refusals word for word, and the sort key widths."""
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import helpers_geo as G
from helpers_facets import facet_columns, numpy_pass, random_filters
from seekstorm_b200 import DistanceUnit, FacetFilter, Index, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "seekstorm_b200", "csrc")

# stdin, one request per line (decimal integers):
#   v TYPE RAW                                         -> facet_value_key(TYPE, the 8 little-endian bytes of RAW)
#   f TYPE I KIND FACET START END FIRST COUNT N SV...  -> encode_filter of filter I (N = 0: null filter_set_values)
#   w SRC TYPE                                         -> sort_width, facet_type_bytes
#   o BITS                                             -> f64_order_key of the f64 BITS, and the bits f64_of_order_key gives back
DRIVER = r"""
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include "facets.h"
static char g_err[512];
namespace ssb {
void set_error(const char* fmt, ...) { va_list a; va_start(a, fmt); vsnprintf(g_err, sizeof g_err, fmt, a); va_end(a); }
}
using namespace ssb;
int main() {
    char op[4];
    while (scanf("%3s", op) == 1) {
        if (op[0] == 'v') {
            unsigned t; unsigned long long raw; scanf("%u %llu", &t, &raw);
            uint8_t b[8]; memcpy(b, &raw, 8);
            printf("%llu\n", (unsigned long long)facet_value_key(t, b));
        } else if (op[0] == 'f') {
            ssb_facet_filter f{}; unsigned t, i, n; unsigned long long s, e;
            scanf("%u %u %u %u %llu %llu %u %u %u", &t, &i, &f.kind, &f.facet, &s, &e, &f.set_first, &f.set_count, &n);
            f.start = s; f.end = e;
            std::vector<uint64_t> sv(n);
            for (auto& x : sv) { unsigned long long y; scanf("%llu", &y); x = y; }
            FiltDev d{}; std::vector<uint64_t> geo(1, 7);                   // one word already staged: the payload index must follow it
            g_err[0] = 0;
            const int32_t rc = encode_filter(f, i, t, n ? sv.data() : nullptr, &d, geo);
            if (rc != SSB_OK) { printf("err %d %s\n", rc, g_err); continue; }
            printf("ok %u %u %llu %llu %u %u %zu", d.facet, d.kind, (unsigned long long)d.lo, (unsigned long long)d.hi, d.set_first, d.set_n, geo.size() - 1);
            for (size_t j = 1; j < geo.size(); j++) printf(" %llu", (unsigned long long)geo[j]);
            printf("\n");
        } else if (op[0] == 'w') {
            unsigned src, t; scanf("%u %u", &src, &t);
            printf("%u %u\n", sort_width(src, t), facet_type_bytes(t));
        } else {
            unsigned long long bits; scanf("%llu", &bits);
            double x; memcpy(&x, &bits, 8);
            const uint64_t k = f64_order_key(x);
            const double y = f64_of_order_key(k); uint64_t yb; memcpy(&yb, &y, 8);
            printf("%llu %llu\n", (unsigned long long)k, (unsigned long long)yb);
        }
    }
}
"""

M64 = (1 << 64) - 1
E_INVALID = -1                                                              # SSB_E_INVALID
TYPES = {"u8": _lib.FACET_U8, "u16": _lib.FACET_U16, "u32": _lib.FACET_U32, "u64": _lib.FACET_U64, "i8": _lib.FACET_I8,
         "i16": _lib.FACET_I16, "i32": _lib.FACET_I32, "i64": _lib.FACET_I64, "ts": _lib.FACET_TIMESTAMP, "f32": _lib.FACET_F32,
         "f64": _lib.FACET_F64, "s16": _lib.FACET_STRING16, "s32": _lib.FACET_STRING32}


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    d = tmp_path_factory.mktemp("facets")
    src, exe = d / "facets.cpp", d / "facets"
    src.write_text(DRIVER)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-Wall", "-Werror", "-Wno-unused-result", "-I", CSRC, str(src),
                           "-o", str(exe)])

    def go(lines):
        out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout.splitlines()
        assert len(out) == len(lines)
        return out
    return go


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", float(x)))[0]


def _raw(a):
    """the value's bytes as the low bytes of a u64"""
    return int.from_bytes(np.ascontiguousarray(a).tobytes().ljust(8, b"\0"), "little")


def _index(cols):
    """an Index with just the facet schema: _encode_filters needs nothing more"""
    ix = Index.__new__(Index)
    ix._facet_schema = {name: (i, TYPES[name]) for i, name in enumerate(cols)}
    return ix


def test_value_keys_keep_the_typed_order(run):
    cols, _ = facet_columns(400, 11)
    for name, c in cols.items():
        t = TYPES[name]
        if c.dtype.kind == "f":
            c = np.concatenate([c, np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, np.finfo(c.dtype).max, -np.finfo(c.dtype).max,
                                             np.finfo(c.dtype).tiny, -np.finfo(c.dtype).tiny], dtype=c.dtype)])
        elif c.dtype.kind in "iu":
            ii = np.iinfo(c.dtype)
            c = np.concatenate([c, np.array([ii.min, ii.max, 0], dtype=c.dtype)])
        keys = [int(k) for k in run([f"v {t} {_raw(x)}" for x in c])]
        for x, k in zip(c.tolist(), keys):
            if isinstance(x, float):
                want = M64 if x != x else (_bits(x + 0.0) ^ M64 if x < 0 else _bits(x + 0.0) | 1 << 63)   # +0.0: -0.0 == +0.0
            elif c.dtype.kind == "i":
                want = (x + (1 << 63)) & M64
            else:
                want = x
            assert k == want, (name, x, k, want)
        # the key order is the typed order (NaN above +inf)
        vals = [(1, 0.0) if isinstance(x, float) and x != x else (0, x) for x in c.tolist()]
        for (a, ka), (b, kb) in zip(sorted(zip(vals, keys)), sorted(zip(vals, keys))[1:]):
            assert (ka < kb) == (a < b) and (ka == kb) == (a == b), (name, a, b)
    # Point: the Morton code itself
    assert [int(k) for k in run([f"v {_lib.FACET_POINT} {G.encode(52.52, 13.405)}"])] == [G.encode(52.52, 13.405)]


def test_f64_order_key_round_trip(run):
    xs = [0.0, -0.0, 1.5, -1.5, math.inf, -math.inf, 5e-324, -5e-324, 1.7976931348623157e308, 3.4028234663852886e38]
    for x, line in zip(xs, run([f"o {_bits(x)}" for x in xs])):
        k, back = map(int, line.split())
        assert back == _bits(x + 0.0), (x, k, back)
    k, _ = map(int, run([f"o {_bits(math.nan)}"])[0].split())
    assert k == M64


def test_range_and_set_bounds_agree_with_is_facet_filter(run):
    n = 300
    cols, _ = facet_columns(n, 12)
    ix = _index(cols)
    filters = random_filters(cols, 13, 150) + [[FacetFilter("f64", -0.0, 0.0)], [FacetFilter("f32", 0.0, np.inf)],
                                               [FacetFilter("i64", -2**63, 2**63 - 1)], [FacetFilter("u64", 0, 2**64 - 1)],
                                               [FacetFilter("f32", np.nan, 1.0)], [FacetFilter("i8", 5, -5)]]
    flat = [f for fl in filters for f in fl]
    offs, arr, sv = ix._encode_filters([flat])
    assert int(offs[1]) == len(flat)
    req = [f"f {TYPES[f.field]} {i} {arr[i].kind} {arr[i].facet} {arr[i].start} {arr[i].end} {arr[i].set_first} {arr[i].set_count} "
           f"{len(sv)} " + " ".join(str(int(x)) for x in sv) for i, f in enumerate(flat)]
    names = list(cols)
    key_of = {name: [int(k) for k in run([f"v {TYPES[name]} {_raw(x)}" for x in cols[name]])] for name in names}
    n_checked = 0
    for i, (f, line) in enumerate(zip(flat, run(req))):
        st, facet, kind, lo, hi, first, cnt, ngeo = line.split()[:8]
        facet, kind, lo, hi, first, cnt = int(facet), int(kind), int(lo), int(hi), int(first), int(cnt)
        assert st == "ok" and facet == names.index(f.field) and int(ngeo) == 0, line
        if f.values is not None:
            assert (kind, first, cnt) == (1, int(arr[i].set_first), len(f.values)), line   # FILT_SET, values where they are
            continue
        nan_bound = TYPES[f.field] in (_lib.FACET_F32, _lib.FACET_F64) and (math.isnan(float(f.start)) or math.isnan(float(f.end)))
        assert kind == (2 if nan_bound else 0), line                        # FILT_NEVER / FILT_RANGE
        for d in range(n):
            passes = kind == 0 and lo <= key_of[f.field][d] < hi
            assert passes == numpy_pass(cols, [f], d), (f, d, cols[f.field][d])
            n_checked += 1
    assert n_checked > 10000


def test_point_interval_and_payload(run):
    ix = Index.__new__(Index)
    ix._facet_schema = {"loc": (1, _lib.FACET_POINT)}
    cases = [((52.52, 13.405), 0.0, 25.0, DistanceUnit.Kilometers),       # Berlin: a proper interval
             ((51.5072, -0.1276), 0.0, 100.0, DistanceUnit.Kilometers),    # London: the box crosses longitude 0, empty
             ((-0.5, 20.0), 1.0, 200.0, DistanceUnit.Miles),               # the box crosses latitude 0
             ((90.0, 10.0), 0.0, 50.0, DistanceUnit.Kilometers),           # the pole: the encode saturates
             ((math.nan, 10.0), 0.0, 10.0, DistanceUnit.Miles),            # NaN base
             ((10.0, 10.0), math.nan, 10.0, DistanceUnit.Kilometers),      # NaN start
             ((10.0, 10.0), 0.0, math.inf, DistanceUnit.Kilometers),       # end = inf
             ((-33.9, 151.2), 5.0, 80.0, DistanceUnit.Miles)]
    flat = [FacetFilter("loc", s, e, base=b, unit=u) for b, s, e, u in cases]
    offs, arr, sv = ix._encode_filters([flat])
    req = [f"f {_lib.FACET_POINT} {i} {arr[i].kind} {arr[i].facet} {arr[i].start} {arr[i].end} {arr[i].set_first} {arr[i].set_count} "
           f"{len(sv)} " + " ".join(str(int(x)) for x in sv) for i in range(len(flat))]
    saw = set()
    for (base, start, end, unit), line in zip(cases, run(req)):
        w = line.split()
        assert w[0] == "ok" and int(w[1]) == 1 and int(w[7]) == 5, line
        kind, lo, hi, first = int(w[2]), int(w[3]), int(w[4]), int(w[5])
        wlo, whi = G.morton_range(base, end, int(unit))
        assert (lo, hi) == (wlo, whi), (base, end, line)
        assert kind == (3 if lo < hi and start == start else 2), line      # FILT_POINT / FILT_NEVER
        assert first == 1                                                   # behind the word already staged
        assert [int(x) for x in w[8:]] == [_bits(base[0]), _bits(base[1]), _bits(start), _bits(end), _bits(G.RADIUS[int(unit)])], line
        saw.add(kind)
        if base == (90.0, 10.0):
            assert G.decode(hi)[1] == 2147483647 / 1e7 and G.decode(lo)[1] == -2147483648 / 1e7
    assert saw == {2, 3}


def test_refusals_word_for_word(run):
    P, S16, F64 = _lib.FACET_POINT, _lib.FACET_STRING16, _lib.FACET_F64
    FR, FS, FP = _lib.FILTER_RANGE, _lib.FILTER_SET, _lib.FILTER_POINT
    km, bad_unit = [_bits(1.0), _bits(2.0), 0], [_bits(1.0), _bits(2.0), 7]
    cases = [(f"{P} 3 {FR} 0 0 0 0 0 0", "a Point facet takes SSB_FILTER_POINT and only it"),
             (f"{F64} 4 {FP} 0 0 0 0 3 3 " + " ".join(map(str, km)), "a Point facet takes SSB_FILTER_POINT and only it"),
             (f"{P} 5 {FP} 0 0 0 0 2 3 " + " ".join(map(str, km)), "SSB_FILTER_POINT takes 3 filter_set_values (lat, lon, unit), not 2"),
             (f"{P} 6 {FP} 0 0 0 0 3 0", "null filter_set_values"),
             (f"{P} 7 {FP} 0 0 0 0 3 3 " + " ".join(map(str, bad_unit)), "bad distance unit 7"),
             (f"{S16} 8 {FR} 0 0 5 0 0 0", "a String facet takes SSB_FILTER_SET"),
             (f"{F64} 9 {FS} 0 0 0 0 1 1 4", "SSB_FILTER_SET needs a String16 / String32 facet"),
             (f"{S16} 10 {FS} 0 0 0 0 2 0", "null filter_set_values"),
             (f"{F64} 11 9 0 0 0 0 0 0", "bad kind 9")]
    for (args, msg), line in zip(cases, run([f"f {a}" for a, _ in cases])):
        assert line == f"err {E_INVALID} facet filter {args.split()[1]}: {msg}", (args, line)
    # an empty value set needs no values
    assert run([f"f {S16} 0 {FS} 2 0 0 0 0 0"]) == ["ok 2 1 0 0 0 0 0"]


def test_sort_widths(run):
    width = {_lib.FACET_U8: 8, _lib.FACET_I8: 8, _lib.FACET_U16: 16, _lib.FACET_I16: 16, _lib.FACET_STRING16: 16, _lib.FACET_U32: 32,
             _lib.FACET_I32: 32, _lib.FACET_F32: 32, _lib.FACET_STRING32: 32}
    types = list(range(_lib.FACET_POINT + 1)) + [99]
    out = run([f"w 0 {t}" for t in types] + [f"w 1 {t}" for t in (0, 13)])
    for t, line in zip(types, out):
        w, nbytes = map(int, line.split())
        assert w == width.get(t, 64), (t, line)                         # 64-bit types, Point distances (and no other type reaches it)
        assert nbytes == (0 if t == 99 else width.get(t, 64) // 8), (t, line)
    assert out[-2:] == ["32 1", "32 8"]                                   # _id: the doc id's 32 bits
