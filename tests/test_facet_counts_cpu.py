"""Facet counts without a GPU: the request encoder of seekstorm_b200/csrc/facets.h (encode_facet_request) compiled with g++ — range-start
keys on every type against the typed binning of the reference's facet_count (add_result.rs:487-640), and every refusal — and the host-side
assembly of Index.search(query_facets=...) (RangeType, labels, the label prefix, zero bins, string prefixes as value-order rank intervals,
the Topk rule) against a plain restatement of facet_count and search.rs:3598-3750 / 2038-2048."""
import math
import os
import random
import struct
import subprocess

import numpy as np
import pytest

import seekstorm_b200.index as I
from seekstorm_b200 import Index, QueryFacet, QueryType, RangeType, ResultType, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "seekstorm_b200", "csrc")

# stdin, one request per line (decimal integers):
#   r TYPE HAS_ORDER MAX_KEY HAS_BASES  KIND LENGTH HAS_PREFIX LO HI UNIT NULL_STARTS N S...  -> encode_facet_request of request 3
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
        unsigned t, has_order, has_bases, null_starts, n; unsigned long long max_key;
        ssb_facet_request r{};
        scanf("%u %u %llu %u %u %u %u %u %u %u %u %u", &t, &has_order, &max_key, &has_bases, &r.kind, &r.length, &r.has_prefix, &r.rank_lo,
              &r.rank_hi, &r.unit, &null_starts, &n);
        std::vector<uint64_t> s(n + 1);
        for (unsigned j = 0; j < n; j++) { unsigned long long y; scanf("%llu", &y); s[j] = y; }
        r.n_ranges = n; r.range_starts = null_starts ? nullptr : s.data(); r.facet = 5;
        FacetReqDev d{}; std::vector<uint64_t> starts(2, 9);             // two keys already staged: start_first must follow them
        g_err[0] = 0;
        const int32_t rc = encode_facet_request(r, 3, t, has_order != 0, max_key, has_bases != 0, &d, starts);
        if (rc != SSB_OK) { printf("err %d %s\n", rc, g_err); continue; }
        uint64_t rb; memcpy(&rb, &d.radius, 8);
        printf("ok %u %u %u %u %u %u %u %u %u %llu", d.facet, d.kind, d.n_bins, d.is_float, d.start_first, d.length, d.has_prefix, d.rank_lo,
               d.rank_hi, (unsigned long long)rb);
        for (size_t j = 2; j < starts.size(); j++) printf(" %llu", (unsigned long long)starts[j]);
        printf("\n");
    }
}
"""

M64 = (1 << 64) - 1
E_INVALID, E_STATE, E_UNSUPPORTED = -1, -4, -5
VALUES, RANGES = _lib.FACET_COUNT_VALUES, _lib.FACET_COUNT_RANGES
NP = {_lib.FACET_U8: np.uint8, _lib.FACET_U16: np.uint16, _lib.FACET_U32: np.uint32, _lib.FACET_U64: np.uint64, _lib.FACET_I8: np.int8,
      _lib.FACET_I16: np.int16, _lib.FACET_I32: np.int32, _lib.FACET_I64: np.int64, _lib.FACET_TIMESTAMP: np.int64,
      _lib.FACET_F32: np.float32, _lib.FACET_F64: np.float64}


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    d = tmp_path_factory.mktemp("facet_counts")
    src, exe = d / "facet_counts.cpp", d / "facet_counts"
    src.write_text(DRIVER)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-Wall", "-Werror", "-Wno-unused-result", "-I", CSRC, str(src),
                           "-o", str(exe)])

    def go(lines):
        out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout.splitlines()
        assert len(out) == len(lines)
        return out
    return go


def f64_bits(x):
    return struct.unpack("<Q", struct.pack("<d", float(x)))[0]


def order_key(x):
    """f64_order_key restated: -0.0 folds into +0.0, negatives flip every bit, the others set the sign bit"""
    if x == 0:
        x = 0.0
    b = f64_bits(x)
    return (~b & M64) if b >> 63 else b | (1 << 63)


def widened(t, v):
    """a range start as the ABI takes it (like SSB_FILTER_RANGE bounds)"""
    if t in (_lib.FACET_F32, _lib.FACET_F64, _lib.FACET_POINT):
        return f64_bits(v)
    return int(v) & M64


def value_key(t, v):
    if t in (_lib.FACET_F32, _lib.FACET_F64):
        return order_key(float(v))
    if t in (_lib.FACET_I8, _lib.FACET_I16, _lib.FACET_I32, _lib.FACET_I64, _lib.FACET_TIMESTAMP):
        return (int(v) & M64) ^ (1 << 63)
    return int(v)


def line(t, kind, starts=(), length=0, has_order=1, max_key=99, has_bases=0, has_prefix=0, lo=0, hi=0, unit=0, null_starts=0, raw=False):
    ws = list(starts) if raw else [widened(t, s) for s in starts]
    return " ".join(str(x) for x in ["r", t, has_order, max_key, has_bases, kind, length, has_prefix, lo, hi, unit, null_starts, len(ws), *ws])


def ok(out):
    p = out.split()
    assert p[0] == "ok", out
    return dict(facet=int(p[1]), kind=int(p[2]), n_bins=int(p[3]), is_float=int(p[4]), start_first=int(p[5]), length=int(p[6]),
                has_prefix=int(p[7]), lo=int(p[8]), hi=int(p[9]), radius=struct.unpack("<d", struct.pack("<Q", int(p[10])))[0],
                keys=[int(x) for x in p[11:]])


EXTREMES = {
    _lib.FACET_U8: [0, 1, 200, 255], _lib.FACET_U16: [0, 7, 65535], _lib.FACET_U32: [0, 5, 2**32 - 1], _lib.FACET_U64: [0, 3, 2**63, M64],
    _lib.FACET_I8: [-128, -1, 0, 127], _lib.FACET_I16: [-32768, -5, 0, 32767], _lib.FACET_I32: [-2**31, -1, 0, 2**31 - 1],
    _lib.FACET_I64: [-2**63, -1, 0, 2**63 - 1], _lib.FACET_TIMESTAMP: [-2**63, -86400, 0, 2**62],
    _lib.FACET_F32: [-math.inf, -3.5, -0.0, 1e-30, 2.5, math.inf], _lib.FACET_F64: [-math.inf, -1e300, -5e-324, 0.0, 5e-324, 1e300, math.inf],
}


@pytest.mark.parametrize("t", sorted(EXTREMES))
def test_range_start_keys_and_typed_bins(run, t):
    """the starts' keys are the column keys of the same values, and binning in key space (last start <= key) is the reference's binary
    search over the typed starts — np.searchsorted(starts, v, 'right') - 1, a value below the first start or NaN not counted"""
    starts = EXTREMES[t]
    r = ok(run([line(t, RANGES, starts)])[0])
    assert r["kind"] == 1 and r["n_bins"] == len(starts) and r["start_first"] == 2 and r["facet"] == 5
    assert r["is_float"] == (t in (_lib.FACET_F32, _lib.FACET_F64))
    assert r["keys"] == [value_key(t, s) for s in starts]
    assert r["keys"] == sorted(set(r["keys"]))
    rng = np.random.default_rng(t)
    dt = NP[t]
    if np.issubdtype(dt, np.floating):
        vals = np.concatenate([np.asarray(starts, dtype=dt), rng.normal(0, 10, 200).astype(dt), np.array([np.nan, -0.0, 0.0], dtype=dt)])
    else:
        info = np.iinfo(dt)
        vals = np.concatenate([np.asarray(starts, dtype=dt), rng.integers(info.min, info.max, 200, dtype=dt, endpoint=True)])
    typed = np.asarray(starts, dtype=dt)
    for v in vals:
        want = -1 if (np.issubdtype(dt, np.floating) and np.isnan(v)) else int(np.searchsorted(typed, v, "right")) - 1
        k = value_key(t, v) if not (np.issubdtype(dt, np.floating) and np.isnan(v)) else M64
        got = sum(1 for s in r["keys"] if s <= k) - 1
        if r["is_float"] and k == M64:
            got = -1                                                     # NaN: not counted
        assert got == want, (t, v)


def test_point_and_values(run):
    r = ok(run([line(_lib.FACET_POINT, RANGES, [0.0, 1.5, 10.0, math.inf], has_bases=1, unit=1)])[0])
    assert r["kind"] == 2 and r["keys"] == [order_key(x) for x in (0.0, 1.5, 10.0, math.inf)] and r["radius"] == 3958.761315801475
    r = ok(run([line(_lib.FACET_POINT, RANGES, [-0.0, 5.0], has_bases=1, unit=0)])[0])
    assert r["keys"][0] == order_key(0.0) and r["radius"] == 6371.0087714
    r = ok(run([line(_lib.FACET_STRING32, VALUES, length=1024, max_key=70000, has_prefix=1, lo=3, hi=9)])[0])
    assert (r["kind"], r["n_bins"], r["length"], r["has_prefix"], r["lo"], r["hi"], r["keys"]) == (0, 70001, 1024, 1, 3, 9, [])
    r = ok(run([line(_lib.FACET_STRING16, VALUES, length=0, has_order=0)])[0])   # not collected, no order needed
    assert r["length"] == 0 and r["n_bins"] == 100


@pytest.mark.parametrize("args,rc,msg", [
    (dict(t=_lib.FACET_F64, kind=RANGES, starts=[0.0, math.nan]), E_INVALID, "facet request 3: range start 1 is NaN"),
    (dict(t=_lib.FACET_F32, kind=RANGES, starts=[math.nan]), E_INVALID, "facet request 3: range start 0 is NaN"),
    (dict(t=_lib.FACET_POINT, kind=RANGES, starts=[math.nan], has_bases=1), E_INVALID, "facet request 3: range start 0 is NaN"),
    (dict(t=_lib.FACET_U32, kind=RANGES, starts=[5, 5]), E_INVALID, "facet request 3: range starts must ascend strictly (start 1)"),
    (dict(t=_lib.FACET_I32, kind=RANGES, starts=[0, -1]), E_INVALID, "facet request 3: range starts must ascend strictly (start 1)"),
    (dict(t=_lib.FACET_F64, kind=RANGES, starts=[0.0, -0.0]), E_INVALID, "facet request 3: range starts must ascend strictly (start 1)"),
    (dict(t=_lib.FACET_U8, kind=RANGES, starts=list(range(257))), E_UNSUPPORTED, "facet request 3: 257 ranges, at most 256"),
    (dict(t=_lib.FACET_U8, kind=RANGES, starts=[]), E_INVALID, "facet request 3: no ranges"),
    (dict(t=_lib.FACET_U8, kind=RANGES, starts=[1], null_starts=1), E_INVALID, "facet request 3: null range_starts"),
    (dict(t=_lib.FACET_U32, kind=VALUES, length=5), E_INVALID, "facet request 3: SSB_FACET_COUNT_VALUES needs a String16 / String32 facet"),
    (dict(t=_lib.FACET_POINT, kind=VALUES, length=5), E_INVALID, "facet request 3: SSB_FACET_COUNT_VALUES needs a String16 / String32 facet"),
    (dict(t=_lib.FACET_STRING16, kind=RANGES, starts=[0]), E_INVALID, "facet request 3: a String facet takes SSB_FACET_COUNT_VALUES"),
    (dict(t=_lib.FACET_STRING16, kind=VALUES, length=5, has_prefix=1, has_order=0), E_STATE,
     "facet request 3: a prefix needs the facet's value order (ssb_set_facet_value_order)"),
    (dict(t=_lib.FACET_STRING16, kind=VALUES, length=5, has_prefix=1, lo=4, hi=3), E_INVALID, "facet request 3: rank_lo 4 above rank_hi 3"),
    (dict(t=_lib.FACET_STRING32, kind=VALUES, length=1025), E_UNSUPPORTED, "facet request 3: length 1025 above 1024"),
    (dict(t=_lib.FACET_POINT, kind=RANGES, starts=[0.0], has_bases=0), E_INVALID, "facet request 3: a Point facet needs the queries' bases"),
    (dict(t=_lib.FACET_POINT, kind=RANGES, starts=[0.0], has_bases=1, unit=2), E_INVALID, "facet request 3: bad distance unit 2"),
    (dict(t=_lib.FACET_U8, kind=7), E_INVALID, "facet request 3: bad kind 7"),
])
def test_refusals(run, args, rc, msg):
    t = args.pop("t"); kind = args.pop("kind")
    out = run([line(t, kind, **args)])[0]
    assert out == f"err {rc} {msg}"


# ---- host assembly against a plain restatement of the reference ----
def ref_facets(values, labels_or_strings, qf, kind, matches):
    """facet_count over the matching docs + the shard assembly (search.rs:3598-3750) + Search::search's per-label sums and sort by count /
    truncation (search.rs:1932-1936, 2038-2048); ties in count by value id / range order (this library's documented order)"""
    counts = {}
    if kind == "range":
        starts = np.asarray([r[1] for r in qf.ranges], dtype=values.dtype)
        for d in matches:
            v = values[d]
            if np.issubdtype(values.dtype, np.floating) and np.isnan(v):
                continue
            i = int(np.searchsorted(starts, v, "right")) - 1
            if i >= 0:
                counts[i] = counts.get(i, 0) + 1
        if qf.range_type == RangeType.CountAboveRange:
            s = 0
            for i in sorted(counts, reverse=True):
                s += counts[i]; counts[i] = s
        elif qf.range_type == RangeType.CountBelowRange:
            s = 0
            for i in sorted(counts):
                s += counts[i]; counts[i] = s
        v = [(qf.ranges[i][0], counts[i]) for i in sorted(counts) if not qf.prefix or qf.ranges[i][0].startswith(qf.prefix)]
        return label_sums(v, 65535)
    for d in matches:
        counts[int(values[d])] = counts.get(int(values[d]), 0) + 1
    ids = sorted(counts, key=lambda i: (-counts[i], i))
    v = [(labels_or_strings[i], counts[i]) for i in ids if not qf.prefix or labels_or_strings[i].startswith(qf.prefix)][:qf.length]
    return label_sums(v, qf.length)


def label_sums(v, length):
    labels = list(dict.fromkeys(lab for lab, _ in v))
    sums = [(lab, sum(c for l2, c in v if l2 == lab)) for lab in labels]
    return sorted(sums, key=lambda x: -x[1])[:length]


def device_raw(values, strings, order, qf, kind, matches):
    """what ssb_search_lexical_facets returns for one query: every range's raw count, or the top `length` ids in the rank interval"""
    if kind == "range":
        starts = np.asarray([r[1] for r in qf.ranges], dtype=values.dtype)
        out = [0] * len(qf.ranges)
        for d in matches:
            v = values[d]
            if np.issubdtype(values.dtype, np.floating) and np.isnan(v):
                continue
            i = int(np.searchsorted(starts, v, "right")) - 1
            if i >= 0:
                out[i] += 1
        return out
    lo, hi = I.prefix_rank_interval(order, qf.prefix.encode()) if qf.prefix else (0, len(order))
    rank = {s: i for i, s in enumerate(order)}
    counts = {}
    for d in matches:
        counts[int(values[d])] = counts.get(int(values[d]), 0) + 1
    ids = [i for i in sorted(counts, key=lambda i: (-counts[i], i)) if lo <= rank[strings[i].encode()] < hi]
    return [(i, counts[i]) for i in ids[:qf.length]]


def fake_index(schema, strings):
    ix = Index.__new__(Index)
    ix._facet_schema = schema
    ix._string_values = {k: v for k, v in strings.items()}
    ix._string_order = {k: sorted(set(s.encode() for s in v)) for k, v in strings.items()}
    return ix


STRS = ["apple", "app", "apricot", "b", "banana", "app", "", "ap", "éclair", "apple", "zz", "aÿ", "ab"]


def test_prefix_rank_interval_brute_force():
    order = sorted(set(s.encode() for s in STRS))
    for p in ["", "a", "ap", "app", "apple", "appx", "b", "z", "zz", "zzz", "é", "aÿ", "ÿ", "c"]:
        lo, hi = I.prefix_rank_interval(order, p.encode())
        assert [s for s in order if s.startswith(p.encode())] == order[lo:hi], p
    assert I.prefix_rank_interval([b"a\xff", b"a\xff\xff", b"b"], b"a\xff") == (0, 2)


@pytest.mark.parametrize("seed", range(6))
def test_assembly_matches_restatement(seed):
    rng = random.Random(seed)
    n = 400
    nprng = np.random.default_rng(seed)
    price = nprng.integers(0, 100, n).astype(np.uint32)
    temp = nprng.normal(0, 10, n).astype(np.float64)
    temp[::37] = np.nan
    brand = nprng.integers(0, len(STRS), n).astype(np.uint16)
    schema = {"price": (0, _lib.FACET_U32), "temp": (1, _lib.FACET_F64), "brand": (2, _lib.FACET_STRING16)}
    ix = fake_index(schema, {"brand": STRS})
    cols = {"price": price, "temp": temp, "brand": brand}
    for _ in range(20):
        matches = sorted(rng.sample(range(n), rng.randint(0, n)))
        rt = RangeType(rng.randint(0, 2))
        qfs = [QueryFacet("price", range_type=rt, ranges=[("cheap", 10), ("mid", 40), ("mid2", 60), ("dear", 90), ("mid", 95)],
                          prefix=rng.choice(["", "mid", "x"])),
               QueryFacet("temp", range_type=rt, ranges=[("cold", -5.0), ("zero", 0.0), ("warm", 7.5)]),
               QueryFacet("brand", prefix=rng.choice(["", "a", "ap", "app", "b", "q"]), length=rng.choice([0, 1, 3, 50]))]
        raw = {}
        for qf in qfs:
            kind = "values" if qf.field == "brand" else "range"
            raw[qf.field] = device_raw(cols[qf.field], STRS, ix._string_order.get(qf.field), qf, kind, matches)
        got = ix.assemble_facets(raw, qfs)
        want = {}
        for qf in qfs:
            kind = "values" if qf.field == "brand" else "range"
            v = ref_facets(cols[qf.field], STRS, qf, kind, matches)
            if v:
                want[qf.field] = v
        assert got == want


def test_zero_bins_dropped_and_running_sums():
    ix = fake_index({"p": (0, _lib.FACET_U8)}, {})
    qf = QueryFacet("p", ranges=[("a", 0), ("b", 10), ("c", 20), ("d", 30)], range_type=RangeType.CountAboveRange)
    assert ix.assemble_facets({"p": [3, 0, 5, 1]}, [qf]) == {"p": [("a", 9), ("c", 6), ("d", 1)]}
    qf = QueryFacet("p", ranges=qf.ranges, range_type=RangeType.CountBelowRange)
    assert ix.assemble_facets({"p": [3, 0, 5, 1]}, [qf]) == {"p": [("d", 9), ("c", 8), ("a", 3)]}
    assert ix.assemble_facets({"p": [0, 0, 0, 0]}, [qf]) == {}


def test_topk_rule_and_request_shapes(monkeypatch):
    """Index.search asks for facet counts unless the effective result type is Topk (search.rs:1748); a request of the wrong shape for its
    field, or on an unknown field, is ignored; the last request on a field wins"""
    ix = fake_index({"p": (0, _lib.FACET_U32), "s": (1, _lib.FACET_STRING32)}, {"s": ["x", "y"]})
    ix.term_key_fn = lambda t: 8
    calls = []
    monkeypatch.setattr(Index, "search_lexical_batch", lambda self, *a, **k: ([[(1, 1.0)]], np.array([1], dtype=np.uint64)))

    def fake_facets(self, keys, qt, qfs, *a, **k):
        calls.append(qfs)
        return [{"p": [0, 4], "s": [(1, 4)]}]
    monkeypatch.setattr(Index, "search_lexical_facets", fake_facets)
    qfs = [QueryFacet("p", ranges=[("lo", 0), ("hi", 5)]), QueryFacet("s", length=3)]
    assert ix.search("t", result_type=ResultType.Topk, query_facets=qfs).facets == {}
    assert calls == []
    ro = ix.search("t", result_type=ResultType.TopkCount, query_facets=qfs)
    assert ro.facets == {"p": [("hi", 4)], "s": [("y", 4)]} and len(calls) == 1
    assert ix.search("t", result_type=ResultType.Count, query_facets=qfs).facets == ro.facets
    assert ix.search("t", length=0, result_type=ResultType.TopkCount, query_facets=qfs).facets == ro.facets   # length 0: Count
    with pytest.raises(NotImplementedError):
        ix.search("", query_facets=qfs)
    with pytest.raises(NotImplementedError):                      # checked before the Topk rule
        ix.search("t", result_type=ResultType.Topk, query_facets=["p"])
    from seekstorm_b200 import SearchMode
    with pytest.raises(NotImplementedError):
        ix.search("t", search_mode=SearchMode.Vector(), query_facets=qfs)
    _, n, _, meta = ix._facet_requests([QueryFacet("p", length=3), QueryFacet("s", ranges=[("a", 1)]), QueryFacet("nope", length=2),
                                        QueryFacet("s", length=1), QueryFacet("s", length=7, prefix="x")])
    assert n == 1 and meta[0][0] == "s" and meta[0][2].length == 7
