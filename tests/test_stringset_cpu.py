"""Multi-value string facets (StringSet16 / StringSet32) without a GPU: the literal restatement of the reference against the numpy
formulation over the library's layout (combination ids + CSR of member ids) on random data and on a fixture of the quirks, the Python
mirror's ingest, CSR and filter resolution against the restatement, and the host encoders of seekstorm_b200/csrc/facets.h compiled with
g++ (member filters, value requests, the first-member sort ranks, refusals word for word)."""
import os
import subprocess

import numpy as np
import pytest

import helpers_stringset as S
from seekstorm_b200 import FacetFilter, Index, _lib
from seekstorm_b200.index import prefix_rank_interval, string_set_facet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "seekstorm_b200", "csrc")

# the quirks: "a_b" shares the joined key of ["a", "b"] (the first list is kept), a repeated member, empty lists, byte order "Z" < "a" < "é"
FIXTURE = [["b", "a"], ["a_b"], ["x", "x"], [], ["é", "Z", "a"], ["a"], ["a", "b"], ["x"], [], ["Z"], ["ab", "a"], ["x", "x"], ["é"]]


def _random_docs(seed, n=3000, tags=60):
    r = np.random.default_rng(seed)
    words = [f"t{i:02d}" for i in range(tags)] + ["t01_t02", "Zeta", "é", "a"]
    p = 1.0 / np.arange(1, len(words) + 1)
    p /= p.sum()
    return [[words[i] for i in r.choice(len(words), int(r.integers(0, 5)), p=p)] for _ in range(n)]


def _check_agree(docs, filters):
    values, ids = S.ingest(docs)
    single = S.single_term_ids(values)
    ss = string_set_facet(docs)
    members, offs, mem = S.csr(values)
    col = np.asarray(ids, dtype=np.int64)
    # the mirror's ingest is the restatement's
    assert ss.ids.tolist() == ids and ss.combos == [v[0] for v in values.values()]
    assert [m.decode("utf-8") for m in ss.members] == members and ss.offsets.tolist() == offs.tolist() and ss.member_ids.tolist() == mem.tolist()
    for strings in filters:
        want = S.passes(ids, S.resolve_filter(values, single, strings))
        got = S.combination_mask(offs, mem, ss.filter_values(strings))[col]
        assert (got == want).all(), strings
        # counts of the passing docs: the shard assembly vs one bincount over member occurrences
        bins = {}
        for d in np.nonzero(want)[0]:
            bins[ids[d]] = bins.get(ids[d], 0) + 1
        ref = S.member_counts(values, bins)
        cnt = S.numpy_member_counts(offs, mem, len(members), col, np.nonzero(want)[0])
        assert {members[i]: int(c) for i, c in enumerate(cnt) if c} == {k: v for k, v in ref.items() if v}
        for prefix, length in (("", 10), ("t0", 3), ("a", 1024), ("é", 5), ("zz", 4)):
            lo, hi = prefix_rank_interval(ss.members, prefix.encode("utf-8"))
            assert [(members[i], c) for i, c in S.numpy_top(cnt, lo, hi, length)] == S.top(ref, prefix, length)
    # the index-wide counts (ingest counters) are the counts over every row
    allc = S.numpy_member_counts(offs, mem, len(members), col, np.arange(len(ids)))
    assert {members[i]: int(c) for i, c in enumerate(allc) if c} == S.index_member_counts(values)
    return values, ids, ss


def test_restatements_agree_on_random_data():
    docs = _random_docs(5)
    _check_agree(docs, [["t00"], ["t01", "t03"], ["t01_t02"], ["nope"], ["é", "Zeta"], [], ["a", "t59", "t01_t02"]])


def test_fixture_quirks():
    values, ids, ss = _check_agree(FIXTURE, [["a"], ["a_b"], ["b"], ["x"], ["x_x"], [""], ["Z", "é"], ["ab"], ["a_b", "x"]])
    assert list(values) == ["a_b", "x_x", "", "Z_a_é", "a", "x", "Z", "a_ab", "é"]
    assert values["a_b"] == (["a", "b"], 3) and ids[:2] == [0, 0] and ids[6] == 0     # ["a_b"] takes the id and the list of ["b", "a"]
    assert [m.decode("utf-8") for m in ss.members] == ["Z", "a", "ab", "b", "x", "é"]   # "a_b" is never a member
    # joined keys that are no member resolve to their combination, flagged: "a_b" (held by no list), "x_x", and "" (the empty list)
    assert ss.filter_values(["a_b"]) == [C | 0] and ss.filter_values(["x_x"]) == [C | 1] and ss.filter_values([""]) == [C | 2]
    assert ss.filter_values(["a"]) == [1]                                             # ["a"]'s id holds "a": the member id suffices
    # a repeated member counts twice
    assert S.index_member_counts(values) == {"a": 6, "b": 3, "x": 5, "Z": 2, "é": 2, "ab": 1}
    # the byte order of the members and a prefix at an interval end
    order = [m.decode("utf-8") for m in ss.members]
    assert order == sorted(order, key=lambda m: m.encode("utf-8")) and order.index("Z") < order.index("a") < order.index("é")
    assert prefix_rank_interval(ss.members, "é".encode()) == (len(order) - 1, len(order))
    assert prefix_rank_interval(ss.members, b"Z") == (0, 1)


def test_sort_comparator_and_ranks(run):
    values, ids = S.ingest(FIXTURE)
    _, offs, mem = S.csr(values)
    out = run([f"k {len(offs) - 1} " + " ".join(str(int(x)) for x in offs) + " " + " ".join(str(int(x)) for x in mem)])
    rank = [int(x) for x in out[0].split()]
    n = len(values)
    for a in range(n):
        for b in range(n):
            for desc in (False, True):
                c = S.first_member_cmp(values, a, b, desc)
                want = 0 if rank[a] == rank[b] else ((1 if rank[a] > rank[b] else -1) if desc else (1 if rank[a] < rank[b] else -1))
                assert c == want, (a, b, desc)
    assert rank[list(values).index("")] == 0 and max(rank) <= n


def test_mirror_limit_and_filter_encoding():
    with pytest.raises(ValueError, match="65535 combinations"):
        string_set_facet([[f"v{i}"] for i in range(65536)], 16)
    assert len(string_set_facet([[f"v{i}"] for i in range(65535)], 16).combos) == 65535
    ix = Index.__new__(Index)
    ss = string_set_facet(FIXTURE)
    ix._facet_schema = {"tags": (0, _lib.FACET_STRINGSET16)}
    ix._string_sets = {"tags": ss}
    offs, arr, sv = ix._encode_filters([[FacetFilter("tags", values=["a", "a_b", "nope"])], [FacetFilter("tags", values=[])]])
    assert offs.tolist() == [0, 1, 2] and arr[0].kind == _lib.FILTER_SET and arr[1].kind == _lib.FILTER_SET and arr[1].set_count == 0
    assert [int(x) for x in sv[arr[0].set_first:arr[0].set_first + arr[0].set_count]] == [1, C | 0]      # "a", then "a_b"; "nope": none


# ---------------------------------------------------------------- the host encoders (g++)
# stdin, one request per line (decimal integers):
#   f TYPE KIND COUNT NSETS NVALUES SV...          -> encode_filter of filter 2 (set_first 0; COUNT values)
#   r TYPE HAS_ORDER MAX_KEY KIND LENGTH PREFIX LO HI -> encode_facet_request of request 3
#   k NSETS OFFSETS... MEMBERS...                  -> string_set_sort_ranks
#   w TYPE                                         -> sort_width, facet_type_bytes, facet_value_key of the bytes 0x01 .. 0x08
DRIVER = r"""
#include <stdarg.h>
#include <stdio.h>
#include "facets.h"
static char g_err[512];
namespace ssb {
void set_error(const char* fmt, ...) { va_list a; va_start(a, fmt); vsnprintf(g_err, sizeof g_err, fmt, a); va_end(a); }
}
using namespace ssb;
int main() {
    char op[4];
    while (scanf("%3s", op) == 1) {
        g_err[0] = 0;
        if (op[0] == 'f') {
            ssb_facet_filter f{}; unsigned t, ns, nv;
            scanf("%u %u %u %u %u", &t, &f.kind, &f.set_count, &ns, &nv);
            std::vector<uint64_t> sv(f.set_count + 1);
            for (uint32_t j = 0; j < f.set_count; j++) { unsigned long long y; scanf("%llu", &y); sv[j] = y; }
            FiltDev d{}; std::vector<uint64_t> pay(1, 7);
            const int32_t rc = encode_filter(f, 2, t, sv.data(), &d, pay, ns, nv);
            if (rc != SSB_OK) { printf("err %d %s\n", rc, g_err); continue; }
            printf("ok %u %u %u", d.kind, d.set_first, d.set_n);
            for (size_t j = 1; j < pay.size(); j++) printf(" %llu", (unsigned long long)pay[j]);
            printf("\n");
        } else if (op[0] == 'r') {
            ssb_facet_request r{}; unsigned t, ho; unsigned long long mk;
            scanf("%u %u %llu %u %u %u %u %u", &t, &ho, &mk, &r.kind, &r.length, &r.has_prefix, &r.rank_lo, &r.rank_hi);
            FacetReqDev d{}; std::vector<uint64_t> starts;
            const int32_t rc = encode_facet_request(r, 3, t, ho != 0, mk, false, &d, starts);
            if (rc != SSB_OK) { printf("err %d %s\n", rc, g_err); continue; }
            printf("ok %u %u %u %u %u %u\n", d.kind, d.n_bins, d.length, d.has_prefix, d.rank_lo, d.rank_hi);
        } else if (op[0] == 'k') {
            unsigned ns; scanf("%u", &ns);
            std::vector<uint64_t> off(ns + 1);
            for (auto& x : off) { unsigned long long y; scanf("%llu", &y); x = y; }
            std::vector<uint32_t> mem(off[ns]);
            for (auto& x : mem) scanf("%u", &x);
            for (uint32_t r : string_set_sort_ranks(off.data(), mem.data(), ns)) printf("%u ", r);
            printf("\n");
        } else {
            unsigned t; scanf("%u", &t);
            const uint8_t b[8] = {1, 2, 3, 4, 5, 6, 7, 8};
            printf("%u %u %llu\n", sort_width(SORT_SRC_FACET, t), facet_type_bytes(t), (unsigned long long)facet_value_key(t, b));
        }
    }
}
"""


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    d = tmp_path_factory.mktemp("stringset")
    src, exe = d / "drv.cpp", d / "drv"
    src.write_text(DRIVER)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-Wno-unused-result", "-I", CSRC, str(src), "-o", str(exe)])

    def go(lines):
        return subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout.splitlines()
    return go


SS16, SS32 = _lib.FACET_STRINGSET16, _lib.FACET_STRINGSET32
C = _lib.SET_COMBINATION


def test_types(run):
    assert run([f"w {SS16}", f"w {SS32}"]) == ["16 2 513", "32 4 67305985"]


def test_member_filter_payload(run):
    out = run([f"f {SS16} {_lib.FILTER_SET} 6 5 9 7 {C | 3} 2 7 {C | 1} 0",
               f"f {SS32} {_lib.FILTER_SET} 0 5 9",
               f"f {SS32} {_lib.FILTER_SET} 1 5 9 {C | 4}"])
    # kind FILT_MEMBERS (4), payload after the one word already staged: {F, flagged ascending, members ascending and unique}
    assert out == ["ok 4 1 6 2 1 3 0 2 7", "ok 4 1 1 0", "ok 4 1 2 1 4"]


@pytest.mark.parametrize("line, rc, msg", [
    (f"f {SS16} {_lib.FILTER_SET} 1 5 9 9", -1, "facet filter 2: member id 9 of 9"),
    (f"f {SS16} {_lib.FILTER_SET} 1 5 9 {C | 5}", -1, "facet filter 2: combination id 5 of 5"),
    (f"f {SS32} {_lib.FILTER_SET} 1 0 0 1", -4, "facet filter 2: a StringSet facet needs its string sets (ssb_set_facet_string_sets)"),
    (f"f {SS16} {_lib.FILTER_RANGE} 0 5 9", -1, "facet filter 2: a String facet takes SSB_FILTER_SET"),
    (f"f {SS16} {_lib.FILTER_POINT} 0 5 9", -1, "facet filter 2: a Point facet takes SSB_FILTER_POINT and only it"),
    (f"r {SS16} 1 8 {_lib.FACET_COUNT_RANGES} 0 0 0 0", -1, "facet request 3: a StringSet facet takes SSB_FACET_COUNT_VALUES"),
    (f"r {SS32} 0 8 {_lib.FACET_COUNT_VALUES} 10 0 0 0", -4, "facet request 3: a StringSet facet needs its string sets (ssb_set_facet_string_sets)"),
    (f"r {SS32} 1 8 {_lib.FACET_COUNT_VALUES} 1025 0 0 0", -5, "facet request 3: length 1025 above 1024"),
    (f"r {SS32} 1 8 {_lib.FACET_COUNT_VALUES} 10 1 5 4", -1, "facet request 3: rank_lo 5 above rank_hi 4"),
])
def test_refusals_word_for_word(run, line, rc, msg):
    assert run([line]) == [f"err {rc} {msg}"]


def test_value_requests(run):
    # n_bins = the member count (max_key = n_values - 1); the prefix interval passes through as member ids
    assert run([f"r {SS16} 1 8 {_lib.FACET_COUNT_VALUES} 10 1 2 5", f"r {SS32} 1 {(1 << 64) - 1} {_lib.FACET_COUNT_VALUES} 3 0 0 0"]) == \
        ["ok 0 9 10 1 2 5", "ok 0 0 3 0 0 0"]
