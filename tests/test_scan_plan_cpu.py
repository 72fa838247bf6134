"""plan_scan (seekstorm_b200/csrc/scan_plan.h), the one place that picks the vector scan a search runs, compiled with g++ and
compared over a grid of inputs around every boundary with the rule as DESIGN.md §3.2 states it."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "seekstorm_b200", "csrc")

DRIVER = r"""
#include <stdio.h>
#include "scan_plan.h"
using namespace ssb::vec;
int main() {
    const uint32_t nqs[] = {1, 16, 17, 128, 129, 256, 257, 384, 385, 512, 640, 1024, 4096}, ks[] = {1, 16, 17, 32};
    for (uint32_t kernel = 0; kernel <= SSB_VEC_KERNEL_TCGEN05_FILTER_N256_PAIR; kernel++)
        for (uint32_t sim = 0; sim <= SSB_SIM_EUCLIDEAN; sim++)
            for (int i8 = 0; i8 < 2; i8++)
                for (int plane = 0; plane < 2; plane++)
                    for (int paging = 0; paging < 2; paging++)
                        for (uint32_t k : ks)
                            for (uint32_t nq : nqs) {
                                const Scan s = plan_scan(kernel, sim, i8, plane, nq, k, paging);
                                printf("%u %u %d %d %d %u %u %d %u %d %d\n", kernel, sim, i8, plane, paging, k, nq, (int)s,
                                       queries_per_pass(s), is_filter(s), is_tensor_core(s));
                            }
}
"""

# the Scan enum, in declaration order
SCANS = ["Ffma", "Tf32_64", "Tf32_128", "Bf16_64", "Bf16_128", "Bf16_256", "I8_128", "F16f_128", "F16f_256", "F16f_256Pair"]
QUERIES_PER_PASS = {"Ffma": 16, "Tf32_64": 64, "Bf16_64": 64, "Bf16_256": 256, "F16f_256": 256, "F16f_256Pair": 256}   # others: 128
EUCLIDEAN = 2


def spec(kernel, sim, i8, plane, paging, k, nq):
    if i8:
        return "I8_128"
    if sim == EUCLIDEAN:
        return "Ffma"
    filterable = k <= 16 and not paging and plane
    exact = "Bf16_256" if -(-nq // 256) * 237 < -(-nq // 128) * 108 else "Bf16_128"
    if kernel == 0:
        if filterable:
            return "F16f_128" if nq <= 128 else "F16f_256"
        return "Ffma" if nq <= 16 else exact
    fixed = {1: "Ffma", 2: "Tf32_128", 3: "Tf32_64", 4: "Bf16_128", 5: "Bf16_64", 6: "Bf16_256"}
    if kernel in fixed:
        return fixed[kernel]
    if kernel == 7:
        return "F16f_128" if filterable else "Bf16_128"
    if filterable:
        return "F16f_256" if kernel == 8 else "F16f_256Pair"
    return exact


def test_plan_scan_matches_the_stated_rule(tmp_path):
    src, exe = tmp_path / "plan.cpp", tmp_path / "plan"
    src.write_text(DRIVER)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", CSRC, str(src), "-o", str(exe)])
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(lines) == 10 * 3 * 2 * 2 * 2 * 4 * 13
    seen = set()
    for line in lines:
        kernel, sim, i8, plane, paging, k, nq, s, qpp, filt, tc = map(int, line.split())
        want = spec(kernel, sim, i8, plane, paging, k, nq)
        assert SCANS[s] == want, (line, want)
        assert qpp == QUERIES_PER_PASS.get(want, 128), line
        assert filt == want.startswith("F16f") and tc == (want != "Ffma"), line
        seen.add(want)
    assert seen == set(SCANS)   # the grid reaches every variant
