"""The C++ host mirror's empty query (include/seekstorm_b200.hpp: ssb::Index::search with enable_empty_query) compiled with g++ against
the C-ABI library and run on the reference's 4-doc fixture (tests/cpp/test_empty_query.cpp)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_empty_query.cpp")
OUT_DIR = os.path.join(ROOT, "tests", "cpp", "_build")
EXE = os.path.join(OUT_DIR, "test_empty_query")


def _build():
    os.makedirs(OUT_DIR, exist_ok=True)
    lib_dir = os.path.join(ROOT, "seekstorm_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), SRC, "-o", EXE, "-L", lib_dir,
                           "-lseekstorm_b200", f"-Wl,-rpath,{lib_dir}", "-L/usr/local/cuda/lib64", "-lcudart"])


def test_cpp_empty_query_compiles_and_fails_loudly_without_gpu():
    import torch
    _build()
    if not torch.cuda.is_available():
        r = subprocess.run([EXE], capture_output=True, text=True, timeout=120)
        assert r.returncode == 3 and "no CUDA device" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_cpp_empty_query_mirror():
    _build()
    r = subprocess.run([EXE], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout + r.stderr
