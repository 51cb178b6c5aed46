"""The greedy head (csrc/greedy.cuh), compiled for the host, against a NumPy restatement of Julia's findmax (no GPU).

findmax is a left-to-right reduction in Base.isless order: the first maximum wins, NaN ranks above every number (the first NaN
wins) and -0.0 ranks below 0.0.  The same header is what evaluate_tc_kernel and the staged greedy selection run."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
HD = os.path.join(HERE, "hostdev")
CSRC = os.path.join(os.path.dirname(HERE), "reinforcementlearning.jl_b200", "csrc")

DRIVER = r"""
#include <cuda_runtime.h>
#include "greedy.cuh"
struct Desc { int nout, heads2; };
extern "C" int hd_findmax(const float* v, int n) {
    float z[16] = {};
    for (int i = 0; i < n; ++i) z[i] = v[i];
    return greedy::findmax_index(z, n);
}
extern "C" unsigned hd_greedy(int nout, int heads2, const float* v) {
    float z[4] = {v[0], v[1], v[2], v[3]};
    return greedy::greedy_action(Desc{nout, heads2}, z);
}
"""


@pytest.fixture(scope="module")
def gh(tmp_path_factory):
    d = tmp_path_factory.mktemp("greedy")
    src, so = d / "greedy_driver.cpp", d / "libgreedy.so"
    src.write_text(DRIVER)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wno-unknown-pragmas",
                           "-I", HD, "-I", CSRC, "-shared", "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    L.hd_findmax.restype, L.hd_findmax.argtypes = C.c_int, [C.c_void_p, C.c_int]
    L.hd_greedy.restype, L.hd_greedy.argtypes = C.c_uint, [C.c_int, C.c_int, C.c_void_p]
    return L


def _isless(a, b):
    """Base.isless(::Float32, ::Float32)"""
    if np.isnan(a):
        return False
    if np.isnan(b):
        return True
    if a == b:
        return bool(np.signbit(a)) and not np.signbit(b)
    return bool(a < b)


def _findmax(v):
    best = 0
    for i in range(1, len(v)):
        if _isless(v[best], v[i]):
            best = i
    return best


def _call(gh, v):
    v = np.ascontiguousarray(v, np.float32)
    return gh.hd_findmax(v.ctypes.data_as(C.c_void_p), v.size)


EDGE = [
    [1.0, 1.0], [2.0, 5.0, 5.0, 1.0], [3.0, 3.0, 3.0],                              # ties: the first maximum
    [np.nan, 1.0, 2.0], [1.0, np.nan, 2.0], [1.0, 2.0, np.nan], [np.nan, np.nan],    # NaN first / later / all
    [1.0, np.nan, np.nan, 5.0], [np.inf, np.nan], [np.nan, np.inf],
    [-np.inf, -np.inf], [-np.inf, 0.0], [np.inf, np.inf, 1.0], [-1.0, np.inf, np.inf],
    [-0.0, 0.0], [0.0, -0.0], [-0.0, -0.0, 0.0, 0.0], [-0.0, -1.0], [-1.0, -0.0, 0.0],
    [5.0], [np.nan], [-0.0],
]


@pytest.mark.parametrize("v", EDGE, ids=[str(e) for e in EDGE])
def test_findmax_edge_cases(gh, v):
    assert _call(gh, v) == _findmax(np.float32(v))


def test_findmax_isless_order_spelled_out(gh):
    """the rules themselves, not only agreement with the restatement"""
    assert _call(gh, [1.0, 1.0]) == 0
    assert _call(gh, [1.0, np.nan, np.nan]) == 1
    assert _call(gh, [np.nan, 7.0]) == 0
    assert _call(gh, [-0.0, 0.0]) == 1 and _call(gh, [0.0, -0.0]) == 0
    assert _call(gh, [np.inf, np.nan]) == 1


def test_findmax_random_vectors(gh):
    rng = np.random.default_rng(0)
    pool = np.float32([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, np.nan, 2.5])
    for trial in range(4000):
        n = int(rng.integers(1, 17))
        if trial % 2:
            v = rng.choice(pool, n)                           # many ties, signed zeros, NaN, inf
        else:
            v = rng.standard_normal(n).astype(np.float32)
        assert _call(gh, v) == _findmax(v), v


def test_greedy_action_bits(gh):
    rng = np.random.default_rng(1)
    for _ in range(2000):
        nout = int(rng.integers(1, 5))
        z = rng.standard_normal(4).astype(np.float32)
        assert gh.hd_greedy(nout, 0, z.ctypes.data_as(C.c_void_p)) == _findmax(z[:nout]) + 1     # 1-based, only the first nout
    specials = np.float32([0.0, -0.0, np.inf, -np.inf, 1e-45, -3.4e38, 123.456, np.nan])
    mus = np.concatenate([specials, rng.standard_normal(500).astype(np.float32) * 10])
    for mu in mus:
        z = np.array([mu, 7.0, 0.0, 0.0], np.float32)                  # Gaussian: (mu, raw sigma) -> mu's exact bits
        assert gh.hd_greedy(2, 1, z.ctypes.data_as(C.c_void_p)) == int(z[:1].view(np.uint32)[0])
