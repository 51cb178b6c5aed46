"""Host side of the dueling Q-network (no GPU).

csrc/duel.cuh (the combine the forward kernels apply to the head rows, and its backward in the DQN loss kernel) compiled for the
host, bit for bit against the NumPy restatement of networks.jl:518-522 in dueling_ref.py: n = 1, 2, 3, ties, ±0, sums that round
and large |adv|.  The oracle's MLP forward gives the head rows of the same flat vector; the hand-written dueling TD-loss backward
(the formulas the kernel implements) is checked against torch float64 autograd; b200rl_net_nparams / refusals for kind 3."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import dueling_ref as D
import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))
HD = os.path.join(HERE, "hostdev")
CSRC = os.path.join(os.path.dirname(HERE), "reinforcementlearning.jl_b200", "csrc")

DRIVER = r"""
#include <cuda_runtime.h>
// the rounded single-precision intrinsics duel.cuh spells out (g++ runs with -ffp-contract=off: each operation rounds once)
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
#include "duel.cuh"
// z (4, N) head rows -> q (4, N), rows >= n zeroed
extern "C" void hd_combine(const float* z, int n, long long N, float* q) {
    for (long long i = 0; i < N; ++i) {
        float r[4] = {z[4 * i], z[4 * i + 1], z[4 * i + 2], z[4 * i + 3]};
        duel::combine(r, n);
        for (int k = 0; k < 4; ++k) q[4 * i + k] = r[k];
    }
}
extern "C" void hd_backward(float g, int a, int n, float* dz) {
    float r[4];
    duel::backward(g, a, n, r);
    for (int k = 0; k < 4; ++k) dz[k] = r[k];
}
"""


@pytest.fixture(scope="module")
def dh(tmp_path_factory):
    d = tmp_path_factory.mktemp("duel")
    src, so = d / "duel_driver.cpp", d / "libduel.so"
    src.write_text(DRIVER)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wno-unknown-pragmas",
                           "-I", HD, "-I", CSRC, "-shared", "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    L.hd_combine.restype = None
    L.hd_combine.argtypes = [C.c_void_p, C.c_int, C.c_longlong, C.c_void_p]
    L.hd_backward.restype = None
    L.hd_backward.argtypes = [C.c_float, C.c_int, C.c_int, C.c_void_p]
    return L


def device_combine(dh, z):
    """z (n + 1, N) -> the header's Q (n, N)"""
    n, N = z.shape[0] - 1, z.shape[1]
    zz = np.zeros((N, 4), np.float32)
    zz[:, :n + 1] = np.asarray(z, np.float32).T
    q = np.full((N, 4), np.nan, np.float32)
    dh.hd_combine(zz.ctypes.data_as(C.c_void_p), n, N, q.ctypes.data_as(C.c_void_p))
    assert np.all(q[:, n:] == 0)
    return q[:, :n].T


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def check(dh, z):
    got, ref = device_combine(dh, z), D.combine(z)
    assert np.array_equal(bits(got), bits(ref)), (z, got, ref)
    return got


@pytest.mark.parametrize("n", [1, 2, 3])
def test_combine_random_bit_exact(dh, n):
    rng = np.random.default_rng(n)
    z = (rng.standard_normal((n + 1, 4096)) * 10.0 ** rng.integers(-3, 4, (n + 1, 4096))).astype(np.float32)
    check(dh, z)


def test_combine_sums_that_round(dh):
    """1/3-like advantages whose running sum and mean round: the order (0 + a1) + a2 + a3 and the divide by Float32(n) matter"""
    a = np.array([[1e8, 1.0, -1e8], [0.1, 0.2, 0.3], [1 / 3, 1 / 3, 1 / 3], [16777216.0, 1.0, 1.0]], np.float32).T
    z = np.vstack([np.float32([0.7, -0.1, 1e-3, 3.0]), a])
    q = check(dh, z)
    # (0 + 1e8) + 1 rounds back to 1e8, so the Float32 mean of {1e8, 1, -1e8} is 0, not 1/3: Q_2 = (0.7 + 1) - 0
    assert q[1, 0] == np.float32(np.float32(0.7) + np.float32(1.0))
    # a plain float32 pairwise-free left-to-right sum, not numpy's reduction order, is what the restatement follows
    s = np.float32(0)
    for v in (16777216.0, 1.0, 1.0):
        s = np.float32(s + np.float32(v))
    assert s == np.float32(16777216.0)                        # 2^24 + 1 + 1 rounds back twice


def test_combine_ties_zeros_and_large(dh):
    z = np.array([
        [0.0, 0.0, 0.0, 0.0],                                  # all +0
        [-0.0, -0.0, -0.0, -0.0],                              # all -0: the sum starts at +0f0, so μ = +0 and Q = (-0 + -0) - 0 = -0
        [1.0, 2.0, 2.0, 1.0],                                  # a tie between the first two actions
        [0.5, 3e38, 3e38, -3e38],                              # large |adv|: the running sum overflows to Inf
        [-1.0, -0.0, 0.0, -0.0],
    ], np.float32).T
    q = check(dh, z)
    assert bits(q[:, 1]).tolist() == bits(np.float32([-0.0] * 3)).tolist()
    assert q[0, 2] == q[1, 2]
    assert np.isinf(q[:, 3]).all() or np.isnan(q[:, 3]).any()


def test_n_one_is_the_value(dh):
    """one action: μ = a_1, Q_1 = (v + a_1) - a_1 (rounded, not always v)"""
    z = np.array([[1.0, 1e-8, 3.0], [1e-8, 1.0, 4.0]], np.float32)     # rows {v, a_1}, three samples
    q = check(dh, z)
    assert q.shape == (1, 3) and q[0, 0] == np.float32(1.0) and q[0, 2] == np.float32(3.0)


@pytest.mark.parametrize("n", [1, 2, 3])
def test_backward_formula(dh, n):
    dz = np.zeros(4, np.float32)
    for g in (np.float32(0.37), np.float32(-1e-3), np.float32(2.0)):
        for a in range(n):
            dh.hd_backward(g, a, n, dz.ctypes.data_as(C.c_void_p))
            gn = np.float32(g / np.float32(n))
            ref = [g] + [np.float32((g if j == a else np.float32(0)) - gn) for j in range(n)] + [0.0] * (3 - n)
            assert bits(dz).tolist() == bits(np.float32(ref)).tolist()


@pytest.mark.parametrize("n,act", [(2, 0), (3, 1), (1, 0)])
def test_oracle_forward_of_the_head_rows(n, act):
    """the oracle MLP on the reordered vector gives the head rows; the dueling Q is ``combine`` of them and equals the float64
    restatement of DuelingNetwork up to float32 rounding"""
    ns, H = 4, 64
    p = D.glorot_params(ns, H, n, 7) + np.float32(0.05) * np.random.default_rng(2).standard_normal(D.nparams(ns, H, n)).astype(np.float32)
    obs = np.asfortranarray(np.random.default_rng(3).standard_normal((ns, 300)).astype(np.float32))
    q = D.oracle_q(p, ns, H, n, act, obs)
    import torch
    ref = D._torch_net(torch.tensor(p.astype(np.float64)), ns, H, n, act)(torch.tensor(obs.T.astype(np.float64))).numpy().T
    np.testing.assert_allclose(q, ref, rtol=1e-5, atol=2e-6)
    # the value row really is Wv·h2 + bv: zero advantage weights and equal biases make Q = v for every action
    p0 = p.copy()
    trunk = H * ns + H + H * H + H
    p0[trunk + H + 1:trunk + H + 1 + n * H] = 0.0
    p0[trunk + H + 1 + n * H:] = 0.25
    q0 = D.oracle_q(p0, ns, H, n, act, obs)
    v = O.q_values(O.ac_desc(ns, H, n + 1, act), D.to_single_head(p0, ns, H, n), obs)[0]
    assert np.all(q0 == q0[:1]) and np.allclose(q0[0], v, rtol=0, atol=1e-6)


@pytest.mark.parametrize("huber,double_dqn,weighted,act,n", [(True, False, False, 0, 2), (False, False, True, 1, 3), (True, True, True, 0, 3),
                                                             (False, True, False, 1, 1)])
def test_dueling_td_backward_matches_autograd(huber, double_dqn, weighted, act, n):
    ns, H, B = 3, 64, 200
    rng = np.random.default_rng(11)
    p = D.glorot_params(ns, H, n, 5) + np.float32(0.1) * rng.standard_normal(D.nparams(ns, H, n)).astype(np.float32)
    pt = (p * np.float32(0.9)).astype(np.float32)
    s, s2 = rng.standard_normal((ns, B)).astype(np.float32), rng.standard_normal((ns, B)).astype(np.float32)
    a = rng.integers(1, n + 1, B).astype(np.int32)
    r = (3.0 * rng.standard_normal(B)).astype(np.float32)
    t = (rng.random(B) < 0.2).astype(np.uint8)
    w = rng.random(B).astype(np.float32) if weighted else None
    g, loss, td = D.dqn_loss_grad(p, pt, ns, H, n, act, s, a, r, t, s2, w, 0.99, huber, double_dqn)
    gm, lm, tdm = D.dqn_loss_grad_manual(p, pt, ns, H, n, act, s, a, r, t, s2, w, 0.99, huber, double_dqn)
    np.testing.assert_allclose(td, tdm, rtol=1e-12, atol=1e-12)
    assert loss == pytest.approx(lm, rel=1e-12)
    np.testing.assert_allclose(gm, g, rtol=1e-9, atol=1e-12)
    assert g.size == D.nparams(ns, H, n)


def test_nparams_and_refusals(pkg):
    """b200rl_net_nparams needs no device: kind 3 counts Flux.destructure's parameters; n_out = 4 and bad shapes are refused"""
    lib = pkg._lib.load()
    out = C.c_int64()
    for ns, H, n in ((4, 64, 2), (2, 128, 3), (3, 64, 1), (4, 128, 3)):
        d = pkg._lib.NetDesc(ns, H, 0, n, 3)
        assert lib.b200rl_net_nparams(C.byref(d), C.byref(out)) == pkg._lib.OK
        assert out.value == H * ns + H + H * H + H + (H + 1) + n * (H + 1) == D.nparams(ns, H, n)
        d2 = pkg._lib.NetDesc(ns, H, 0, n + 1, 2)                  # the same count as a plain Q-network with n + 1 outputs
        assert lib.b200rl_net_nparams(C.byref(d2), C.byref(out)) == pkg._lib.OK and out.value == D.nparams(ns, H, n)
    for bad, code in (((4, 64, 0, 4, 3), pkg._lib.ERR_UNSUPPORTED), ((4, 64, 0, 0, 3), pkg._lib.ERR_UNSUPPORTED),
                      ((4, 96, 0, 2, 3), pkg._lib.ERR_UNSUPPORTED), ((6, 64, 0, 2, 3), pkg._lib.ERR_UNSUPPORTED), ((4, 64, 0, 2, 4), pkg._lib.ERR_INVALID)):
        out.value = -7
        assert lib.b200rl_net_nparams(C.byref(pkg._lib.NetDesc(*bad)), C.byref(out)) == code, bad
        assert out.value == -7
    assert pkg.KIND_DUELING == 3 and pkg.KIND_DUELING in pkg.learners.Q_KINDS
