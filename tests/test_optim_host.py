"""Host side of the optimiser step (no GPU).

csrc/optim.cuh (the clip rule and the Adam element update that clip_adam_kernel, K8 and K7's tail run) compiled for the host and
checked bit for bit against the oracle's clip_by_global_norm / adam_step: max_norm below, exactly at and above the global norm, zero
and denormal gradients, several consecutive steps carrying beta^t.  max_norm = 0 (no clipping, the DQN default) is checked against the
unclipped step: the oracle's rule would scale the gradient to zero there."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))
HD = os.path.join(HERE, "hostdev")
CSRC = os.path.join(os.path.dirname(HERE), "reinforcementlearning.jl_b200", "csrc")

DRIVER = r"""
#include <cuda_runtime.h>
#include <cstdint>
#include "optim.cuh"

// one optimiser step on n elements as the kernels run it: gn (computed by the caller, like the kernels' double sum) -> scale ->
// clipped gradient -> Adam with this step's beta^t -> beta^t advanced
extern "C" void hd_step(float* p, float* g, float* m, float* v, float* beta_t, long long n, float gn, float max_norm, float lr, float b1,
                        float b2, float eps) {
    const float sc = optim::clip_scale(gn, max_norm);
    const float bt1 = beta_t[0], bt2 = beta_t[1];
    for (long long k = 0; k < n; ++k) {
        const float gk = g[k] * sc;
        g[k] = gk;
        const optim::AdamOut a = optim::adam_update(gk, m[k], v[k], p[k], lr, b1, b2, eps, bt1, bt2);
        m[k] = a.m; v[k] = a.v; p[k] = a.p;
    }
    optim::beta_advance(beta_t, bt1, bt2, b1, b2);
}
extern "C" float hd_clip_scale(float gn, float max_norm) { return optim::clip_scale(gn, max_norm); }
"""

HYPER = dict(lr=1e-3, b1=0.9, b2=0.999, eps=1e-8)


@pytest.fixture(scope="module")
def oh(tmp_path_factory):
    d = tmp_path_factory.mktemp("optim")
    src, so = d / "optim_driver.cpp", d / "liboptim.so"
    src.write_text(DRIVER)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wno-unknown-pragmas",
                           "-I", HD, "-I", CSRC, "-shared", "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    vp, f = C.c_void_p, C.c_float
    L.hd_step.restype = None
    L.hd_step.argtypes = [vp, vp, vp, vp, vp, C.c_longlong, f, f, f, f, f, f]
    L.hd_clip_scale.restype, L.hd_clip_scale.argtypes = f, [f, f]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def global_norm(g):
    """the oracle's global norm (a double sum in element order, as the kernels' sums are for a single CTA)"""
    return O.clip_by_global_norm(g, np.inf)[1]


def header_step(oh, state, g, max_norm):
    p, m, v, bt = state
    g = np.ascontiguousarray(g, np.float32).copy()
    oh.hd_step(_p(p), _p(g), _p(m), _p(v), _p(bt), p.size, float(global_norm(g)), float(max_norm), HYPER["lr"], HYPER["b1"], HYPER["b2"],
               HYPER["eps"])
    return g


def oracle_step(state, g, max_norm):
    p, m, v, bt = state
    gc, gn = O.clip_by_global_norm(g, max_norm)
    O.adam_step(p, gc, m, v, bt, **HYPER)
    return gc, gn


def fresh(n, seed):
    rng = np.random.default_rng(seed)
    p = rng.standard_normal(n).astype(np.float32)
    return [p, np.zeros(n, np.float32), np.zeros(n, np.float32), np.array([HYPER["b1"], HYPER["b2"]], np.float32)]


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def assert_same(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(bits(x), bits(y))


def gradient(kind, n, rng):
    if kind == "normal":
        return rng.standard_normal(n).astype(np.float32)
    if kind == "zero":
        return np.zeros(n, np.float32)
    if kind == "denormal":   # |g| below 2^-126, mixed signs and exact zeros
        g = rng.integers(0, 1 << 23, n, dtype=np.uint32) | (rng.integers(0, 2, n, dtype=np.uint32) << 31)
        g[::7] = 0
        return g.view(np.float32)
    if kind == "mixed":      # large, tiny and denormal entries in one vector
        g = rng.standard_normal(n).astype(np.float32) * np.float32(1e3)
        g[1::3] = np.float32(1e-30)
        g[2::5] = np.uint32(5).view(np.float32)
        return g
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["normal", "zero", "denormal", "mixed"])
@pytest.mark.parametrize("where", ["below", "at", "above"])
def test_clip_and_adam_match_the_oracle(oh, kind, where):
    """max_norm below, exactly at and above the global norm: the clipped gradient, m, v, p and beta^t equal the oracle's bit for bit,
    over several consecutive steps (beta^t carried from step to step)."""
    rng = np.random.default_rng(7)
    n = 1000
    dev, ref = fresh(n, 1), fresh(n, 1)
    for step in range(5):
        g = gradient(kind, n, rng)
        gn = global_norm(g)
        if where == "below":
            max_norm = np.float32(0.5) * gn if gn > 0 else np.float32(0.5)
        elif where == "at":
            max_norm = gn if gn > 0 else np.float32(0.0)
        else:
            max_norm = np.float32(2.0) * gn + np.float32(1.0)
        if max_norm == 0:    # a zero gradient has norm 0: "at" would be the unclipped max_norm = 0 case, covered below
            max_norm = np.float32(1.0)
        gd = header_step(oh, dev, g, max_norm)
        gr, _ = oracle_step(ref, g, max_norm)
        assert np.array_equal(bits(gd), bits(gr)), step
        assert_same(dev, ref)
    assert np.all(np.isfinite(dev[0]))


@pytest.mark.parametrize("kind", ["normal", "zero", "denormal", "mixed"])
def test_max_norm_zero_does_not_clip(oh, kind):
    """max_norm = 0 skips the clip (the device rule; the DQN default): the step equals the oracle's Adam on the unclipped gradient."""
    rng = np.random.default_rng(11)
    n = 777
    dev, ref = fresh(n, 2), fresh(n, 2)
    for step in range(4):
        g = gradient(kind, n, rng)
        gd = header_step(oh, dev, g, np.float32(0.0))
        assert np.array_equal(bits(gd), bits(g)), step
        O.adam_step(ref[0], g, ref[1], ref[2], ref[3], **HYPER)
        assert_same(dev, ref)


def test_clip_scale_rule(oh):
    """The factor itself: 1 unless 0 < max_norm <= gn, then max_norm / max(max_norm, gn) (exactly 1 at max_norm = gn)."""
    f = oh.hd_clip_scale
    assert f(2.0, 0.5) == np.float32(0.5) / np.float32(2.0)
    assert f(2.0, 2.0) == 1.0
    assert f(2.0, 3.0) == 1.0
    assert f(2.0, 0.0) == 1.0
    assert f(0.0, 0.0) == 1.0
    assert f(float("inf"), 1.0) == 0.0
    assert f(float("nan"), 1.0) == 1.0
