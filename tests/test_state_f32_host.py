"""StateTransformedEnv(env; state_mapping = s -> Float32.(s)) on the device source compiled for the host (no GPU).

The Float32 mirror a Float64 env keeps for the learners (csrc/env_device.cuh: store_obs_f32, written behind the Float64 observation
by every env kernel) must be the round-to-nearest of the env's own Float64 observation: np.float32 of the oracle's state(env) along
seeded trajectories, auto-resets included, for all five Float64 variants the learners take, and for Pendulum angles far outside
[-pi, pi] (sin / cos through the Float64 rem_pio2 tree, then rounded)."""
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
#include <vector>
#include "env_device.cuh"
using namespace envdev;
// state: (n, NS) doubles, one env's state contiguous (the device layout); out: the (NOBS, n) Float32 mirror
template <class Env> static int mirror(const double* state, int64_t n, float* out) {
    static_assert(HasObsF32<Env>::value, "a Float64 env with a mirror");
    std::vector<double> buf((size_t)n * Env::NOBS * 2);   // the observation, then the mirror behind it (half as many bytes)
    EnvArrays a{};
    a.obs = buf.data();
    for (int64_t i = 0; i < n; ++i) store_obs_f32<Env>(a, i, n, Env::load(state, i));
    const float* m = obs_f32<Env>(a, n);
    for (int64_t k = 0; k < n * Env::NOBS; ++k) out[k] = m[k];
    return Env::NOBS;
}
extern "C" int hd_obs_f32(int variant, const double* state, int64_t n, float* out) {
    static_assert(!HasObsF32<CartPoleD<float>>::value && !HasObsF32<AcrobotD>::value, "Float32 envs and Acrobot keep no mirror");
    switch (variant) {
        case 0: return mirror<CartPoleD<double, false>>(state, n, out);
        case 1: return mirror<PendulumD<true, double>>(state, n, out);
        case 2: return mirror<PendulumD<false, double>>(state, n, out);
        case 3: return mirror<MountainCarD<false, double>>(state, n, out);
        case 4: return mirror<MountainCarD<true, double>>(state, n, out);
    }
    return -1;
}
"""


@pytest.fixture(scope="module")
def hd(tmp_path_factory):
    d = tmp_path_factory.mktemp("state_f32")
    src, so = d / "state_f32_driver.cpp", d / "libstatef32.so"
    src.write_text(DRIVER)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-Wno-unknown-pragmas",
                           "-I", HD, "-I", CSRC, "-shared", "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    L.hd_obs_f32.restype, L.hd_obs_f32.argtypes = C.c_int, [C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    return L


# (hostdev variant, oracle kind, discrete action count or None, action bound)
VARIANTS = [
    pytest.param(0, O.KIND_CARTPOLE, 2, None, id="CartPole-f64"),
    pytest.param(1, O.KIND_PENDULUM, None, 2.0, id="Pendulum-f64-continuous"),
    pytest.param(2, O.KIND_PENDULUM, 3, None, id="Pendulum-f64-discrete"),
    pytest.param(3, O.KIND_MOUNTAINCAR, 3, None, id="MountainCar-f64"),
    pytest.param(4, O.KIND_MOUNTAINCAR_CONT, None, 1.0, id="MountainCar-f64-continuous"),
]


def _oracle(okind, variant, n, seeds):
    params = None
    if variant == 2:
        params = O.default_params(O.KIND_PENDULUM, "f64").copy()
        params[8] = 0
    return O.OracleVecEnv(okind, n, seeds, dtype="f64", params=params)


def _mirror(hd, variant, ref):
    state = np.ascontiguousarray(ref.get(O.F_STATE), np.float64)
    n = state.shape[0]
    out = np.empty(n * 4, np.float32)
    nobs = hd.hd_obs_f32(variant, O._p(state), n, O._p(out))
    return out[: n * nobs].reshape(n, nobs)


def _same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a, np.float32).view(np.uint32), np.ascontiguousarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize("variant,okind,n_act,bound", VARIANTS)
def test_mirror_is_float32_of_the_float64_observation(hd, variant, okind, n_act, bound):
    n, steps = 700, 430                                      # > 2 episodes of 200 steps: auto-resets inside the trajectory
    seeds = O.splitmix_states_fast(n, 901 + variant)
    ref = _oracle(okind, variant, n, seeds)
    ref.reset(force=True)
    r = np.random.default_rng(variant)
    assert _same_bits(_mirror(hd, variant, ref), ref.get(O.F_OBS).astype(np.float32)), "after reset"
    resets = 0
    for k in range(steps):
        if n_act:
            a = r.integers(1, n_act + 1, n).astype(np.int32)
        elif okind == O.KIND_PENDULUM:
            a = np.where(np.arange(n) % 2 == 0, bound, r.uniform(-bound, bound, n))   # full torque one way: theta winds up
        else:
            a = r.uniform(-bound, bound, n)
        assert ref.step(a, auto_reset=True) == 0
        resets += int((ref.get(O.F_FLAGS) & 2).astype(bool).sum())
        assert _same_bits(_mirror(hd, variant, ref), ref.get(O.F_OBS).astype(np.float32)), k
    assert resets >= n                                       # every env went through an auto-reset
    if okind == O.KIND_PENDULUM:
        assert np.abs(ref.get(O.F_STATE)[:, 0]).max() > 4 * np.pi


def test_pendulum_far_angles_and_non_finite_values(hd):
    """theta up to 1e6 rad (the rem_pio2 paths of the Float64 sin / cos) and NaN / +-Inf, which pass through the rounding"""
    n = 4096
    seeds = O.splitmix_states_fast(n, 77)
    ref = _oracle(O.KIND_PENDULUM, 1, n, seeds)
    r = np.random.default_rng(3)
    th = np.concatenate([r.uniform(-1e6, 1e6, n // 4), r.uniform(-200, 200, n // 4), r.uniform(-4, 4, n // 4),
                         np.pi / 2 * r.integers(-4000, 4000, n // 4)])
    st = np.stack([th, r.uniform(-8, 8, n)], axis=1)
    ref.set(O.F_STATE, st)
    assert ref.step(r.uniform(-2, 2, n), auto_reset=False) == 0    # (the oracle writes state(env) on a step)
    assert _same_bits(_mirror(hd, 1, ref), ref.get(O.F_OBS).astype(np.float32))
    assert np.abs(ref.get(O.F_STATE)[:, 0]).max() > 1e5
    special = np.array([[np.nan, 1.0], [np.inf, -np.inf], [0.5, np.nan], [-np.inf, np.inf]], np.float64)
    out = np.empty(4 * 4, np.float32)
    hd.hd_obs_f32(1, O._p(np.ascontiguousarray(special)), 4, O._p(out))
    m = out[:12].reshape(4, 3)
    assert np.isnan(m[0, :2]).all() and m[0, 2] == 1.0                 # sin / cos of NaN
    assert np.isnan(m[1, :2]).all() and m[1, 2] == -np.inf              # sin / cos of Inf are NaN; thetadot passes through
    assert np.isnan(m[2, 2]) and m[3, 2] == np.inf
    cp = np.array([[np.nan, np.inf, -np.inf, 1e300], [-1e-300, 3.4028235677973366e38, -0.0, 1.0]], np.float64)
    out = np.empty(2 * 4, np.float32)
    hd.hd_obs_f32(0, O._p(np.ascontiguousarray(cp)), 2, O._p(out))
    with np.errstate(over="ignore"):
        assert _same_bits(out, cp.astype(np.float32).ravel())            # overflow -> Inf, underflow -> -0, round to nearest
