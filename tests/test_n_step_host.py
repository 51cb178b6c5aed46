"""Host side of the n-step sampler (no GPU).

csrc/nstep.cuh (the window walk sample_gather_kernel<PRIO, true> runs per batch slot) compiled for the host, bit for bit against
the NumPy restatement in nstep_ref.py on synthetic rings: wrap-around, terminals inside and at the start of a window, the
straddling entry of a forced reset, the lane head, n beyond everything available, n = 1, γ ∈ {0, 0.5, 0.99, 1} and rewards
whose sums are not representable.  The host ring model is checked against the oracle's ring through its 1-step gather."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import nstep_ref as N
import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))
HD = os.path.join(HERE, "hostdev")
CSRC = os.path.join(os.path.dirname(HERE), "reinforcementlearning.jl_b200", "csrc")

DRIVER = r"""
#include <cuda_runtime.h>
// the rounded single-precision intrinsics nstep.cuh spells out (g++ runs with -ffp-contract=off: a + b and a * b round once)
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fmul_rn(float a, float b) { return a * b; }
#include "nstep.cuh"
extern "C" void hd_window(const float* reward, const unsigned char* flag, long long lanes, long long cap, const long long* keys, long long B,
                          int n, float gamma, float* G, unsigned char* term, long long* next_slot, float* disc, int* m) {
    Ring r;
    r.ns = 1; r.lanes = lanes; r.cap = cap;
    r.reward = const_cast<float*>(reward); r.flag = const_cast<uint8_t*>(flag);
    for (long long k = 0; k < B; ++k) {
        const NStepWindow w = nstep::window(r, keys[k], n, gamma);
        G[k] = w.G; term[k] = w.terminal; next_slot[k] = w.next_slot; disc[k] = w.discount; m[k] = w.m;
    }
}
"""


@pytest.fixture(scope="module")
def nh(tmp_path_factory):
    d = tmp_path_factory.mktemp("nstep")
    src, so = d / "nstep_driver.cpp", d / "libnstep.so"
    src.write_text(DRIVER)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wno-unknown-pragmas",
                           "-I", HD, "-I", CSRC, "-shared", "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    vp = C.c_void_p
    L.hd_window.restype = None
    L.hd_window.argtypes = [vp, vp, C.c_longlong, C.c_longlong, vp, C.c_longlong, C.c_int, C.c_float, vp, vp, vp, vp, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def device_windows(nh, ring, keys, n, gamma):
    keys = np.ascontiguousarray(keys, np.int64)
    B = keys.size
    G, t, ns_, d, m = np.empty(B, np.float32), np.empty(B, np.uint8), np.empty(B, np.int64), np.empty(B, np.float32), np.empty(B, np.int32)
    nh.hd_window(_p(ring.reward), _p(ring.flag), ring.lanes, ring.cap, _p(keys), B, n, gamma, _p(G), _p(t), _p(ns_), _p(d), _p(m))
    return G, t, ns_, d, m


def check_all(nh, ring, n, gamma, keys=None):
    """every sampleable key (or `keys`): the header's window equals the restatement bit for bit; returns the horizons"""
    keys = ring.sampleable_keys() if keys is None else keys
    assert keys.size
    G, t, nslot, d, m = device_windows(nh, ring, keys, n, gamma)
    for k, key in enumerate(keys):
        rG, rt, rns, rd, rm = N.window(ring.flag, ring.reward, ring.lanes, ring.cap, key, n, gamma)
        assert (G[k].view(np.uint32), t[k], nslot[k], d[k].view(np.uint32), m[k]) == (np.float32(rG).view(np.uint32), rt, rns,
                                                                                     np.float32(rd).view(np.uint32), rm), (key, n, gamma)
    return m


def odd_rewards(rng, size):
    """rewards whose discounted sums round: a spread of magnitudes, non-dyadic fractions"""
    return (rng.standard_normal(size) * 10.0 ** rng.integers(-3, 4, size) + 1 / 3).astype(np.float32)


def fill(ring, rng, frames, p_term=0.15, auto_reset=True, reset_at=()):
    obs = rng.standard_normal((ring.ns, ring.lanes)).astype(np.float32)
    ring.push_episode_start(obs)
    for k in range(frames):
        if k in reset_at:                                   # forced reset (ResetAfterNSteps / re-entering run): every lane
            ring.push_episode_start(rng.standard_normal((ring.ns, ring.lanes)).astype(np.float32))
        t = (rng.random(ring.lanes) < p_term).astype(np.uint8) * (3 if auto_reset else 1)
        nxt = rng.standard_normal((ring.ns, ring.lanes)).astype(np.float32)
        ring.push(rng.integers(1, 3, ring.lanes).astype(np.int32), odd_rewards(rng, ring.lanes), t, nxt)
        if not auto_reset:
            ring.push_episode_start(rng.standard_normal((ring.ns, ring.lanes)).astype(np.float32), pending_only=True)


GAMMAS = [0.0, 0.5, 0.99, 1.0]


@pytest.mark.parametrize("gamma", GAMMAS)
@pytest.mark.parametrize("n", [1, 2, 3, 5, 8])
def test_wrapped_ring_with_terminals_and_forced_reset(nh, n, gamma):
    rng = np.random.default_rng(n * 10 + int(gamma * 100))
    ring = N.HostRing(3, 7, 16)
    fill(ring, rng, 45, reset_at=(30,))                     # wraps ~3 times; the forced reset's straddling entry is still in the ring
    m = check_all(nh, ring, n, gamma)
    assert m.max() == n and (n == 1 or m.min() == 1)


@pytest.mark.parametrize("auto_reset", [True, False])
def test_soft_reset_ring(nh, auto_reset):
    rng = np.random.default_rng(4)
    ring = N.HostRing(2, 5, 24)
    fill(ring, rng, 60, p_term=0.2, auto_reset=auto_reset)
    for n in (2, 4, 7):
        check_all(nh, ring, n, 0.9)


def _single_lane(rewards, terms, cap, resets=()):
    """lane of 1: transitions with these rewards / terminal bits (auto-reset), forced resets before the listed steps"""
    ring = N.HostRing(1, 1, cap)
    ring.push_episode_start(np.zeros((1, 1), np.float32))
    for k, (r, t) in enumerate(zip(rewards, terms)):
        if k in resets:
            ring.push_episode_start(np.full((1, 1), -1.0, np.float32))
        ring.push(np.ones(1, np.int32), np.array([r], np.float32), np.array([3 if t else 0], np.uint8), np.full((1, 1), k + 1.0, np.float32))
    return ring


def test_known_windows(nh):
    cap = 12
    # steps 0..8, terminal at step 3 (entry 3), forced reset before step 6
    ring = _single_lane([1, 2, 4, 8, 16, 32, 64, 128, 256], [0, 0, 0, 1, 0, 0, 0, 0, 0], cap, resets=(6,))
    # slots: s0 e0 | e1 | e2 | e3(T) | start | e4 | e5 | straddle | e6 | e7 | e8 | head
    keys = np.array([0, 1, 2, 3, 5, 6, 8, 9, 10], np.int64)
    G, t, nslot, d, m = device_windows(nh, ring, keys, 4, 1.0)
    assert m.tolist() == [4, 3, 2, 1, 2, 1, 3, 2, 1]                  # terminal at 3, reset straddle after 6, lane head after 10
    assert G.tolist() == [15, 14, 12, 8, 48, 32, 448, 384, 256]
    assert t.tolist() == [1, 1, 1, 1, 0, 0, 0, 0, 0]
    assert nslot.tolist() == [4, 4, 4, 4, 7, 7, 11, 11, 11]
    assert d.tolist() == [1.0] * 9
    check_all(nh, ring, 4, 1.0, keys)
    # the terminal at a window's first entry: length 1 whatever n is
    _, t0, _, _, m0 = device_windows(nh, ring, np.array([3], np.int64), 32, 0.5)
    assert (m0[0], t0[0]) == (1, 1)


def test_wrap_across_the_last_slot(nh):
    cap = 6                                                              # 7 slots; 10 pushes wrap the lane
    ring = _single_lane([0.1 * k for k in range(10)], [0] * 10, cap)
    keys = ring.sampleable_keys()
    assert keys.size == cap and ring.head[0] == 4
    m = check_all(nh, ring, 3, 0.99, keys)
    _, _, nslot, _, _ = device_windows(nh, ring, keys, 3, 0.99)
    assert sorted(zip(keys.tolist(), nslot.tolist(), m.tolist())) == [(0, 3, 3), (1, 3, 2), (2, 3, 1), (4, 0, 3), (5, 1, 3), (6, 2, 3)]


def test_n_larger_than_anything_available(nh):
    ring = _single_lane([1.5, 2.5, 3.5], [0, 0, 0], 40)
    G, t, nslot, d, m = device_windows(nh, ring, ring.sampleable_keys(), 32, 0.5)
    assert m.tolist() == [3, 2, 1] and nslot.tolist() == [3, 3, 3]
    assert G.tolist() == [np.float32(1.5 + 0.5 * (2.5 + 0.5 * 3.5)), np.float32(2.5 + 0.5 * 3.5), 3.5]
    assert d.tolist() == [0.125, 0.25, 0.5]
    check_all(nh, ring, 32, 0.5)


def test_n_one_is_the_one_step_gather(nh):
    rng = np.random.default_rng(9)
    ring = N.HostRing(4, 6, 10)
    fill(ring, rng, 25)
    keys = ring.sampleable_keys()
    G, t, nslot, d, m = device_windows(nh, ring, keys, 1, np.float32(0.99))
    assert np.array_equal(G, ring.reward[keys]) and np.array_equal(t, ring.flag[keys] & 1)
    assert np.array_equal(nslot, (keys // 6 + 1) % 11) and np.all(m == 1) and np.all(d == np.float32(0.99))


def test_rounding_follows_discount_rewards_order(nh):
    """not the forward sum Σ γ^j r_j, not an FMA: the backward recursion with two roundings per step"""
    rng = np.random.default_rng(17)
    rewards = odd_rewards(rng, 20)
    ring = _single_lane(rewards, [0] * 20, 32)
    keys = ring.sampleable_keys()
    assert np.array_equal(keys, np.arange(20))
    m = check_all(nh, ring, 8, 0.99, keys)
    G, _, _, _, _ = device_windows(nh, ring, keys, 8, 0.99)
    g = np.float32(0.99)
    fwd = [np.float32(sum(np.float64(g) ** j * np.float64(rewards[k + j]) for j in range(m[k]))) for k in range(len(keys))]
    assert np.any(G != np.array(fwd, np.float32))                    # the order matters at these magnitudes
    # windows that run to the lane head are the oracle's discount_rewards of the series, bit for bit
    G32, _, _, _, m32 = device_windows(nh, ring, keys, 32, 0.99)
    assert np.array_equal(m32, 20 - keys)
    ref = O.discount_rewards(rewards, np.float32(0.99), dtype=np.float32)
    assert np.array_equal(G32.view(np.uint32), ref.astype(np.float32).view(np.uint32))


def test_host_ring_matches_the_oracle_ring():
    """the HostRing model used for the synthetic rings pushes like the oracle ring: same 1-step batches from the same streams"""
    rng = np.random.default_rng(23)
    ns, lanes, cap, B = 3, 9, 14, 512
    ring, ref = N.HostRing(ns, lanes, cap), O.OracleTraj(ns, lanes, cap)
    obs = rng.standard_normal((ns, lanes)).astype(np.float32)
    ring.push_episode_start(obs); ref.push_state(obs)
    for k in range(40):
        if k == 25:
            obs = rng.standard_normal((ns, lanes)).astype(np.float32)
            ring.push_episode_start(obs); ref.push_state(obs)
        a, r = rng.integers(1, 3, lanes).astype(np.int32), odd_rewards(rng, lanes)
        t, nxt = ((rng.random(lanes) < 0.2) * 3).astype(np.uint8), rng.standard_normal((ns, lanes)).astype(np.float32)
        ring.push(a, r, t, nxt); ref.push(a, r, t, nxt)
    assert ref.n_sampleable() == ring.sampleable_keys().size
    rb = ref.sample(O.splitmix_states_fast(B, 3), B)
    one = N.nstep_batch(ring.export(), ns, lanes, cap, rb["key"], 1, 0.99)
    assert np.array_equal(one["reward"], rb["reward"]) and np.array_equal(one["terminal"], rb["terminal"])
    assert np.array_equal(one["next_state"], rb["next_state"])
    assert np.array_equal(ring.action[rb["key"]], rb["action"])
