"""Host side of the device DQN agent loop (no GPU).

csrc/explore.cuh (one BatchExplorer column: get_ϵ, the uniform draw, findmax / break-tie, Lemire's rand(1:n)) compiled for the
host, bit-exact against explorers.py and the oracle; csrc/replay_schedule.h (the InsertSampleRatioController schedule that
b200rl_replay_run computes ahead of its launches) against learners.InsertSampleRatioController."""
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
#include "explore.cuh"
#include "replay_schedule.h"
static b200rl_explorer mk(const double* e6) {
    b200rl_explorer e;
    e.eps_stable = e6[0]; e.eps_init = e6[1]; e.warmup_steps = (int64_t)e6[2]; e.decay_steps = (int64_t)e6[3]; e.step = 0;
    e.kind = (int32_t)e6[4]; e.is_break_tie = (int32_t)e6[5];
    return e;
}
extern "C" double hd_get_eps(const double* e6, long long step) { return explore::explorer_eps(mk(e6), step); }
// BatchExplorer over the columns of qv (na, n) with column i at step0 + i; rng (n, 4) advanced in place
extern "C" void hd_plan(const double* e6, long long step0, const float* qv, int na, long long n, unsigned long long* rng, int* out) {
    const b200rl_explorer e = mk(e6);
    for (long long i = 0; i < n; ++i) {
        unsigned long long st[4] = {rng[4 * i], rng[4 * i + 1], rng[4 * i + 2], rng[4 * i + 3]};
        out[i] = explore::select(e, step0 + i, qv + (long long)na * i, na, st);
        for (int k = 0; k < 4; ++k) rng[4 * i + k] = st[k];
    }
}
// m of every step of a window, the counters advanced in c4 = {ratio, threshold, n_inserted, n_sampled}
extern "C" int hd_schedule(double* c4, long long n_steps, long long* m_out) {
    b200rl_insert_sample_ratio c{c4[0], (int64_t)c4[1], (int64_t)c4[2], (int64_t)c4[3]};
    if (!replay::controller_ok(c)) return 0;
    for (long long j = 0; j < n_steps; ++j) m_out[j] = replay::insert_then_sample(c);
    c4[2] = (double)c.n_inserted; c4[3] = (double)c.n_sampled;
    return 1;
}
"""


@pytest.fixture(scope="module")
def rh(tmp_path_factory):
    d = tmp_path_factory.mktemp("replay")
    src, so = d / "replay_driver.cpp", d / "libreplay.so"
    src.write_text(DRIVER)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wno-unknown-pragmas",
                           "-I", HD, "-I", CSRC, "-shared", "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    vp = C.c_void_p
    L.hd_get_eps.restype, L.hd_get_eps.argtypes = C.c_double, [vp, C.c_longlong]
    L.hd_plan.restype, L.hd_plan.argtypes = None, [vp, C.c_longlong, vp, C.c_int, C.c_longlong, vp, vp]
    L.hd_schedule.restype, L.hd_schedule.argtypes = C.c_int, [vp, C.c_longlong, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


SCHEDULES = [(0.05, 1.0, 0, 100, "linear"), (0.01, 0.9, 1500, 3000, "linear"), (0.1, 1.0, 7, 1, "linear"), (0.2, 0.2, 0, 0, "linear"),
             (0.05, 1.0, 0, 100, "exp"), (0.01, 0.9, 1500, 3000, "exp"), (0.0, 1.0, 3, 17, "exp")]


@pytest.mark.parametrize("sch", SCHEDULES, ids=[f"{s[4]}-{s[2]}-{s[3]}" for s in SCHEDULES])
def test_get_eps_matches_python_and_oracle(pkg, rh, sch):
    eps_stable, eps_init, warm, decay, kind = sch
    ex = pkg.EpsilonGreedyExplorer(eps_stable, kind=kind, eps_init=eps_init, warmup_steps=warm, decay_steps=decay)
    ex6 = O.explorer6(eps_stable, eps_init, warm, decay, kind)
    steps = sorted(set([0, 1, 2, warm - 1, warm, warm + 1, warm + decay - 1, warm + decay, warm + decay + 1, 10 ** 9]
                       + list(np.random.default_rng(3).integers(0, 3 * (warm + decay) + 10, 300))))
    for step in steps:
        v = rh.hd_get_eps(_p(ex6), int(step))
        assert v == ex.get_eps(int(step)) == O.get_eps(ex6, int(step)), step


@pytest.mark.parametrize("brk", [False, True])
@pytest.mark.parametrize("na", [2, 3, 4])
def test_column_selection_matches_oracle(rh, brk, na):
    n = 5000
    rng = np.random.default_rng(na + 10 * brk)
    qv = rng.standard_normal((na, n)).astype(np.float32)
    qv[:, ::7] = qv[0, ::7]                                   # all-tie columns
    qv[1 % na, 3::11] = qv[0, 3::11]                          # partial ties
    qv = np.asfortranarray(qv)
    ex6 = O.explorer6(0.05, 0.9, 1000, 2500, "linear", brk)   # the batch straddles warm-up, decay and the stable tail
    seeds = O.splitmix_states_fast(n, 7 + na)
    a, r = np.empty(n, np.int32), seeds.copy()
    rh.hd_plan(_p(ex6), 500, _p(qv), na, n, _p(r), _p(a))
    ref_rng = seeds.copy()
    ref = O.egreedy_plan(ex6, 500, qv, ref_rng)
    assert np.array_equal(a, ref) and np.array_equal(r, ref_rng)
    assert not np.array_equal(r, seeds)                       # every column drew


def test_break_tie_spreads_over_the_maxima(rh):
    n, na = 30000, 3
    qv = np.zeros((na, n), np.float32, order="F")
    ex6 = O.explorer6(0.0, 0.0, 0, 0, "linear", True)          # eps = 0: still one uniform draw, then rand(1:3) among the ties
    a, r = np.empty(n, np.int32), O.splitmix_states_fast(n, 5)
    rh.hd_plan(_p(ex6), 1, _p(qv), na, n, _p(r), _p(a))
    np.testing.assert_allclose(np.bincount(a, minlength=na + 1)[1:] / n, 1.0 / na, atol=0.01)


def _python_schedule(pkg, ratio, threshold, n_ins, n_smp, steps):
    c = pkg.InsertSampleRatioController(ratio=ratio, threshold=threshold, n_inserted=n_ins, n_sampled=n_smp)
    ms = []
    for _ in range(steps):
        c.on_insert(1)
        m = 0
        while c.on_sample():
            m += 1
        ms.append(m)
    return ms, c


def _c_schedule(rh, ratio, threshold, n_ins, n_smp, steps):
    c4 = np.array([ratio, threshold, n_ins, n_smp], np.float64)
    m = np.zeros(steps, np.int64)
    assert rh.hd_schedule(_p(c4), steps, _p(m)) == 1
    return m.tolist(), int(c4[2]), int(c4[3])


@pytest.mark.parametrize("ratio", [0.25, 1.0, 2.0, 0.1, 1 / 3, 0.7, 3.5, 0.0])
def test_schedule_matches_the_controller(pkg, rh, ratio):
    rng = np.random.default_rng(int(ratio * 1000))
    for _ in range(60):
        threshold = int(rng.integers(0, 40))
        n_ins = int(rng.integers(0, 60))
        n_smp = int(rng.integers(0, 80))
        steps = int(rng.integers(1, 200))
        ms, c = _python_schedule(pkg, ratio, threshold, n_ins, n_smp, steps)
        mc, ins, smp = _c_schedule(rh, ratio, threshold, n_ins, n_smp, steps)
        assert mc == ms and ins == c.n_inserted and smp == c.n_sampled


def test_schedule_random_ratios(pkg, rh):
    rng = np.random.default_rng(11)
    for _ in range(300):
        ratio = float(rng.choice([rng.uniform(0, 3), rng.integers(0, 5) / 4]))
        threshold, n_ins, n_smp, steps = (int(x) for x in (rng.integers(0, 100), rng.integers(0, 100), rng.integers(0, 100), rng.integers(1, 150)))
        ms, c = _python_schedule(pkg, ratio, threshold, n_ins, n_smp, steps)
        mc, ins, smp = _c_schedule(rh, ratio, threshold, n_ins, n_smp, steps)
        assert mc == ms and ins == c.n_inserted and smp == c.n_sampled


def test_schedule_threshold_delays_learning(pkg, rh):
    mc, ins, smp = _c_schedule(rh, 1.0, 50, 0, 0, 30)
    assert mc == [0] * 30 and (ins, smp) == (30, 0)
    mc, _, _ = _c_schedule(rh, 0.25, 4, 0, 0, 20)
    assert mc == _python_schedule(pkg, 0.25, 4, 0, 0, 20)[0] and sum(mc) == 5     # steps 4, 8, 12, 16, 20 (one batch each)


def test_schedule_refuses_bad_controllers(rh):
    m = np.zeros(4, np.int64)
    for c4 in ([np.inf, 1, 0, 0], [np.nan, 1, 0, 0], [-0.5, 1, 0, 0], [1.0, 1, -1, 0], [1.0, 1, 0, -3], [2e6, 1, 0, 0]):
        assert rh.hd_schedule(_p(np.array(c4, np.float64)), 4, _p(m)) == 0
