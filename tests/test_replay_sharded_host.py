"""Host side of the sharded explorer numbering (no GPU).

csrc/explore.cuh compiled for the host: a batch planned as G shards — rank r's N columns at explore::column_step(s, r N, G N, k, i),
each on its own stream — gives, plan after plan, the actions and advanced streams of one BatchExplorer over the G N columns whose
step advances by G N per plan.  Every explorer kind, G = 1, 2, 3; checked against the oracle (ϵ-greedy kinds), the NumPy restatement
of explorers_ref.py (kinds 2-4) and explorers.py's get_eps at the global steps.  G = 1 is the unsharded arithmetic, step + k N + i."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import explorers_ref as R
import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))
HD = os.path.join(HERE, "hostdev")
CSRC = os.path.join(os.path.dirname(HERE), "reinforcementlearning.jl_b200", "csrc")

DRIVER = r"""
#include <cuda_runtime.h>
#include "explore.cuh"
extern "C" {
// plan k of one rank's n columns: column i at explore::column_step(step, col0, stride, k, i); rng (n, 4) advanced in place
void hd_plan_shard(const b200rl_explorer* e, long long step, long long col0, long long stride, long long k, const float* qv, int na,
                   long long n, unsigned long long* rng, int* out) {
    for (long long i = 0; i < n; ++i) {
        unsigned long long st[4] = {rng[4 * i], rng[4 * i + 1], rng[4 * i + 2], rng[4 * i + 3]};
        out[i] = explore::select(*e, explore::column_step(step, col0, stride, k, i), qv + (long long)na * i, na, st);
        for (int j = 0; j < 4; ++j) rng[4 * i + j] = st[j];
    }
}
long long hd_column_step(long long step, long long col0, long long stride, long long k, long long i) {
    return explore::column_step(step, col0, stride, k, i);
}
}
"""


@pytest.fixture(scope="module")
def sh(tmp_path_factory):
    d = tmp_path_factory.mktemp("sharded")
    src, so = d / "sharded_driver.cpp", d / "libsharded.so"
    src.write_text(DRIVER)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wno-unknown-pragmas",
                           "-I", HD, "-I", CSRC, "-shared", "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    vp, ll = C.c_void_p, C.c_longlong
    L.hd_plan_shard.restype, L.hd_plan_shard.argtypes = None, [vp, ll, ll, ll, ll, vp, C.c_int, ll, vp, vp]
    L.hd_column_step.restype, L.hd_column_step.argtypes = ll, [ll, ll, ll, ll, ll]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _explorer(pkg, name, total):
    if name in ("linear", "exp", "break_tie"):   # the decay ends inside the planned window
        return pkg.EpsilonGreedyExplorer(0.05, kind="exp" if name == "exp" else "linear", eps_init=1.0, warmup_steps=total // 3,
                                         decay_steps=total, is_break_tie=name == "break_tie", step=1)
    if name == "speedy":
        return pkg.EpsilonSpeedyExplorer(3.0 / total, step=1)
    return {"weighted": pkg.WeightedSoftmaxExplorer, "gumbel": pkg.GumbelSoftmaxExplorer}[name]()


def _reference(pkg, name, ex, step, q, rng):
    """one plan of the whole batch (every rank's columns) by the oracle / the NumPy restatement"""
    st = ex.as_struct()
    if st.kind <= 1:
        ex6 = O.explorer6(ex.eps_stable, ex.eps_init, ex.warmup_steps, ex.decay_steps, ex.kind, ex.is_break_tie)
        return O.egreedy_plan(ex6, step, np.asfortranarray(q), rng)
    return R.plan(st.kind, q, rng, step0=step, beta=st.beta)


KINDS = ["linear", "exp", "break_tie", "speedy", "weighted", "gumbel"]


@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("name", KINDS)
def test_shards_plan_like_one_batch_explorer_over_the_union(pkg, sh, name, world):
    n, na, plans = 37, 3, 4
    total = world * n
    rng0 = O.splitmix_states_fast(total, 1000 + world)
    qs = [np.random.default_rng(10 * k + world).standard_normal((na, total)).astype(np.float32) for k in range(plans)]
    for q in qs:
        q[:, ::5] = q[0, ::5]                                    # ties for break-tie
    ex_g = _explorer(pkg, name, plans * total)                    # one BatchExplorer over the union
    exs = [_explorer(pkg, name, plans * total) for _ in range(world)]   # each rank's copy
    ref_rng, rngs = rng0.copy(), [rng0[r * n:(r + 1) * n].copy() for r in range(world)]
    s_w = int(exs[0].as_struct().step)                           # explorer step at the start of the window, the same on every rank
    for k in range(plans):
        s0 = int(ex_g.as_struct().step)
        ref = _reference(pkg, name, ex_g, s0, qs[k], ref_rng)
        ex_g.advance(total)
        got = np.empty(total, np.int32)
        for r in range(world):
            st = exs[r].as_struct()
            a = np.empty(n, np.int32)
            qr = np.asfortranarray(qs[k][:, r * n:(r + 1) * n])
            assert st.step == (s0 if hasattr(ex_g, "step") else 0)       # each rank's copy holds the global step
            sh.hd_plan_shard(C.byref(st), s_w, r * n, total, k, _p(qr), na, n, _p(rngs[r]), _p(a))
            got[r * n:(r + 1) * n] = a
        for r in range(world):
            exs[r].advance(total)                                 # every plan! moves each rank's explorer by G N
        assert np.array_equal(got, ref), (name, world, k)
        assert np.array_equal(np.concatenate(rngs), ref_rng)
    if hasattr(ex_g, "step"):
        assert all(e.step == ex_g.step == 1 + plans * total for e in exs)
    assert not np.array_equal(ref_rng, rng0)


@pytest.mark.parametrize("world", [1, 2, 3])
def test_global_steps_and_epsilons(pkg, sh, world):
    n, plans = 50, 6
    ex = pkg.EpsilonGreedyExplorer(0.1, eps_init=1.0, warmup_steps=40, decay_steps=world * n * 3)
    seen = []
    for k in range(plans):
        for r in range(world):
            for i in range(n):
                seen.append(sh.hd_column_step(7, r * n, world * n, k, i))
    # every global step 7 .. 7 + plans G N - 1 once, in BatchExplorer order
    assert seen == list(range(7, 7 + plans * world * n))
    for s in seen[::17]:
        assert O.get_eps(O.explorer6(0.1, 1.0, 40, world * n * 3, "linear"), s) == ex.get_eps(s)


def test_one_gpu_is_the_unsharded_arithmetic(sh):
    for step, n, k, i in ((1, 127, 0, 0), (1, 127, 5, 126), (2 ** 40, 4096, 9, 4095), (-3, 1, 3, 0)):
        assert sh.hd_column_step(step, 0, n, k, i) == step + k * n + i
