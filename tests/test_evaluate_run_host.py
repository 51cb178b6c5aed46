"""run() of an evaluation policy on the fused path, host side (no GPU).

csrc/stop_episodes.cuh's stretch rule of b200rl_eval_run_episodes (stop::eval_stretch) compiled for the host and checked against its
contract; run()'s dispatch of EvaluationPolicy / QBasedPolicy to run_episodes on stub envs and policies, and to the stage loop where
the fused path does not apply; the Julia glue's ccall of the new entry point against the ABI."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_stop_episodes_host import CSRC, HD, PERIODS, StubEnv, _julia_ccalls, stage_reference, stage_reference_steps

DRIVER = r"""
#include <cuda_runtime.h>
#include "stop_episodes.cuh"
extern "C" long long hd_eval_stretch(long long left, long long remaining, long long n, int counting) {
    return stop::eval_stretch(left, remaining, n, counting != 0);
}
extern "C" long long hd_eval_stretch_max() { return stop::kEvalStretchMax; }
extern "C" long long hd_eval_stretch_marked() { return stop::kEvalStretchMarked; }
"""


@pytest.fixture(scope="module")
def sh(tmp_path_factory):
    d = tmp_path_factory.mktemp("eval_stretch")
    src, so = d / "eval_driver.cpp", d / "libeval.so"
    src.write_text(DRIVER)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-I", HD, "-I", CSRC, "-shared", "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    L.hd_eval_stretch.restype = C.c_longlong
    L.hd_eval_stretch.argtypes = [C.c_longlong, C.c_longlong, C.c_longlong, C.c_int]
    L.hd_eval_stretch_max.restype = L.hd_eval_stretch_marked.restype = C.c_longlong
    return L


def test_stretch_constants(sh):
    assert (sh.hd_eval_stretch_max(), sh.hd_eval_stretch_marked()) == (1024, 64)


@pytest.mark.parametrize("left", [1, 7, 64, 65, 1023, 1024, 1025, 1 << 40])
def test_stretch_without_budget(sh, left):
    """StopAfterNSteps: every stretch as long as the cap allows, whatever the (unused) remaining budget"""
    for n in (1, 96, 65_537):
        for remaining in (-5, 0, 1, 10 ** 9):
            assert sh.hd_eval_stretch(left, remaining, n, 0) == min(left, 1024)


def test_stretch_with_budget(sh):
    rng = np.random.default_rng(7)
    cases = [(left, rem, n) for left in (1, 20, 64, 100, 1024, 5000, 1 << 40) for n in (1, 4, 96, 65_537)
             for rem in (-3, 0, 1, n, 63 * n, 64 * n, 64 * n + 1, 65 * n, 1000 * n, 5000 * n + 17)]
    cases += [(int(rng.integers(1, 3000)), int(rng.integers(-10, 10 ** 7)), int(rng.integers(1, 70_000))) for _ in range(3000)]
    for left, rem, n in cases:
        s = sh.hd_eval_stretch(left, rem, n, 1)
        assert 1 <= s <= min(left, 1024), (left, rem, n, s)
        unmarked = (rem - 1) // n if rem > 0 else 0   # the longest stretch that cannot reach the budget
        assert s == (min(left, 1024, unmarked) if unmarked >= 64 else min(left, 64)), (left, rem, n, s)
        if rem <= n * s:                              # run_stretches marks a stretch that could reach the budget ...
            assert s <= 64                            # ... and a rollback re-runs at most 64 steps
        if unmarked >= 64:
            assert n * s < rem


def test_stretches_cover_a_run_and_end_marked(sh):
    """a budget of many episodes: unmarked stretches shrink with the budget until the marked ones of 64 steps take over, and no
    unmarked stretch could have crossed"""
    n, budget = 8, 40_000
    remaining, kinds = budget, []
    while remaining > 0:
        s = sh.hd_eval_stretch(1 << 40, remaining, n, 1)
        marked = remaining <= n * s
        kinds.append(marked)
        if marked:
            break
        remaining -= n * s                                  # the most episodes s steps of n lanes can end
    assert kinds[-1] and not any(kinds[:-1]) and len(kinds) > 3


# ---- run() dispatch -----------------------------------------------------------------------------------------------------------
class StubEvalPolicy:
    """an evaluation policy stand-in: the stage protocol steps the env through act_; run_episodes(env, ...) steps it up to the
    crossing, or max_steps steps without a budget; eval_handle is None where the library would refuse the pair"""

    def __init__(self, fusable=True, supported=True):
        self.fusable, self.supported = fusable, supported
        self.calls = []

    def push(self, stage, env, action=None):
        pass

    def optimise(self, stage):
        pass

    def plan(self, env):
        return np.zeros(env.n, np.int32)

    def eval_handle(self, env):
        return object() if self.supported else None

    def run_episodes(self, env, max_steps, budget):
        self.calls.append((max_steps, budget))
        steps = episodes = 0
        while steps < max_steps:
            env.step()
            steps += 1
            if budget is None:
                continue
            episodes += int(env.term.sum())
            if episodes >= budget:
                break
        return steps, episodes


@pytest.mark.parametrize("k,cur", [(1, 0), (9, 0), (30, 2), (5, 5), (5, 9)])
@pytest.mark.parametrize("capacity", [None, 4])
def test_dispatch_episodes(pkg, k, cur, capacity):
    env, pol = StubEnv(PERIODS), StubEvalPolicy()
    stop = pkg.StopAfterNEpisodes(k, cur)
    hook = pkg.EmptyHook() if capacity is None else pkg.DeviceEpisodeLog(env.n, capacity=capacity)
    pkg.run(pol, env, stop, hook)
    assert pol.calls and pol.calls[0][1] == k - cur
    assert (env.steps, stop.cur) == stage_reference(pkg, k, cur)
    if capacity is not None:
        assert all(m == capacity for m, _ in pol.calls) and env.flushes >= len(pol.calls)


@pytest.mark.parametrize("n,cur", [(1, 1), (13, 1), (13, 4), (7, 9)])
def test_dispatch_steps(pkg, n, cur):
    env, pol = StubEnv(PERIODS), StubEvalPolicy()
    stop = pkg.StopAfterNSteps(n, cur)
    pkg.run(pol, env, stop, pkg.DeviceEpisodeLog(env.n, capacity=3))
    assert pol.calls and all(budget is None for _, budget in pol.calls)
    assert (env.steps, stop.cur) == stage_reference_steps(pkg, n, cur)


def test_dispatch_stage_loop(pkg):
    """not fusable, refused by the library, an episode count on a sharded ctx, a per-step hook: the stage loop, the same steps"""
    k = 9
    ref = stage_reference(pkg, k)
    for env, pol, hook in ((StubEnv(PERIODS), StubEvalPolicy(fusable=False), pkg.EmptyHook()),
                           (StubEnv(PERIODS), StubEvalPolicy(supported=False), pkg.EmptyHook()),
                           (StubEnv(PERIODS, world=2), StubEvalPolicy(), pkg.EmptyHook()),
                           (StubEnv(PERIODS), StubEvalPolicy(), pkg.BatchStepsPerEpisode(4))):
        stop = pkg.StopAfterNEpisodes(k)
        pkg.run(pol, env, stop, hook)
        assert not pol.calls
        assert (env.steps, stop.cur) == ref


def test_julia_ccall_matches_the_abi(pkg):
    def kind_jl(t):
        return "ptr" if t.startswith(("Ptr{", "Ref{")) else {"Int64": "i64", "Cint": "i32", "Int32": "i32"}[t]

    def kind_c(t):
        return {C.c_void_p: "ptr", C.c_int64: "i64", C.c_int: "i32", C.c_int32: "i32"}.get(t, "ptr")
    for name in ("b200rl_eval_create", "b200rl_eval_run_episodes", "b200rl_eval_destroy"):
        calls = _julia_ccalls(name)
        assert calls, f"{name} is not called from julia/B200RL.jl"
        want = [kind_c(t) for t in pkg._lib.SIGNATURES[name][1]]
        for args in calls:
            assert [kind_jl(a) for a in args if a] == want, (name, args)
