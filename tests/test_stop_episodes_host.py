"""StopAfterNEpisodes on the fused loops, host side (no GPU).

csrc/stop_episodes.cuh's crossing arithmetic (the first step at which the per-step episode counts reach the remaining budget)
compiled for the host and compared with a NumPy restatement; run()'s dispatch of StopAfterNEpisodes to the fused library calls
(b200rl_*_run_episodes) on stub envs and agents, and to the stage loop where the fused path does not apply; the same dispatch for
StopAfterNSteps (no episode budget)."""
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
#include "stop_episodes.cuh"
extern "C" void hd_crossing(const unsigned long long* counts, long long s, long long remaining, long long* out) {
    const StopCrossing c = stop::crossing(counts, s, remaining);
    out[0] = c.step; out[1] = c.episodes;
}
"""


@pytest.fixture(scope="module")
def sh(tmp_path_factory):
    d = tmp_path_factory.mktemp("stop_episodes")
    src, so = d / "stop_driver.cpp", d / "libstop.so"
    src.write_text(DRIVER)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-I", HD, "-I", CSRC, "-shared", "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    L.hd_crossing.restype = None
    L.hd_crossing.argtypes = [C.c_void_p, C.c_longlong, C.c_longlong, C.c_void_p]
    return L


def header_crossing(sh, counts, remaining):
    counts = np.ascontiguousarray(counts, np.uint64)
    out = np.zeros(2, np.int64)
    sh.hd_crossing(counts.ctypes.data_as(C.c_void_p), counts.size, int(remaining), out.ctypes.data_as(C.c_void_p))
    return int(out[0]), int(out[1])


def numpy_crossing(counts, remaining):
    """the stage loop: cur += count_t after step t, stop once cur >= k; remaining = k - cur on entry"""
    csum = np.cumsum(np.asarray(counts, np.int64))
    hit = np.nonzero(csum >= remaining)[0]
    if hit.size == 0:
        return 0, int(csum[-1]) if csum.size else 0
    return int(hit[0]) + 1, int(csum[hit[0]])


def terminal_counts(flags):
    """per-step counts from an (N, s) terminal matrix"""
    return np.asarray(flags, bool).sum(axis=0).astype(np.uint64)


CASES = {
    "budget_spent": ([3, 0, 5], 0),               # cur >= k on entry: exactly one step
    "budget_negative": ([0, 0, 2], -4),           # (one step even when it ends no episode)
    "first_step": ([7, 1, 1], 5),
    "exact_hit": ([1, 2, 3, 4], 6),
    "overshoot": ([1, 2, 3, 4], 5),
    "no_crossing": ([1, 0, 2, 0], 10),
    "last_step": ([0, 0, 0, 9], 1),
    "empty_steps": ([0, 0, 0, 0], 1),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_crossing_cases(sh, name):
    counts, remaining = CASES[name]
    got = header_crossing(sh, counts, remaining)
    assert got == numpy_crossing(counts, remaining)
    if remaining <= 0:
        assert got[0] == 1


def test_crossing_all_lanes_together(sh):
    """N lanes that all terminate on the same steps (a fixed episode length): counts of N on those steps, 0 elsewhere"""
    n, length, s = 64, 5, 23
    flags = np.zeros((n, s), bool)
    flags[:, length - 1::length] = True
    counts = terminal_counts(flags)
    for remaining in (1, n - 1, n, n + 1, 2 * n, 4 * n, 4 * n + 1, 10 * n):
        got = header_crossing(sh, counts, remaining)
        assert got == numpy_crossing(counts, remaining), remaining
    assert header_crossing(sh, counts, n) == (length, n)
    assert header_crossing(sh, counts, n + 1) == (2 * length, 2 * n)


def test_crossing_random(sh):
    rng = np.random.default_rng(7)
    for _ in range(200):
        n, s = int(rng.integers(1, 300)), int(rng.integers(1, 40))
        flags = rng.random((n, s)) < rng.uniform(0.0, 0.3)
        counts = terminal_counts(flags)
        remaining = int(rng.integers(-3, int(counts.sum()) + 5))
        assert header_crossing(sh, counts, remaining) == numpy_crossing(counts, remaining)


# ---- run() dispatch ---------------------------------------------------------------------------------------------------------
class StubCtx:
    h = None

    def __init__(self, world=1):
        self.world = world

    def rank_world(self):
        return 0, self.world


class StubEnv:
    """N lanes; lane i terminates every period[i] steps (auto-reset); an episode log that records nothing"""

    def __init__(self, periods, auto_reset=True, world=1):
        self.periods = np.asarray(periods, np.int64)
        self.n = len(self.periods)
        self.auto_reset = auto_reset
        self.ctx = StubCtx(world)
        self.t = np.zeros(self.n, np.int64)
        self.term = np.zeros(self.n, bool)
        self.steps = 0
        self.flushes = 0

    def reset_(self, is_force=True):
        if is_force:
            self.t[:] = 0
        self.term[:] = False

    def step(self):
        self.t += 1
        self.term = self.t % self.periods == 0
        self.steps += 1

    def is_terminated(self):
        return self.term

    def act_(self, action):
        self.step()

    def check(self):
        pass

    def episode_stats(self, reset=False):
        return None

    def episode_log(self, capacity):
        pass

    def episode_log_buffer(self, records):
        return np.zeros(0), 0

    def episode_log_flush(self, addr, records):
        self.flushes += 1

    def episode_log_read(self, arr, addr):
        return np.zeros(0, [("env", np.int64), ("ret", np.float32), ("len", np.int32)])


class StubAgent:
    """a device agent stand-in: the stage protocol steps the env through act_; run_episodes steps it up to the crossing, or
    max_steps steps without a budget"""

    def __init__(self, fusable=True, host_actions=False):
        self.fusable, self.host_actions = fusable, host_actions
        self.calls = []
        self.env = None

    def push(self, stage, env, action=None):
        self.env = env

    def optimise(self, stage):
        pass

    def plan(self, env):
        return np.zeros(env.n, np.int32)

    def run_episodes(self, max_steps, budget):
        self.calls.append((max_steps, budget))
        steps = episodes = 0
        while steps < max_steps:
            self.env.step()
            steps += 1
            if budget is None:
                continue
            episodes += int(self.env.term.sum())
            if episodes >= budget:
                break
        return steps, episodes


PERIODS = [3, 5, 7, 4]


def stage_reference(pkg, k, cur=0):
    """steps and stop.cur of the stage loop with a per-step hook"""
    env, agent = StubEnv(PERIODS), StubAgent(fusable=False)
    stop = pkg.StopAfterNEpisodes(k, cur)
    pkg.run(agent, env, stop, pkg.BatchStepsPerEpisode(env.n))
    assert not agent.calls
    return env.steps, stop.cur


def make_hook(pkg, which, n):
    return {"empty": lambda: pkg.EmptyHook(), "stats": lambda: pkg.DeviceEpisodeStats(),
            "log": lambda: pkg.DeviceEpisodeLog(n, capacity=4),
            "composed": lambda: pkg.DeviceEpisodeStats() + pkg.DeviceEpisodeLog(n, capacity=3)}[which]()


@pytest.mark.parametrize("which", ["empty", "stats", "log", "composed"])
@pytest.mark.parametrize("k,cur", [(1, 0), (9, 0), (30, 2), (5, 5), (5, 9)])
def test_dispatch_fused(pkg, which, k, cur):
    env, agent = StubEnv(PERIODS), StubAgent()
    stop = pkg.StopAfterNEpisodes(k, cur)
    hook = make_hook(pkg, which, env.n)
    pkg.run(agent, env, stop, hook, pkg.ResetIfEnvTerminated())
    assert agent.calls, "the fused call was not taken"
    assert (env.steps, stop.cur) == stage_reference(pkg, k, cur)
    window = {"empty": None, "stats": None, "log": 4, "composed": 3}[which]
    if window is None:
        assert len(agent.calls) == 1
    else:
        assert all(m == window for m, _ in agent.calls)
        assert len(agent.calls) == -(-env.steps // window)
        assert env.flushes >= len(agent.calls)
    assert agent.calls[0][1] == k - cur


def stage_reference_steps(pkg, n, cur):
    """steps and stop.cur of the stage loop for StopAfterNSteps(n, cur) with a per-step hook"""
    env, agent = StubEnv(PERIODS), StubAgent(fusable=False)
    stop = pkg.StopAfterNSteps(n, cur)
    pkg.run(agent, env, stop, pkg.BatchStepsPerEpisode(env.n))
    assert not agent.calls
    return env.steps, stop.cur


@pytest.mark.parametrize("which", ["empty", "log", "composed"])
@pytest.mark.parametrize("n,cur", [(1, 1), (12, 1), (13, 1), (13, 4), (7, 9)])
def test_dispatch_fused_steps(pkg, which, n, cur):
    """StopAfterNSteps through the same call, without an episode budget: windows of none, 4 and 3 steps"""
    env, agent = StubEnv(PERIODS), StubAgent()
    stop = pkg.StopAfterNSteps(n, cur)
    pkg.run(agent, env, stop, make_hook(pkg, which, env.n), pkg.ResetIfEnvTerminated())
    assert agent.calls, "the fused call was not taken"
    assert all(budget is None for _, budget in agent.calls)
    assert (env.steps, stop.cur) == stage_reference_steps(pkg, n, cur)
    window = {"empty": None, "log": 4, "composed": 3}[which]
    if window is None:
        assert agent.calls == [(env.steps, None)]
    else:
        assert [m for m, _ in agent.calls] == [min(window, env.steps - j) for j in range(0, env.steps, window)]
        assert env.flushes >= len(agent.calls)


def test_dispatch_stage_loop(pkg):
    k = 9
    ref = stage_reference(pkg, k)
    # a per-step hook, a soft-reset env, host actions, a sharded ctx: the stage loop, the same steps
    for env, agent, hook in ((StubEnv(PERIODS), StubAgent(), pkg.BatchStepsPerEpisode(4)),
                             (StubEnv(PERIODS, auto_reset=False), StubAgent(), pkg.EmptyHook()),
                             (StubEnv(PERIODS), StubAgent(fusable=False, host_actions=True), pkg.EmptyHook()),
                             (StubEnv(PERIODS, world=2), StubAgent(), pkg.EmptyHook())):
        stop = pkg.StopAfterNEpisodes(k)
        pkg.run(agent, env, stop, hook)
        assert not agent.calls
        assert (env.steps, stop.cur) == ref


def test_dispatch_other_reset_condition(pkg):
    env, agent = StubEnv(PERIODS), StubAgent()
    pkg.run(agent, env, pkg.StopAfterNEpisodes(9), pkg.EmptyHook(), pkg.ResetAfterNSteps(1000))
    assert not agent.calls


# ---- the Julia glue's calls ---------------------------------------------------------------------------------------------------
def _julia_ccalls(name):
    """argument type tuples of every ccall of `name` in julia/B200RL.jl"""
    import re
    src = open(os.path.join(os.path.dirname(HERE), "reinforcementlearning.jl_b200", "julia", "B200RL.jl")).read()
    out = []
    for m in re.finditer(r"ccall\(\(:" + name + r", LIB\), Cint,\s*\(", src):
        depth, i = 1, m.end()
        while depth:
            depth += {"(": 1, ")": -1}.get(src[i], 0)
            i += 1
        args, depth, cur = [], 0, ""
        for ch in src[m.end():i - 1]:
            if ch == "," and depth == 0:
                args.append(cur.strip()); cur = ""
                continue
            depth += {"{": 1, "}": -1}.get(ch, 0)
            cur += ch
        args.append(cur.strip())
        out.append(args)
    return out


@pytest.mark.parametrize("name", ["b200rl_onpolicy_run_episodes", "b200rl_replay_run_episodes"])
def test_julia_ccalls_match_the_abi(pkg, name):
    """the Julia _run's StopAfterNEpisodes branch calls both entry points with the argument kinds include/b200rl.h declares"""
    def kind_jl(t):
        return "ptr" if t.startswith(("Ptr{", "Ref{")) else {"Int64": "i64", "Cint": "i32", "Int32": "i32"}[t]

    def kind_c(t):
        return {C.c_void_p: "ptr", C.c_int64: "i64", C.c_int: "i32"}.get(t, "ptr")
    calls = _julia_ccalls(name)
    assert calls, f"{name} is not called from julia/B200RL.jl"
    want = [kind_c(t) for t in pkg._lib.SIGNATURES[name][1]]
    for args in calls:
        assert [kind_jl(a) for a in args] == want, args
