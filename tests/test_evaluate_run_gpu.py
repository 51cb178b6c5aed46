"""GPU tests of run(EvaluationPolicy | QBasedPolicy, env, StopAfterNSteps | StopAfterNEpisodes, hook) on the fused evaluation kernel
(b200rl_eval_run_episodes).

Every case runs two twins built from the same seeds: one through the stage loop (a per-step hook forces it; it records the per-step
episode counts, and a DeviceEpisodeLog written by the env-step kernel or BatchStepsPerEpisode), one through the fused path
(DeviceEpisodeLog of a small capacity, so that the windows split, or EmptyHook).  Both must stop after the same step with the same
stop.cur and the same episode lists, and leave every env field, the policy or explorer streams and the explorer step the same bit for
bit (the Float64 sum of the episode returns is reduced in another order by the two kernels, through Float32 warp sums: it agrees to
1e-6 relative); the network,
its target and step are only read.  The budgets k come from a probe twin's per-step counts, so that the stop lands where each case
says."""
import ctypes as C
import types

import numpy as np
import pytest

import oracle_lib as O
import test_evaluate_explore_gpu as TX
import test_evaluate_gpu as TE
import test_replay_sharded_gpu as SH
from test_stop_episodes_gpu import StepCounts, budget_for

pytestmark = pytest.mark.gpu

N = 96
CAP = 20           # DeviceEpisodeLog capacity: run() windows of 20 steps
MARKED = 64        # stop::kEvalStretchMarked: the stretch length once fewer than 64 N episodes remain
STRETCH_MAX = 1024  # stop::kEvalStretchMax

# kind, env keywords, policy (greedy | sample | an explorer name), MaxTimeoutEnv, Float64 behind set_state_float32, hidden, act,
# dueling, tensor cores
CONFIGS = {
    "greedy-cartpole": dict(kind="CartPole", policy="greedy"),
    "sample-cartpole": dict(kind="CartPole", policy="sample", act=1),
    "greedy-pendulum": dict(kind="Pendulum", envkw=dict(continuous=True), policy="greedy", timeout=10),
    "sample-pendulum": dict(kind="Pendulum", envkw=dict(continuous=True), policy="sample", timeout=9),
    "greedy-mountaincar": dict(kind="MountainCar", policy="greedy", timeout=17),
    "sample-cartpole-f64": dict(kind="CartPole", envkw=dict(T=np.float64), f64=True, policy="sample"),
    "greedy-pendulum-f64": dict(kind="Pendulum", envkw=dict(T=np.float64, continuous=True), f64=True, policy="greedy", timeout=8),
    "greedy-cartpole-timeout": dict(kind="CartPole", policy="greedy", timeout=6),
    "q-linear": dict(kind="CartPole", policy="linear"),
    "q-exp": dict(kind="MountainCar", policy="exp", timeout=15),
    "q-speedy": dict(kind="CartPole", policy="speedy"),
    "q-weighted": dict(kind="CartPole", policy="weighted", act=1),
    "q-gumbel": dict(kind="MountainCar", policy="gumbel", timeout=12),
    "q-greedy": dict(kind="CartPole", policy="greedy-explorer"),
    "duel-linear": dict(kind="CartPole", policy="linear", dueling=True),
    "duel-gumbel": dict(kind="CartPole", policy="gumbel", dueling=True, act=1),
    "h128-greedy": dict(kind="CartPole", policy="greedy", hidden=128),
    "notc-sample-pendulum": dict(kind="Pendulum", envkw=dict(continuous=True), policy="sample", timeout=10, tc=False),
    "notc-q-exp": dict(kind="CartPole", policy="exp", tc=False),
    "h128-duel-greedy": dict(kind="MountainCar", policy="greedy-explorer", dueling=True, hidden=128, timeout=14),
}
EVAL_MODES = ("greedy", "sample")


def _set_tc(pkg, ctx, on):
    pkg._lib.check(ctx.lib.b200rl_set_tensor_cores(1 if on else 0))


def _make(pkg, ctx, cfg, n):
    kind = cfg["kind"]
    env = pkg.B200VecEnv(ctx, kind, n, O.splitmix_states_fast(n, 31), auto_reset=True, **cfg.get("envkw", {}))
    if cfg.get("f64"):
        env.set_state_float32()
    if cfg.get("timeout"):
        env.set_max_timeout(cfg["timeout"])
    hidden, act = cfg.get("hidden", 64), cfg.get("act", 0)
    if cfg["policy"] in EVAL_MODES:
        net = TE._net(pkg, ctx, env, kind, act, hidden)
        rng = O.splitmix_states_fast(n, 5150) if cfg["policy"] == "sample" else None
        pol = pkg.EvaluationPolicy(net, n, mode=cfg["policy"], rng=rng)
    else:
        net = TX._qnet(pkg, ctx, kind, hidden, act, cfg.get("dueling", False))
        name = "greedy" if cfg["policy"] == "greedy-explorer" else cfg["policy"]
        pol = TX._policy(pkg, ctx, net, TX._explorer(pkg, name, n * 60), n)
    return env, net, pol


def _streams(cfg, pol):
    if cfg["policy"] == "sample":
        return {"prng": pol.rng_state()}
    if cfg["policy"] not in EVAL_MODES:
        return {"xrng": pol.explorer_rng(), "xstep": np.array([getattr(pol.explorer, "step", 0)], np.int64)}
    return {}


def _net_state(pkg, net):
    st = {k: np.array(v, copy=True) for k, v in pkg.checkpoint.checkpoint(net=net).items()}
    st["step"] = np.array([net.step_count()], np.int64)
    if net.kind in (pkg.KIND_Q, pkg.KIND_DUELING):
        st["target"] = np.array(net.get(pkg.learners.NET_TARGET), copy=True)
    return st


def _same_env(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        x, y = np.ascontiguousarray(a[k]), np.ascontiguousarray(b[k])
        assert x.dtype == y.dtype and x.shape == y.shape, k
        if k == "env/episode_stats":   # {episodes, return sum, length sum, env steps}: the return sum is reduced in another order
            assert np.array_equal(x[[0, 2, 3]], y[[0, 2, 3]])
            assert abs(x[1] - y[1]) <= 1e-6 * max(1.0, abs(y[1])), (x[1], y[1])
            continue
        assert x.tobytes() == y.tobytes(), k


def _twin(pkg, ctx, cfg, stops, fused, n=N, hook_kind="log", cap=CAP, warm=0):
    """warm steps (the stage loop), then run(policy, env, stop, hook) for each stop of `stops` (factories)"""
    _set_tc(pkg, ctx, cfg.get("tc", True))
    try:
        env, net, pol = _make(pkg, ctx, cfg, n)
        if warm:
            pol.fusable = False
            pkg.run(pol, env, pkg.StopAfterNSteps(warm), StepCounts())
        net0 = _net_state(pkg, net)
        outs = []
        for make_stop in stops:
            stop = make_stop()
            pol.fusable = fused
            steps_before = env.episode_stats()["env_steps"] / n
            log = pkg.DeviceEpisodeLog(n, capacity=cap) if hook_kind == "log" else None
            counts, lengths = StepCounts(), pkg.BatchStepsPerEpisode(n)
            if fused:
                hook = log if log is not None else pkg.EmptyHook()
            else:
                hook = pkg.core.ComposedHook(counts, log if log is not None else lengths)
            l0 = ctx.launch_count()
            pkg.run(pol, env, stop, hook)
            launches = ctx.launch_count() - l0
            if log is not None:
                lists = (log.rewards, log.steps)
            else:
                lists = None if fused else lengths.steps
            outs.append(dict(steps=round(env.episode_stats()["env_steps"] / n - steps_before), cur=stop.cur, lists=lists,
                             env=pkg.checkpoint.checkpoint(env=env), streams=_streams(cfg, pol), launches=launches,
                             counts=None if fused else counts.counts, handle=pol._eval is not None))
            if log is not None:
                log.close()
        assert all(np.array_equal(v, _net_state(pkg, net)[k]) for k, v in net0.items()), "the network was written"
        pol.close(); net.close(); env.close()
    finally:
        _set_tc(pkg, ctx, True)
    return outs


def _probe(pkg, ctx, cfg, steps, n=N, warm=0):
    return _twin(pkg, ctx, cfg, [lambda: pkg.StopAfterNSteps(steps)], False, n=n, hook_kind="empty", warm=warm)[0]["counts"]


def _compare(pkg, ctx, cfg, stops, n=N, hook_kind="log", warm=0):
    a = _twin(pkg, ctx, cfg, stops, False, n=n, hook_kind=hook_kind, warm=warm)
    b = _twin(pkg, ctx, cfg, stops, True, n=n, hook_kind=hook_kind, warm=warm)
    for x, y in zip(a, b):
        assert y["handle"], "the fused path was not taken"
        assert (x["steps"], x["cur"]) == (y["steps"], y["cur"])
        _same_env(x["env"], y["env"])
        for k in x["streams"]:
            assert np.array_equal(x["streams"][k], y["streams"][k]), k
        if y["lists"] is not None:
            assert x["lists"] == y["lists"]
    return a, b


# (target step, exact hit, hook, where s* must land).  With DeviceEpisodeLog(capacity = 20) the windows are 20 steps; with EmptyHook
# a run whose budget is within 64 N episodes runs stretches of 64 steps.
CASES = {
    "first-step": (1, True, "log", lambda s: s == 1),
    "inside-window": (7, False, "log", lambda s: s % CAP != 0),
    "window-boundary": (CAP, True, "log", lambda s: s % CAP == 0),
    "inside-stretch": (30, True, "empty", lambda s: s % MARKED != 0),
    "stretch-last-step": (MARKED, True, "empty", lambda s: s == MARKED),
}


@pytest.mark.parametrize("config", sorted(CONFIGS))
@pytest.mark.parametrize("case", sorted(CASES))
def test_stops_where_the_stage_loop_stops(pkg, ctx, config, case):
    cfg = CONFIGS[config]
    target, exact, hook_kind, where = CASES[case]
    counts = _probe(pkg, ctx, cfg, 90)
    if not any(c > 0 and where(j + 1) for j, c in enumerate(counts) if j + 1 >= target):
        pytest.skip("no episode of this configuration ends on a step of the case (fixed-length episodes, or none on step 1)")
    k, s_star = budget_for(counts, target, exact, where=where)
    a, b = _compare(pkg, ctx, cfg, [lambda: pkg.StopAfterNEpisodes(k)], hook_kind=hook_kind)
    assert b[0]["steps"] == s_star and where(s_star) and b[0]["cur"] >= k


@pytest.mark.parametrize("config", ["greedy-cartpole", "sample-pendulum", "q-exp", "duel-gumbel", "h128-greedy", "notc-q-exp"])
def test_spent_budget_overshoot_and_second_run(pkg, ctx, config):
    cfg = CONFIGS[config]
    counts = _probe(pkg, ctx, cfg, 60, warm=5)
    k, _ = budget_for(counts, 4, exact=False)
    k2, _ = budget_for(counts[4:], 9, exact=True)
    for hook_kind in ("log", "empty"):
        a, b = _compare(pkg, ctx, cfg, [lambda: pkg.StopAfterNEpisodes(k), lambda: pkg.StopAfterNEpisodes(k2)], hook_kind=hook_kind, warm=5)
        assert b[0]["steps"] >= 4 and b[1]["steps"] >= 1
    for cur in (5, 9):      # budget 0 (cur >= k on entry): exactly one step
        a, b = _compare(pkg, ctx, cfg, [lambda: pkg.StopAfterNEpisodes(5, cur)], hook_kind="empty", warm=5)
        assert b[0]["steps"] == 1


@pytest.mark.parametrize("config", ["greedy-cartpole-timeout", "q-exp", "notc-sample-pendulum"])
def test_long_run_through_unmarked_stretches(pkg, ctx, config):
    """k >> 64 N: stretches of up to 1024 steps run unmarked (no shadow) before the marked ones that cross"""
    cfg, n = CONFIGS[config], 4
    steps = 2600
    counts = _probe(pkg, ctx, cfg, steps, n=n)
    k, s_star = budget_for(counts, 2300, exact=False)
    assert k > 2 * MARKED * n                               # the first stretches cannot reach the budget: they run unmarked
    a, b = _compare(pkg, ctx, cfg, [lambda: pkg.StopAfterNEpisodes(k)], n=n, hook_kind="empty")
    assert b[0]["steps"] == s_star
    if cfg.get("tc", True):   # one fused launch, a crossing kernel (and a mark) per stretch: far fewer launches than steps
        assert b[0]["launches"] < s_star // 8, (b[0]["launches"], s_star)


@pytest.mark.parametrize("config", ["greedy-cartpole", "sample-cartpole-f64", "greedy-pendulum", "q-speedy", "duel-linear",
                                    "h128-duel-greedy", "notc-sample-pendulum"])
@pytest.mark.parametrize("n", [1, 127, 1000, 65_537])
def test_stop_after_n_steps(pkg, ctx, config, n):
    """StopAfterNSteps: windows of the log's capacity (one launch each on the fused kernel) or one run of all steps"""
    cfg = CONFIGS[config]
    steps = 45 if n < 65_537 else 12
    for hook_kind in ("log", "empty"):
        a, b = _compare(pkg, ctx, cfg, [lambda: pkg.StopAfterNSteps(steps), lambda: pkg.StopAfterNSteps(7)], n=n, hook_kind=hook_kind)
        assert [x["steps"] for x in b] == [steps, 7]
        fused_kernel = cfg.get("tc", True) and cfg.get("hidden", 64) == 64
        for x, y in zip(a, b):
            windows = -(-x["steps"] // CAP) if hook_kind == "log" else 1
            if fused_kernel:   # the reset, then one launch per window (+ three launches per flush of the log, one more at the end)
                flushes = windows + 1 if hook_kind == "log" else 0
                assert y["launches"] <= 3 + windows + 3 * flushes, (y["launches"], windows)
            assert x["launches"] > x["steps"]


def test_stop_after_n_steps_longer_than_a_stretch(pkg, ctx):
    cfg = CONFIGS["q-linear"]
    a, b = _compare(pkg, ctx, cfg, [lambda: pkg.StopAfterNSteps(2500)], n=33, hook_kind="empty")
    assert b[0]["steps"] == 2500 and b[0]["launches"] <= 3 + -(-2500 // STRETCH_MAX)


# ---- refusals -----------------------------------------------------------------------------------------------------------------
def test_refusals_leave_everything_untouched(pkg, ctx):
    L, lib, n = pkg._lib, ctx.lib, 64

    def create(net, env, mode):
        h = C.c_void_p()
        st = lib.b200rl_eval_create(net.h, env.h, mode, C.byref(h))
        if st == L.OK:
            lib.b200rl_eval_destroy(h)
        return st

    cp = pkg.B200VecEnv(ctx, "CartPole", n, O.splitmix_states_fast(n, 1), auto_reset=True)
    cp64 = pkg.B200VecEnv(ctx, "CartPole", n, O.splitmix_states_fast(n, 1), auto_reset=True, T=np.float64)
    acro = pkg.B200VecEnv(ctx, "Acrobot", n, O.splitmix_states_fast(n, 1), auto_reset=True, T=np.float64)
    pend = pkg.B200VecEnv(ctx, "Pendulum", n, O.splitmix_states_fast(n, 1), auto_reset=True, continuous=True)
    mc = pkg.B200VecEnv(ctx, "MountainCar", n, O.splitmix_states_fast(n, 1), auto_reset=True)
    ac = TE._net(pkg, ctx, cp, "CartPole", 0)
    q = TX._qnet(pkg, ctx, "CartPole", 64, 0, False)
    gauss = TE._net(pkg, ctx, pend, "Pendulum", 0)
    qp = pkg.Network(ctx, 3, 64, 1, O.glorot_params(O.ac_desc(3, 64, 1, 0), 3, q_net=True), act=0, kind=pkg.KIND_Q)
    envs = (cp, cp64, acro, pend, mc)
    before = [pkg.checkpoint.checkpoint(env=e) for e in envs]
    assert create(ac, cp64, 0) == L.ERR_UNSUPPORTED          # Float64 without set_state_float32
    assert create(ac, acro, 0) == L.ERR_UNSUPPORTED
    assert create(q, cp, 1) == L.ERR_UNSUPPORTED             # mode 1 on a Q-network
    assert create(qp, pend, 2) == L.ERR_UNSUPPORTED          # a Q-network on a continuous env
    assert create(ac, mc, 0) == L.ERR_INVALID                # input width
    assert create(gauss, cp, 0) == L.ERR_INVALID             # Gaussian head on a discrete env
    assert create(ac, cp, 2) == L.ERR_INVALID                # mode 2 needs a Q-network
    assert create(ac, cp, 3) == L.ERR_INVALID
    for e, b in zip(envs, before):
        _same_env(b, pkg.checkpoint.checkpoint(env=e))

    # run_episodes on a valid handle: refused before any side effect
    pol = TX._policy(pkg, ctx, q, pkg.EpsilonGreedyExplorer(0.1), n)
    h = pol.eval_handle(cp)
    assert h is not None
    b_env, b_rng = pkg.checkpoint.checkpoint(env=cp), pol.explorer_rng()
    steps, eps = C.c_int64(-1), C.c_int64(-1)

    def run(ex, max_steps=10, budget=-1, rng=C.c_void_p(pol._d_rng)):
        return lib.b200rl_eval_run_episodes(h, rng, ex, max_steps, budget, C.byref(steps), C.byref(eps))
    good = pol.explorer.as_struct()
    assert run(C.byref(good), max_steps=0) == L.ERR_INVALID
    assert run(C.byref(good), rng=None) == L.ERR_INVALID
    bad = pol.explorer.as_struct(); bad.eps_stable = 2.0
    assert run(C.byref(bad)) == L.ERR_INVALID
    big = pol.explorer.as_struct(); big.step = (1 << 62) - 5
    assert run(C.byref(big)) == L.ERR_INVALID                  # explorer step overflow
    assert (steps.value, eps.value, good.step, big.step) == (-1, -1, pol.explorer.step, (1 << 62) - 5)
    _same_env(b_env, pkg.checkpoint.checkpoint(env=cp))
    assert np.array_equal(b_rng, pol.explorer_rng())
    pol.close()
    for x in (ac, q, gauss, qp):
        x.close()
    for e in envs:
        e.close()


def test_sharded_budget_is_refused_and_steps_equal_one_rank_over_the_union(pkg):
    """A budget on a sharded ctx: B200RL_ERR_UNSUPPORTED with nothing touched (run() keeps the stage loop).  StopAfterNSteps on the
    shards of two ranks (columns numbered over the union) equals one rank over the union."""
    L, n, steps = pkg._lib, 300, 37
    seeds, xseeds = O.splitmix_states_fast(2 * n, 41), O.splitmix_states_fast(2 * n, 42)
    one = pkg.Context(0)
    ctxs = SH._two_ranks(pkg)
    try:
        def make(ctx, sl):
            env = pkg.B200VecEnv(ctx, "CartPole", sl.stop - sl.start, seeds[sl], auto_reset=True)
            net = TX._qnet(pkg, ctx, "CartPole", 64, 0, False)
            pol = pkg.QBasedPolicy(ctx, types.SimpleNamespace(net=net), TX._explorer(pkg, "linear", 2 * n * steps), xseeds[sl],
                                   sl.stop - sl.start)
            return env, net, pol
        env_u, net_u, pol_u = make(one, slice(0, 2 * n))
        pkg.run(pol_u, env_u, pkg.StopAfterNSteps(steps), pkg.EmptyHook())
        assert pol_u._eval is not None
        for r, ctx in enumerate(ctxs):
            env, net, pol = make(ctx, slice(r * n, (r + 1) * n))
            h = pol.eval_handle(env)
            before, ex = pkg.checkpoint.checkpoint(env=env), pol.explorer.as_struct()
            s, e = C.c_int64(-1), C.c_int64(-1)
            st = ctx.lib.b200rl_eval_run_episodes(h, C.c_void_p(pol._d_rng), C.byref(ex), 100, 10, C.byref(s), C.byref(e))
            assert st == L.ERR_UNSUPPORTED and (s.value, e.value) == (-1, -1) and ex.step == pol.explorer.step
            _same_env(before, pkg.checkpoint.checkpoint(env=env))
            pkg.run(pol, env, pkg.StopAfterNSteps(steps), pkg.EmptyHook())
            assert pol.explorer.step == pol_u.explorer.step
            sl = slice(r * n, (r + 1) * n)
            assert np.array_equal(env.internal_state(), env_u.internal_state()[:, sl])
            for f in ("t", "flags", "reward", "last_action"):
                assert np.array_equal(getattr(env, f)(), getattr(env_u, f)()[sl]), f
            assert np.array_equal(env.rng_state(), env_u.rng_state()[sl])
            assert np.array_equal(pol.explorer_rng(), pol_u.explorer_rng()[sl])
            pol.close(); net.close(); env.close()
        pol_u.close(); net_u.close(); env_u.close()
    finally:
        for c in ctxs:
            c.close()
        one.close()
