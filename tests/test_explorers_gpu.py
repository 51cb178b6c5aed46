"""GPU tests of the speedy and softmax explorers (b200rl_explorer kinds 2-4) on the device DQN path.

b200rl_net_q_explore against the host-compiled explore.cuh on the Q-values net_values returns, bit for bit with the streams;
the device agent loop (fused H = 64 collect, staged H = 128, graphs) against the stage protocol over checkpoint_replay; one
fused launch per update-free window; a mid-run checkpoint restored into other seeds; a change of kind or beta between runs;
refusals before any side effect."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from test_explorers_host import header_plan, xh  # noqa: F401  (xh: the host-compiled header, a fixture)

pytestmark = pytest.mark.gpu

_NA = {"CartPole": 2, "MountainCar": 3, "Pendulum": 3}
_NS = {"CartPole": 4, "MountainCar": 2, "Pendulum": 3}


def _explorer(pkg, kind, beta=2e-4, step=1):
    return {"speedy": lambda: pkg.EpsilonSpeedyExplorer(beta, step=step), "weighted": pkg.WeightedSoftmaxExplorer,
            "gumbel": pkg.GumbelSoftmaxExplorer}[kind]()


_KIND = {"speedy": 2, "weighted": 3, "gumbel": 4}


@pytest.mark.parametrize("kind", ["speedy", "weighted", "gumbel"])
@pytest.mark.parametrize("H,act,tc,N", [(64, 0, True, 65537), (64, 1, False, 127), (128, 1, True, 127), (128, 0, False, 1),
                                        (64, 0, True, 1), (128, 0, True, 65537)])
def test_q_explore_matches_the_host_header(pkg, ctx, xh, kind, H, act, tc, N):  # noqa: F811
    ns, na = 4, 3 if kind != "weighted" else 4
    p = O.glorot_params(O.ac_desc(ns, H, na, act), 5, q_net=True) * np.float32(3.0)    # spread-out Q-values
    net = pkg.Network(ctx, ns, H, na, p.astype(np.float32), act=act, kind=pkg.KIND_Q)
    obs = np.asfortranarray(np.random.default_rng(N).standard_normal((ns, N)).astype(np.float32))
    rng = O.splitmix_states_fast(N, 11)
    ex = _explorer(pkg, kind, beta=1e-5, step=40)
    dobs, dact, drng = ctx.malloc(obs.nbytes), ctx.malloc(N * 4), ctx.malloc(rng.nbytes)
    ctx.h2d(dobs, obs); ctx.h2d(drng, rng)
    ctx.lib.b200rl_set_tensor_cores(1 if tc else 0)
    try:
        q = net.values(obs)
        st = ex.as_struct()
        assert ctx.lib.b200rl_net_q_explore(net.h, C.c_void_p(dobs), N, C.c_void_p(drng), C.byref(st), C.c_void_p(dact)) == 0
        got, grng = ctx.d2h(np.empty(N, np.int32), dact), ctx.d2h(np.empty_like(rng), drng)
        ref, rref = header_plan(xh, pkg, _KIND[kind], q, rng, 40, 1e-5)
        assert np.array_equal(got, ref) and np.array_equal(grng, rref)
        if N > 1000:
            assert len(np.unique(got)) == na
    finally:
        ctx.lib.b200rl_set_tensor_cores(1)
        for d in (dobs, dact, drng):
            ctx.free(d)
        net.close()


def _setup(pkg, ctx, seed, env_kind="CartPole", lanes=127, hidden=64, act=0, cap=16, B=256, prioritized=True, explorer="speedy",
           beta=2e-4, ratio=1.0, threshold=3, target_freq=5, n_step=1, dueling=False):
    kw = dict(params=pkg.pendulum_params(continuous=False, n_actions=3)) if env_kind == "Pendulum" else {}
    env = pkg.B200VecEnv(ctx, env_kind, lanes, O.splitmix_states_fast(lanes, seed), auto_reset=True, **kw)
    ns, na = _NS[env_kind], _NA[env_kind]
    if dueling:
        import dueling_ref as D
        net = pkg.Network(ctx, ns, hidden, na, D.glorot_params(ns, hidden, na, seed + 1), act=act, kind=pkg.KIND_DUELING)
    else:
        net = pkg.Network(ctx, ns, hidden, na, O.glorot_params(O.ac_desc(ns, hidden, na, act), seed + 1, q_net=True), act=act, kind=pkg.KIND_Q)
    traj = pkg.Trajectory(ctx, ns, cap, lanes=lanes, batch_size=B, sampler_rng=O.splitmix_states_fast(B, seed + 2), prioritized=prioritized)
    if n_step > 1:
        traj.set_nstep(n_step, 0.99)
    traj.controller = pkg.InsertSampleRatioController(ratio=ratio, threshold=threshold)
    learner = pkg.DQNLearner(ctx, net, traj, pkg.dqn_config(target_update_freq=target_freq))
    policy = pkg.QBasedPolicy(ctx, learner, _explorer(pkg, explorer, beta), O.splitmix_states_fast(lanes, seed + 3), lanes)
    return dict(env=env, net=net, traj=traj, policy=policy, agent=pkg.Agent(policy, traj), learner=learner)


def _close(s):
    s["agent"].close()
    for k in ("policy", "traj", "net", "env"):
        s[k].close()


def _state(pkg, s):
    ck = pkg.checkpoint.checkpoint_replay(s["env"], s["net"], s["agent"])
    ck["env/episode_stats"] = ck["env/episode_stats"].copy()
    return ck


def _assert_same(a, b, pendulum=False):
    assert sorted(a) == sorted(b)
    for k in a:
        if k == "env/episode_stats" and pendulum:
            assert np.array_equal(a[k][[0, 2, 3]], b[k][[0, 2, 3]])
            np.testing.assert_allclose(a[k][1], b[k][1], rtol=1e-12)
            continue
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


def _run_both(pkg, ctx, windows, switch=None, **kw):
    fast, stage = _setup(pkg, ctx, 100, **kw), _setup(pkg, ctx, 100, **kw)
    stage["agent"].fusable = False
    for j, n in enumerate(windows):
        if switch and j in switch:
            for s in (fast, stage):
                s["policy"].explorer = switch[j](pkg)
        pkg.run(fast["agent"], fast["env"], pkg.StopAfterNSteps(n), pkg.EmptyHook())
        pkg.run(stage["agent"], stage["env"], pkg.StopAfterNSteps(n), pkg.EmptyHook())
    assert fast["agent"]._replay is not None and stage["agent"]._replay is None
    _assert_same(_state(pkg, fast), _state(pkg, stage), pendulum=kw.get("env_kind") == "Pendulum")
    ca, cb = fast["traj"].controller, stage["traj"].controller
    assert (ca.n_inserted, ca.n_sampled) == (cb.n_inserted, cb.n_sampled)
    return fast, stage


CASES = [
    dict(env_kind="CartPole", hidden=64, explorer="speedy"),
    dict(env_kind="CartPole", hidden=64, explorer="weighted", act=1, prioritized=False),
    dict(env_kind="CartPole", hidden=64, explorer="gumbel", ratio=0.25, threshold=1),
    dict(env_kind="MountainCar", hidden=128, explorer="speedy", act=1, ratio=0.25, threshold=2, prioritized=False),
    dict(env_kind="MountainCar", hidden=64, explorer="gumbel", n_step=3),
    dict(env_kind="Pendulum", hidden=64, explorer="weighted", dueling=True, target_freq=3),
    dict(env_kind="Pendulum", hidden=128, explorer="gumbel", act=1, dueling=True),
    dict(env_kind="CartPole", hidden=128, explorer="weighted", n_step=3, ratio=0.25, threshold=1, target_freq=3),
    dict(env_kind="MountainCar", hidden=64, explorer="weighted", cap=8, threshold=100),      # update-free windows, ring wrap
    dict(env_kind="Pendulum", hidden=64, explorer="speedy", beta=0.05, prioritized=False, target_freq=2),
]


@pytest.mark.parametrize("case", CASES, ids=[f"{c['env_kind']}-H{c['hidden']}-{c['explorer']}-{i}" for i, c in enumerate(CASES)])
def test_device_loop_equals_stage_protocol(pkg, ctx, case):
    fast, stage = _run_both(pkg, ctx, [23, 6], **case)
    if case["explorer"] == "speedy":
        assert fast["policy"].explorer.step == 1 + 29 * 127
    _close(fast); _close(stage)


def test_switching_kind_or_beta_recaptures(pkg, ctx):
    switch = {1: lambda p: p.GumbelSoftmaxExplorer(), 2: lambda p: p.EpsilonSpeedyExplorer(1e-3, step=500),
              3: lambda p: p.EpsilonSpeedyExplorer(0.2, step=500), 4: lambda p: p.WeightedSoftmaxExplorer(),
              5: lambda p: p.EpsilonGreedyExplorer(0.1)}
    fast, stage = _run_both(pkg, ctx, [9, 9, 9, 9, 9, 9], switch=switch, env_kind="CartPole", hidden=64, explorer="weighted",
                            threshold=1)
    assert fast["agent"].graph_active()
    _close(fast); _close(stage)


@pytest.mark.parametrize("kind", ["speedy", "weighted", "gumbel"])
def test_a_window_without_updates_is_one_fused_launch(pkg, ctx, kind):
    s = _setup(pkg, ctx, 9, explorer=kind, threshold=1000)
    pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(2), pkg.EmptyHook())
    l0 = ctx.launch_count()
    pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(40), pkg.EmptyHook())
    assert ctx.launch_count() - l0 <= 8
    _close(s)


@pytest.mark.parametrize("kind", ["speedy", "gumbel"])
def test_checkpoint_mid_run_restores_and_continues(pkg, ctx, kind):
    ck_mod = pkg.checkpoint
    a = _setup(pkg, ctx, 300, explorer=kind, threshold=2, target_freq=3)
    pkg.run(a["agent"], a["env"], pkg.StopAfterNSteps(9), pkg.EmptyHook())
    ck = ck_mod.checkpoint_replay(a["env"], a["net"], a["agent"])
    pkg.run(a["agent"], a["env"], pkg.StopAfterNSteps(11), pkg.EmptyHook())
    final_a = _state(pkg, a)
    b = _setup(pkg, ctx, 999, explorer=kind, threshold=2, target_freq=3)
    pkg.run(b["agent"], b["env"], pkg.StopAfterNSteps(4), pkg.EmptyHook())
    ck_mod.restore_replay(ck, b["env"], b["net"], b["agent"])
    pkg.run(b["agent"], b["env"], pkg.StopAfterNSteps(11), pkg.EmptyHook())
    _assert_same(final_a, _state(pkg, b))
    if kind == "speedy":
        assert b["policy"].explorer.step == a["policy"].explorer.step == 1 + 20 * 127
    _close(a); _close(b)


def _refused(pkg, s, call):
    before = _state(pkg, s)
    assert call() == pkg._lib.ERR_INVALID
    _assert_same(before, _state(pkg, s))


def test_refusals_leave_everything_untouched(pkg, ctx):
    lib = ctx.lib
    s = _setup(pkg, ctx, 11, lanes=64, explorer="speedy")
    pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(5), pkg.EmptyHook())
    r, rng = s["agent"]._replay, C.c_void_p(s["policy"]._d_rng)
    obs = C.c_void_p(s["env"].device_ptr(pkg._lib.FIELD_OBS))
    act = ctx.malloc(64 * 4)
    bads = []
    for kind, beta in ((5, 0.0), (-1, 0.0), (2, float("nan")), (2, float("inf")), (2, float("-inf")), (3, 0.5), (4, 1.0)):
        e = s["policy"].explorer.as_struct()
        e.kind, e.beta = kind, beta
        bads.append(e)
    for field, v in (("eps_stable", 0.1), ("eps_init", 1.0), ("warmup_steps", 3), ("decay_steps", 5), ("is_break_tie", 1)):
        for kind in (2, 3, 4):                                       # an ε-greedy field on a kind that does not read it
            e = s["policy"].explorer.as_struct()
            e.kind = kind
            if kind != 2:
                e.beta = 0.0
            setattr(e, field, v)
            bads.append(e)
    for e in bads:
        ctl = pkg._lib.InsertSampleRatio(1.0, 1, 5, 3)
        _refused(pkg, s, lambda: lib.b200rl_replay_run(r, rng, C.byref(e), C.byref(ctl), 4, None))
        _refused(pkg, s, lambda: lib.b200rl_net_q_explore(s["net"].h, obs, 64, rng, C.byref(e), C.c_void_p(act)))
    for ex in (pkg.EpsilonSpeedyExplorer(0.1), pkg.WeightedSoftmaxExplorer(), pkg.GumbelSoftmaxExplorer()):
        e = ex.as_struct()
        ctl = pkg._lib.InsertSampleRatio(1.0, 1, 5, 3)
        _refused(pkg, s, lambda: lib.b200rl_replay_run(r, None, C.byref(e), C.byref(ctl), 4, None))     # no explorer streams
        _refused(pkg, s, lambda: lib.b200rl_net_q_explore(s["net"].h, obs, 64, None, C.byref(e), C.c_void_p(act)))
    ctx.free(act)
    _close(s)
