"""GPU tests of the device DQN agent loop (b200rl_replay_run): run(Agent(QBasedPolicy(DQNLearner, explorer), Trajectory), env,
StopAfterNSteps(n)) with a hook that has nothing to do per step runs on the device — collect launches, updates replayed as CUDA
graphs — and must leave exactly the state the stage protocol (agent.fusable = False) leaves: env fields and streams, the
Q-network (parameters, Adam state, beta^t, target, step), the ring with its sum tree, n_sampleable and sampler streams, the
explorer streams and step, the controller counters, the last TD errors and the episode statistics, bit for bit."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu

_NA = {"CartPole": 2, "MountainCar": 3, "Pendulum": 3}
_NS = {"CartPole": 4, "MountainCar": 2, "Pendulum": 3}


def _setup(pkg, ctx, seed, env_kind="CartPole", lanes=127, hidden=64, act=0, cap=16, B=256, prioritized=True, explorer="linear",
           ratio=1.0, threshold=3, huber=True, double_dqn=False, target_freq=5, max_timeout=0):
    kw = dict(params=pkg.pendulum_params(continuous=False, n_actions=3)) if env_kind == "Pendulum" else {}
    env = pkg.B200VecEnv(ctx, env_kind, lanes, O.splitmix_states_fast(lanes, seed), auto_reset=True, **kw)
    if max_timeout:
        env.set_max_timeout(max_timeout)
    ns, na = _NS[env_kind], _NA[env_kind]
    net = pkg.Network(ctx, ns, hidden, na, O.glorot_params(O.ac_desc(ns, hidden, na, act), seed + 1, q_net=True), act=act, kind=pkg.KIND_Q)
    traj = pkg.Trajectory(ctx, ns, cap, lanes=lanes, batch_size=B, sampler_rng=O.splitmix_states_fast(B, seed + 2), prioritized=prioritized)
    traj.controller = pkg.InsertSampleRatioController(ratio=ratio, threshold=threshold)
    learner = pkg.DQNLearner(ctx, net, traj, pkg.dqn_config(huber=huber, double_dqn=double_dqn, target_update_freq=target_freq))
    if explorer == "greedy":
        ex = pkg.GreedyExplorer()
    else:
        ex = pkg.EpsilonGreedyExplorer(0.05, kind="exp" if explorer == "exp" else "linear", eps_init=1.0, warmup_steps=2 * lanes,
                                       decay_steps=10 * lanes, is_break_tie=explorer == "break_tie")
    policy = pkg.QBasedPolicy(ctx, learner, ex, O.splitmix_states_fast(lanes, seed + 3), lanes)
    agent = pkg.Agent(policy, traj)
    return dict(env=env, net=net, traj=traj, policy=policy, agent=agent, learner=learner)


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
            assert np.array_equal(a[k][[0, 2, 3]], b[k][[0, 2, 3]])      # counts and length sums exact; the return sum
            np.testing.assert_allclose(a[k][1], b[k][1], rtol=1e-12)     # may only be reordered
            continue
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


def _run_both(pkg, ctx, steps, reentry=0, **kw):
    fast, stage = _setup(pkg, ctx, 100, **kw), _setup(pkg, ctx, 100, **kw)
    stage["agent"].fusable = False
    for n in [steps] + ([reentry] if reentry else []):
        pkg.run(fast["agent"], fast["env"], pkg.StopAfterNSteps(n), pkg.EmptyHook())
        pkg.run(stage["agent"], stage["env"], pkg.StopAfterNSteps(n), pkg.EmptyHook())
    assert fast["agent"]._replay is not None and stage["agent"]._replay is None      # the two paths really differ
    a, b = _state(pkg, fast), _state(pkg, stage)
    _assert_same(a, b, pendulum=kw.get("env_kind") == "Pendulum")
    ca, cb = fast["traj"].controller, stage["traj"].controller
    assert (ca.n_inserted, ca.n_sampled) == (cb.n_inserted, cb.n_sampled)
    if ca.ratio >= 1.0 and ca.n_inserted > ca.threshold:
        # every step after the threshold trains: the last update's TD errors are where b200rl_dqn_update leaves them
        assert np.array_equal(fast["learner"].last_td(), stage["learner"].last_td())
    return fast, stage


CASES = [
    dict(env_kind="CartPole", hidden=64, act=0),
    dict(env_kind="CartPole", hidden=128, act=1, prioritized=False, explorer="exp", huber=False, double_dqn=True),
    dict(env_kind="MountainCar", hidden=64, act=1, explorer="break_tie", ratio=2.0),
    dict(env_kind="Pendulum", hidden=64, act=0, explorer="greedy", ratio=0.25, threshold=1),
    dict(env_kind="CartPole", hidden=64, act=0, ratio=1.0, threshold=100),            # the threshold delays learning past the window
    dict(env_kind="CartPole", hidden=128, act=0, cap=8, target_freq=7, max_timeout=9),  # ring wrap-around, MaxTimeoutEnv
    dict(env_kind="MountainCar", hidden=128, act=1, lanes=1, B=32, ratio=0.25, threshold=2),
    dict(env_kind="CartPole", hidden=64, act=1, lanes=1000, explorer="exp", double_dqn=True),
    # H = 64 windows without an update run as one fused launch: the whole window, and one that wraps the ring several times
    dict(env_kind="CartPole", hidden=64, act=0, cap=8, threshold=100, max_timeout=7),
    dict(env_kind="MountainCar", hidden=64, act=0, prioritized=False, explorer="exp", ratio=0.25, threshold=5),
    dict(env_kind="Pendulum", hidden=64, act=1, explorer="break_tie", ratio=0.25, threshold=9, cap=6),
]


@pytest.mark.parametrize("case", CASES, ids=[f"{c['env_kind']}-H{c['hidden']}-{i}" for i, c in enumerate(CASES)])
def test_device_loop_equals_stage_protocol(pkg, ctx, case):
    fast, stage = _run_both(pkg, ctx, 23, reentry=6, **case)
    _close(fast); _close(stage)


def test_device_loop_with_tensor_cores_off(pkg, ctx):
    ctx.lib.b200rl_set_tensor_cores(0)
    try:
        fast, stage = _run_both(pkg, ctx, 17, env_kind="CartPole", hidden=64, act=0, explorer="exp")
    finally:
        ctx.lib.b200rl_set_tensor_cores(1)
    _close(fast); _close(stage)


def test_device_loop_65536_lanes(pkg, ctx):
    fast, stage = _run_both(pkg, ctx, 12, env_kind="CartPole", lanes=65536, hidden=64, cap=8, B=4096, threshold=2, target_freq=4)
    _close(fast); _close(stage)


def test_a_window_without_updates_is_one_fused_launch(pkg, ctx):
    s = _setup(pkg, ctx, 9, ratio=1.0, threshold=1000)                             # H = 64, prioritised, no update in the window
    pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(2), pkg.EmptyHook())        # (warm-up: kernel attributes)
    l0 = ctx.launch_count()
    pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(40), pkg.EmptyHook())
    l1 = ctx.launch_count()
    # the forced reset + episode-start push of run(), then collect + explorer-step tick + one sum-tree rebuild (staged: 6 per step)
    assert l1 - l0 <= 8, l1 - l0
    _close(s)


def test_graphs_are_replayed_after_warm_up(pkg, ctx):
    s = _setup(pkg, ctx, 7, ratio=1.0, threshold=1)
    assert not s["agent"].graph_active()
    pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(10), pkg.EmptyHook())
    assert s["agent"].graph_active()                                              # units of "1 step + 1 update" replayed
    assert s["net"].step_count() == 10 and s["policy"].explorer.step == 1 + 10 * 127
    _close(s)


def test_checkpoint_mid_run_restores_and_continues(pkg, ctx):
    ck_mod = pkg.checkpoint
    a = _setup(pkg, ctx, 300, ratio=1.0, threshold=2, target_freq=3)
    pkg.run(a["agent"], a["env"], pkg.StopAfterNSteps(9), pkg.EmptyHook())
    ck = ck_mod.checkpoint_replay(a["env"], a["net"], a["agent"])
    ctl = a["traj"].controller
    ctl_state = (ctl.n_inserted, ctl.n_sampled)
    pkg.run(a["agent"], a["env"], pkg.StopAfterNSteps(11), pkg.EmptyHook())
    final_a = _state(pkg, a)

    b = _setup(pkg, ctx, 999, ratio=1.0, threshold=2, target_freq=3)                # other seeds
    pkg.run(b["agent"], b["env"], pkg.StopAfterNSteps(4), pkg.EmptyHook())
    ck_mod.restore_replay(ck, b["env"], b["net"], b["agent"])
    assert (b["traj"].controller.n_inserted, b["traj"].controller.n_sampled) == ctl_state
    pkg.run(b["agent"], b["env"], pkg.StopAfterNSteps(11), pkg.EmptyHook())
    _assert_same(final_a, _state(pkg, b))
    _close(a); _close(b)


def _refused(pkg, ctx, s, call):
    before = _state(pkg, s)
    assert call() != pkg._lib.OK
    _assert_same(before, _state(pkg, s))


def test_refusals_leave_everything_untouched(pkg, ctx):
    lib = ctx.lib
    s = _setup(pkg, ctx, 11, lanes=64)
    pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(5), pkg.EmptyHook())
    net, env, traj, cfg = s["net"], s["env"], s["traj"], s["learner"].cfg
    h = C.c_void_p()
    # network that is not a Q-network
    ac = pkg.Network(ctx, 4, 64, 2, O.glorot_params(O.ac_desc(4, 64, 2), 1), kind=pkg.KIND_CATEGORICAL)
    _refused(pkg, ctx, s, lambda: lib.b200rl_replay_create(ctx.h, ac.h, env.h, traj.h, C.byref(cfg), C.byref(h)))
    ac.close()
    # Float64, continuous and Acrobot envs; lanes != N
    for kind, kwargs in (("CartPole", dict(T=np.float64)), ("ContinuousCartPole", {}), ("Acrobot", dict(T=np.float64)), ("CartPole", {})):
        n = 63 if not kwargs and kind == "CartPole" else 64
        e = pkg.B200VecEnv(ctx, kind, n, O.splitmix_states_fast(n, 3), auto_reset=True, **kwargs)
        _refused(pkg, ctx, s, lambda: lib.b200rl_replay_create(ctx.h, net.h, e.h, traj.h, C.byref(cfg), C.byref(h)))
        e.close()
    # state width mismatch (a 2-wide ring)
    t2 = pkg.Trajectory(ctx, 2, 8, lanes=64, batch_size=16, sampler_rng=O.splitmix_states_fast(16, 1))
    _refused(pkg, ctx, s, lambda: lib.b200rl_replay_create(ctx.h, net.h, env.h, t2.h, C.byref(cfg), C.byref(h)))
    t2.close()
    # bad explorer schedule / controller values on a live handle
    r = s["agent"]._replay
    rng = C.c_void_p(s["policy"]._d_rng)
    ex = s["policy"].explorer.as_struct()
    for bad in (dict(eps_stable=1.5), dict(kind=3), dict(decay_steps=-1)):
        e2 = s["policy"].explorer.as_struct()
        for k, v in bad.items():
            setattr(e2, k, v)
        ctl = pkg._lib.InsertSampleRatio(1.0, 1, 5, 3)
        _refused(pkg, ctx, s, lambda: lib.b200rl_replay_run(r, rng, C.byref(e2), C.byref(ctl), 4, None))
    for ratio, ni, ns in ((float("inf"), 5, 3), (float("nan"), 5, 3), (-1.0, 5, 3), (1.0, -1, 0)):
        ctl = pkg._lib.InsertSampleRatio(ratio, 1, ni, ns)
        _refused(pkg, ctx, s, lambda: lib.b200rl_replay_run(r, rng, C.byref(ex), C.byref(ctl), 4, None))
    ctl = pkg._lib.InsertSampleRatio(1.0, 1, 5, 3)
    _refused(pkg, ctx, s, lambda: lib.b200rl_replay_run(r, None, C.byref(ex), C.byref(ctl), 4, None))   # no explorer streams
    _close(s)


def test_stats_of_the_last_update(pkg, ctx):
    s = _setup(pkg, ctx, 5, ratio=1.0, threshold=1)
    st = s["agent"].run_replay(s["env"], 6, want_stats=True)
    assert st["n_updates"] == s["net"].step_count() == 6
    assert np.isfinite(st["loss"]) and st["grad_norm"] > 0
    np.testing.assert_allclose(st["mean_abs_td"], np.abs(s["learner"].last_td()).astype(np.float64).mean(), rtol=1e-6)
    _close(s)
