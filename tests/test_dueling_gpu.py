"""GPU tests of the dueling Q-network (kind 3, DuelingNetwork networks.jl:500-522) on the device DQN path.

Forward (values / act_greedy / q_explore) against the oracle's head rows combined by the restatement; the DQN update against
float64 autograd and the oracle's clip + Adam; the device agent loop and the fused evaluation against the stage protocol bit for
bit; a known answer; refusals of the actor-critic entry points before any side effect."""
import ctypes as C

import numpy as np
import pytest

import dueling_ref as D
import oracle_lib as O

pytestmark = pytest.mark.gpu

_NA = {"CartPole": 2, "MountainCar": 3, "Pendulum": 3}
_NS = {"CartPole": 4, "MountainCar": 2, "Pendulum": 3}


def _params(ns, H, n, seed, scale=0.05):
    return (D.glorot_params(ns, H, n, seed) + np.float32(scale) * np.random.default_rng(seed + 1).standard_normal(D.nparams(ns, H, n))
            .astype(np.float32)).astype(np.float32)


def _tc(ctx, on):
    ctx.lib.b200rl_set_tensor_cores(1 if on else 0)


@pytest.mark.parametrize("H,act,tc,n,ns", [(64, 0, True, 2, 4), (64, 1, True, 3, 3), (64, 0, False, 3, 2), (128, 1, False, 2, 4),
                                           (128, 0, True, 1, 4)])
def test_forward_against_the_oracle(pkg, ctx, H, act, tc, n, ns):
    N = 1000                                                   # not a multiple of the 128 / 64-sample tiles
    p = _params(ns, H, n, 3)
    obs = np.asfortranarray(np.random.default_rng(4).standard_normal((ns, N)).astype(np.float32))
    net = pkg.Network(ctx, ns, H, n, p, act=act, kind=pkg.KIND_DUELING)
    _tc(ctx, tc)
    try:
        q = net.values(obs)
        qt = net.values(obs, use_target=True)
        assert q.shape == (n, N) and np.array_equal(q, qt)     # the target starts as a copy
        ref = D.oracle_q(p, ns, H, n, act, obs)
        np.testing.assert_allclose(q, ref, rtol=1e-5, atol=3e-6)
        # greedy / explorer columns select on exactly the Q that values() returns
        dobs = ctx.malloc(obs.nbytes); ctx.h2d(dobs, obs)
        dact = ctx.malloc(N * 4)
        assert ctx.lib.b200rl_net_act_greedy(net.h, C.c_void_p(dobs), N, C.c_void_p(dact), 1) == 0
        a = ctx.d2h(np.empty(N, np.int32), dact)
        assert np.array_equal(a, q.argmax(0) + 1)
        ex6 = O.explorer6(0.3, eps_init=1.0, warmup_steps=10, decay_steps=500)
        ex = pkg.EpsilonGreedyExplorer(0.3, eps_init=1.0, warmup_steps=10, decay_steps=500, step=7)
        rng = O.splitmix_states_fast(N, 9)
        drng = ctx.malloc(rng.nbytes); ctx.h2d(drng, rng)
        st = ex.as_struct()
        assert ctx.lib.b200rl_net_q_explore(net.h, C.c_void_p(dobs), N, C.c_void_p(drng), C.byref(st), C.c_void_p(dact)) == 0
        got = ctx.d2h(np.empty(N, np.int32), dact)
        r2 = rng.copy()
        assert np.array_equal(got, O.egreedy_plan(ex6, 7, q, r2))
        for d in (dobs, dact, drng):
            ctx.free(d)
    finally:
        _tc(ctx, True)
        net.close()


def _fill(pkg, ctx, ns, lanes, cap, frames, prioritized, B, seed, n_actions):
    tr = pkg.Trajectory(ctx, ns, cap, lanes=lanes, batch_size=B, sampler_rng=O.splitmix_states_fast(B, 900 + seed), prioritized=prioritized)
    ref = O.OracleTraj(ns, lanes, cap, prioritized, 1.0)
    rng = np.random.default_rng(seed)
    obs = rng.standard_normal((ns, lanes)).astype(np.float32)
    tr.push_state(obs); ref.push_state(obs)
    for _ in range(frames):
        a, r = rng.integers(1, n_actions + 1, lanes).astype(np.int32), rng.standard_normal(lanes).astype(np.float32)
        t, obs = (rng.random(lanes) < 0.1).astype(np.uint8), rng.standard_normal((ns, lanes)).astype(np.float32)
        tr.push(a, r, t, obs); ref.push(a, r, t, obs)
    return tr, ref


@pytest.mark.parametrize("H,huber,double_dqn,prioritized,n_step,n", [(128, True, False, True, 1, 2), (64, False, False, False, 1, 3),
                                                                     (128, True, True, True, 3, 3), (64, True, True, False, 3, 2),
                                                                     (64, False, False, True, 1, 1)])
def test_dqn_update_against_autograd_and_adam(pkg, ctx, H, huber, double_dqn, prioritized, n_step, n):
    ns, B, lanes, act = 4, 1024, 32, 0
    tr, ref = _fill(pkg, ctx, ns, lanes, 64, 80, prioritized, B, 5, n)
    if n_step > 1:
        tr.set_nstep(n_step, 0.99)
    p0 = _params(ns, H, n, 2)
    net = pkg.Network(ctx, ns, H, n, p0, act=act, kind=pkg.KIND_DUELING)
    net.set(pkg.learners.NET_TARGET, p0 * np.float32(0.9))
    cfg = pkg.dqn_config(huber=huber, double_dqn=double_dqn, target_update_freq=3, max_grad_norm=10.0, per_beta=0.4)
    learner = pkg.DQNLearner(ctx, net, tr, cfg)
    p, pt = p0.copy(), (p0 * np.float32(0.9)).astype(np.float32)
    m, v, bt = np.zeros_like(p), np.zeros_like(p), np.array([0.9, 0.999], np.float32)
    for it in range(4):
        stats = learner.update(want_stats=True)
        b = tr.batch()
        w = b["weight"] if prioritized else None
        disc = b["discount"] if n_step > 1 else None
        g, loss, td = D.dqn_loss_grad(p, pt, ns, H, n, act, b["state"], b["action"], b["reward"], b["terminal"], b["next_state"], w, 0.99,
                                      huber, double_dqn, disc)
        gc, gn = O.clip_by_global_norm(g.astype(np.float32), 10.0)
        O.adam_step(p, gc, m, v, bt)
        tol = 2e-5 * (1 + it)
        assert stats["loss"] == pytest.approx(loss, rel=10 * tol)
        assert stats["grad_norm"] == pytest.approx(gn, rel=10 * tol)
        dtd = learner.last_td()
        np.testing.assert_allclose(dtd, td, rtol=1e-4, atol=2e-5)
        np.testing.assert_allclose(net.get(pkg.learners.NET_GRAD), gc, rtol=1e-3, atol=1e-6)
        np.testing.assert_allclose(net.get(), p, rtol=0, atol=5e-6)
        if prioritized:                                        # the written-back priorities are (|td| + eps)^alpha of the device's td
            newp = ((np.abs(dtd) + np.float32(1e-6)) ** np.float32(0.6)).astype(np.float32)
            ref.update_priority(b["key"], newp)
            assert tr.total_priority() == pytest.approx(ref.total_priority(), rel=1e-5)
        p = net.get()                                          # teacher forcing: the next step starts from the device's parameters
        m, v, bt = net.get(pkg.learners.NET_M), net.get(pkg.learners.NET_V), net.get(pkg.learners.NET_BETA_T)
        if (it + 1) % 3 == 0:
            pt = p.copy()
            assert np.array_equal(net.get(pkg.learners.NET_TARGET), net.get())
        else:
            pt = net.get(pkg.learners.NET_TARGET)
    net.close(); tr.close()


def _setup(pkg, ctx, seed, env_kind="CartPole", lanes=127, hidden=64, act=0, cap=16, B=256, prioritized=True, explorer="linear",
           ratio=1.0, threshold=3, huber=True, double_dqn=False, target_freq=5):
    kw = dict(params=pkg.pendulum_params(continuous=False, n_actions=3)) if env_kind == "Pendulum" else {}
    env = pkg.B200VecEnv(ctx, env_kind, lanes, O.splitmix_states_fast(lanes, seed), auto_reset=True, **kw)
    ns, na = _NS[env_kind], _NA[env_kind]
    net = pkg.Network(ctx, ns, hidden, na, _params(ns, hidden, na, seed + 1, 0.0), act=act, kind=pkg.KIND_DUELING)
    traj = pkg.Trajectory(ctx, ns, cap, lanes=lanes, batch_size=B, sampler_rng=O.splitmix_states_fast(B, seed + 2), prioritized=prioritized)
    traj.controller = pkg.InsertSampleRatioController(ratio=ratio, threshold=threshold)
    learner = pkg.DQNLearner(ctx, net, traj, pkg.dqn_config(huber=huber, double_dqn=double_dqn, target_update_freq=target_freq))
    ex = pkg.GreedyExplorer() if explorer == "greedy" else pkg.EpsilonGreedyExplorer(0.05, eps_init=1.0, warmup_steps=2 * lanes,
                                                                                    decay_steps=10 * lanes)
    policy = pkg.QBasedPolicy(ctx, learner, ex, O.splitmix_states_fast(lanes, seed + 3), lanes)
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


LOOP_CASES = [
    dict(env_kind="CartPole", hidden=64, act=0),
    dict(env_kind="MountainCar", hidden=64, act=1, explorer="greedy", ratio=0.25, threshold=1),
    dict(env_kind="Pendulum", hidden=64, act=0, ratio=0.25, threshold=2, target_freq=3),
    dict(env_kind="CartPole", hidden=128, act=1, prioritized=False, double_dqn=True, huber=False),
    dict(env_kind="Pendulum", hidden=128, act=0, explorer="greedy", target_freq=2),
    dict(env_kind="MountainCar", hidden=64, act=0, cap=8, threshold=100),              # a window without updates: one fused launch
]


@pytest.mark.parametrize("tc", [True, False])
@pytest.mark.parametrize("case", LOOP_CASES, ids=[f"{c['env_kind']}-H{c['hidden']}-{i}" for i, c in enumerate(LOOP_CASES)])
def test_device_loop_equals_stage_protocol(pkg, ctx, case, tc):
    _tc(ctx, tc)
    try:
        fast, stage = _setup(pkg, ctx, 100, **case), _setup(pkg, ctx, 100, **case)
        stage["agent"].fusable = False
        for n in (19, 6):
            pkg.run(fast["agent"], fast["env"], pkg.StopAfterNSteps(n), pkg.EmptyHook())
            pkg.run(stage["agent"], stage["env"], pkg.StopAfterNSteps(n), pkg.EmptyHook())
        assert fast["agent"]._replay is not None and stage["agent"]._replay is None
        _assert_same(_state(pkg, fast), _state(pkg, stage), pendulum=case["env_kind"] == "Pendulum")
        if case.get("threshold", 3) < 19:
            assert fast["net"].step_count() > 0
    finally:
        _tc(ctx, True)
    _close(fast); _close(stage)


def test_checkpoint_mid_run_restores_and_continues(pkg, ctx):
    ck_mod = pkg.checkpoint
    a = _setup(pkg, ctx, 300, env_kind="MountainCar", ratio=1.0, threshold=2, target_freq=3)
    pkg.run(a["agent"], a["env"], pkg.StopAfterNSteps(9), pkg.EmptyHook())
    ck = ck_mod.checkpoint_replay(a["env"], a["net"], a["agent"])
    assert "net/target" in ck                                  # the dueling net's target network travels with the checkpoint
    ctl = a["traj"].controller
    ctl_state = (ctl.n_inserted, ctl.n_sampled)
    pkg.run(a["agent"], a["env"], pkg.StopAfterNSteps(11), pkg.EmptyHook())
    final_a = _state(pkg, a)
    b = _setup(pkg, ctx, 999, env_kind="MountainCar", ratio=1.0, threshold=2, target_freq=3)     # other seeds
    pkg.run(b["agent"], b["env"], pkg.StopAfterNSteps(4), pkg.EmptyHook())
    ck_mod.restore_replay(ck, b["env"], b["net"], b["agent"])
    assert (b["traj"].controller.n_inserted, b["traj"].controller.n_sampled) == ctl_state
    pkg.run(b["agent"], b["env"], pkg.StopAfterNSteps(11), pkg.EmptyHook())
    _assert_same(final_a, _state(pkg, b))
    _close(a); _close(b)


@pytest.mark.parametrize("env_kind,H,tc", [("CartPole", 64, True), ("Pendulum", 64, True), ("MountainCar", 128, False), ("CartPole", 64, False)])
def test_evaluate_fused_equals_staged_and_stage_protocol(pkg, ctx, env_kind, H, tc):
    ns, na, N = _NS[env_kind], _NA[env_kind], 300
    p = _params(ns, H, na, 21, 0.3)
    kw = dict(params=pkg.pendulum_params(continuous=False, n_actions=3)) if env_kind == "Pendulum" else {}
    out = []
    for mode in ("fused", "staged", "run"):
        env = pkg.B200VecEnv(ctx, env_kind, N, O.splitmix_states_fast(N, 5), auto_reset=True, **kw)
        net = pkg.Network(ctx, ns, H, na, p, act=1, kind=pkg.KIND_DUELING)
        _tc(ctx, tc and mode != "staged")
        try:
            if mode == "run":
                pkg.run(pkg.EvaluationPolicy(net, N), env, pkg.StopAfterNSteps(40), pkg.EmptyHook())
                res = None
            else:
                res = pkg.evaluate(net, env, 40, max_episodes=4)
        finally:
            _tc(ctx, True)
        out.append((res, pkg.checkpoint.checkpoint(env=env)))
        net.close(); env.close()
    (rf, ef), (rs, es), (_, er) = out
    for k in ("returns", "lengths", "counts"):
        assert np.array_equal(np.asarray(rf[k]), np.asarray(rs[k]), equal_nan=True), k     # unreached record slots hold NaN
    _assert_same(ef, es, pendulum=env_kind == "Pendulum")
    _assert_same(ef, er, pendulum=env_kind == "Pendulum")


def test_known_answer_zero_advantage_weights(pkg, ctx):
    """Wa = 0 and equal ba: Q = v for every action, so greedy (findmax, first maximum) picks action 1"""
    ns, H, n, N = 4, 64, 3, 500
    p = _params(ns, H, n, 8, 0.2)
    trunk = H * ns + H + H * H + H
    p[trunk + H + 1:trunk + H + 1 + n * H] = 0.0
    p[trunk + H + 1 + n * H:] = -0.75
    obs = np.random.default_rng(1).standard_normal((ns, N)).astype(np.float32)
    for tc in (True, False):
        _tc(ctx, tc)
        net = pkg.Network(ctx, ns, H, n, p, kind=pkg.KIND_DUELING)
        try:
            q = net.values(obs)
            assert np.all(q == q[:1])
            a = np.empty(N, np.int32)
            assert ctx.lib.b200rl_net_act_greedy(net.h, pkg._lib.ptr(np.asfortranarray(obs)), N, pkg._lib.ptr(a), 0) == 0
            assert np.all(a == 1)
        finally:
            _tc(ctx, True)
            net.close()


def test_refusals_before_any_side_effect(pkg, ctx):
    lib, L = ctx.lib, pkg._lib
    ns, H, n, N = 4, 64, 2, 64
    p = _params(ns, H, n, 4)
    net = pkg.Network(ctx, ns, H, n, p, kind=pkg.KIND_DUELING)
    env = pkg.B200VecEnv(ctx, "CartPole", N, O.splitmix_states_fast(N, 3), auto_reset=True)
    before_env, before_net = pkg.checkpoint.checkpoint(env=env), pkg.checkpoint.checkpoint(net=net)
    obs = np.asfortranarray(np.zeros((ns, N), np.float32))
    rng = O.splitmix_states_fast(N, 2)
    drng = ctx.malloc(rng.nbytes); ctx.h2d(drng, rng)
    outs = np.full(N, 7, np.int32)
    assert lib.b200rl_net_act(net.h, L.ptr(obs), N, C.c_void_p(drng), L.ptr(outs), None, None, None, 0) == L.ERR_INVALID
    cfg = pkg.onpolicy_config(update_freq=4, n_microbatches=1)
    st = np.zeros(6, np.float32)
    assert lib.b200rl_net_ac_step(net.h, C.byref(cfg), L.ptr(obs), L.ptr(np.ones(N, np.int32)), L.ptr(np.zeros(N, np.float32)),
                                  L.ptr(np.zeros(N, np.float32)), L.ptr(np.zeros(N, np.float32)), N, None, N, 0.0, 1.0, 1, L.ptr(st)) == L.ERR_INVALID
    h = C.c_void_p()
    assert lib.b200rl_onpolicy_create(ctx.h, net.h, env.h, C.byref(cfg), L.ptr(rng), C.byref(h)) == L.ERR_INVALID
    ec = L.EvalConfig(1, 5, 2)                                  # mode 1 samples a policy head
    assert lib.b200rl_evaluate(net.h, env.h, C.byref(ec), C.c_void_p(drng), None, None, None, 0) == L.ERR_UNSUPPORTED
    assert np.all(outs == 7) and np.array_equal(ctx.d2h(np.empty_like(rng), drng), rng)
    after_env, after_net = pkg.checkpoint.checkpoint(env=env), pkg.checkpoint.checkpoint(net=net)
    for a, b in ((before_env, after_env), (before_net, after_net)):
        for k in a:
            assert np.array_equal(a[k], b[k]), k
    # n_out = 4 actions: refused at create
    with pytest.raises(L.B200RLError):
        pkg.Network(ctx, ns, H, 4, np.zeros(D.nparams(ns, H, 4), np.float32), kind=pkg.KIND_DUELING)
    ctx.free(drng)
    net.close(); env.close()
