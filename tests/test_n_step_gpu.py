"""GPU tests of the n-step sampler (NStepBatchSampler(n, γ); DESIGN.md §3): the draw is the 1-step sampler's, the window fields
equal the NumPy restatement over the exported ring bit for bit, the DQN update with per-sample discounts matches the oracle, the
device agent loop still equals the stage protocol, n = 1 is the BatchSampler bit for bit, and refusals touch nothing."""
import ctypes as C

import numpy as np
import pytest

import nstep_ref as N
import oracle_lib as O
import q_ref as Q

pytestmark = pytest.mark.gpu

_NA = {"CartPole": 2, "MountainCar": 3, "Pendulum": 3}
_NS = {"CartPole": 4, "MountainCar": 2, "Pendulum": 3}
DRAW_FIELDS = ("state", "action", "key", "priority", "weight")
WINDOW_FIELDS = ("reward", "terminal", "next_state", "discount", "horizon")


def _env(pkg, ctx, kind, lanes, seed, auto_reset=True, max_timeout=0):
    kw = dict(params=pkg.pendulum_params(continuous=False, n_actions=3)) if kind == "Pendulum" else {}
    env = pkg.B200VecEnv(ctx, kind, lanes, O.splitmix_states_fast(lanes, seed), auto_reset=auto_reset, **kw)
    if max_timeout:
        env.set_max_timeout(max_timeout)
    return env


def _drive(env, trajs, ref, steps, forced_reset_at=()):
    """random-policy steps, pushed the way learners.Agent pushes them (forced resets with an episode-start frame for every lane,
    soft resets with one for the lanes that ended); the oracle ring (may be None) gets the same pushes"""
    env.reset_(is_force=True)
    for t in trajs:
        t.push_env(env, first_state_only=True)
    if ref is not None:
        ref.push_state(env.state())
    for k in range(steps):
        if k in forced_reset_at:
            env.reset_(is_force=True)
            for t in trajs:
                t.push_env(env, first_state_only=True)
            if ref is not None:
                ref.push_state(env.state())
        if not env.auto_reset:
            env.reset_(is_force=False)
            for t in trajs:
                t.push_env(env, first_state_only=2)
            if ref is not None:
                ref.push_episode_start(env.state(), pending_only=True)
        env.act_random_()
        for t in trajs:
            t.push_env(env)
        if ref is not None:
            ref.push(env.last_action(), env.reward(), env.flags(), env.state())


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _check_against_restatement(tr, b, n, gamma):
    rb = N.nstep_batch(tr.export_state(), tr.ns, tr.lanes, tr.capacity, b["key"], n, gamma)
    for f in WINDOW_FIELDS:
        assert np.array_equal(_bits(b[f]), _bits(rb[f])), f
    return rb


DRAW_CASES = [
    dict(kind="CartPole", lanes=1, cap=64, steps=150),                                    # one lane, wrapped
    dict(kind="CartPole", lanes=127, cap=24, steps=60, forced_reset_at=(33,)),            # wrapped, a forced reset inside the ring
    dict(kind="MountainCar", lanes=127, cap=40, steps=30, max_timeout=9),                 # MaxTimeoutEnv ends episodes
    dict(kind="Pendulum", lanes=127, cap=16, steps=40, max_timeout=11),                   # non-integer rewards, wrapped
    dict(kind="CartPole", lanes=127, cap=32, steps=45, auto_reset=False),                 # soft resets
    dict(kind="Pendulum", lanes=4096, cap=12, steps=20, forced_reset_at=(7,), auto_reset=False),
    dict(kind="CartPole", lanes=4096, cap=8, steps=19),
]


@pytest.mark.parametrize("prioritized", [False, True])
@pytest.mark.parametrize("n", [2, 3, 5])
@pytest.mark.parametrize("case", DRAW_CASES, ids=[f"{c['kind']}-{c['lanes']}-{i}" for i, c in enumerate(DRAW_CASES)])
def test_same_draws_and_windows(pkg, ctx, case, n, prioritized):
    B, gamma = 1024, 0.97
    kind, lanes, cap = case["kind"], case["lanes"], case["cap"]
    env = _env(pkg, ctx, kind, lanes, 40 + n, case.get("auto_reset", True), case.get("max_timeout", 0))
    slots = O.splitmix_states_fast(B, 7 + n)
    one = pkg.Trajectory(ctx, _NS[kind], cap, lanes=lanes, batch_size=B, sampler_rng=slots, prioritized=prioritized)
    nst = pkg.Trajectory(ctx, _NS[kind], cap, lanes=lanes, batch_size=B, sampler_rng=slots, prioritized=prioritized, n_step=n, gamma=gamma)
    ref = O.OracleTraj(_NS[kind], lanes, cap, prioritized) if lanes < 4096 else None
    _drive(env, [one, nst], ref, case["steps"], case.get("forced_reset_at", ()))
    s = slots.copy()
    horizons = []
    for _ in range(2):
        b1, bn = one.sample(beta=0.5), nst.sample(beta=0.5)
        for f in DRAW_FIELDS:
            assert np.array_equal(b1[f], bn[f]), f
        assert np.array_equal(one.sampler_rng(), nst.sampler_rng())
        if ref is not None:                                    # the 1-step batch is the oracle's
            rb = ref.sample(s, B, prioritized=prioritized, beta=0.5)
            for f in ("state", "action", "reward", "terminal", "next_state", "key"):
                assert np.array_equal(b1[f], rb[f]), f
        _check_against_restatement(nst, bn, n, gamma)
        assert np.all((bn["horizon"] >= 1) & (bn["horizon"] <= n))
        horizons.append(bn["horizon"])
    h = np.concatenate(horizons)
    assert h.max() == n and (h < n).any()                      # full windows and cut ones both occur
    one.close(); nst.close(); env.close()


def test_soft_reset_env_through_the_stage_loop(pkg, ctx):
    """run(Agent(...)) on a soft-reset env (the stage loop: soft resets, episode-start pushes, updates): n-step batches of the ring
    it leaves equal the restatement"""
    lanes, B, n = 96, 512, 4
    env = _env(pkg, ctx, "CartPole", lanes, 5, auto_reset=False)
    net = pkg.Network(ctx, 4, 64, 2, O.glorot_params(O.ac_desc(4, 64, 2), 6, q_net=True), kind=pkg.KIND_Q)
    traj = pkg.Trajectory(ctx, 4, 48, lanes=lanes, batch_size=B, sampler_rng=O.splitmix_states_fast(B, 7), prioritized=True,
                          n_step=n, gamma=0.99)
    traj.controller = pkg.InsertSampleRatioController(ratio=0.25, threshold=4)
    learner = pkg.DQNLearner(ctx, net, traj, pkg.dqn_config(target_update_freq=3))
    policy = pkg.QBasedPolicy(ctx, learner, pkg.EpsilonGreedyExplorer(0.3), O.splitmix_states_fast(lanes, 8), lanes)
    agent = pkg.Agent(policy, traj)
    assert not agent.replay_supported(env)                      # soft resets keep the stage loop
    pkg.run(agent, env, pkg.StopAfterNSteps(40), pkg.EmptyHook())
    assert net.step_count() > 0
    b = traj.sample()
    _check_against_restatement(traj, b, n, 0.99)
    assert (b["horizon"] < n).any() and b["terminal"].any()
    agent.close(); policy.close(); traj.close(); net.close(); env.close()


def test_known_answer_cartpole_gamma_one(pkg, ctx):
    lanes, B, n, cap = 256, 4096, 6, 30
    env = _env(pkg, ctx, "CartPole", lanes, 3)
    tr = pkg.Trajectory(ctx, 4, cap, lanes=lanes, batch_size=B, sampler_rng=O.splitmix_states_fast(B, 4), n_step=n, gamma=1.0)
    _drive(env, [tr], None, 50)
    b = tr.sample()
    # every CartPole step pays 1 except the one that ends the episode (CartPoleEnv: reward = done ? 0 : 1)
    assert np.array_equal(b["reward"], (b["horizon"] - b["terminal"]).astype(np.float32)) and np.all(b["discount"] == 1.0)
    st = tr.export_state()
    F = cap + 1
    slot, lane = b["key"] // lanes, b["key"] % lanes
    newest = (st["head"][lane].astype(np.int64) - 1) % F            # the lane's newest state frame
    reached_head = (slot + b["horizon"]) % F == newest
    short = b["horizon"] < n
    assert np.all(~short | (b["terminal"] == 1) | reached_head)
    assert short.any() and (b["terminal"] == 1).any() and reached_head.any()
    tr.close(); env.close()


def _fill_both(pkg, ctx, ns, lanes, cap, frames, prioritized, B, seed, n=1, gamma=0.99):
    slots = O.splitmix_states_fast(B, 900 + seed)
    tr = pkg.Trajectory(ctx, ns, cap, lanes=lanes, batch_size=B, sampler_rng=slots, prioritized=prioritized, n_step=n, gamma=gamma)
    ref = O.OracleTraj(ns, lanes, cap, prioritized)
    rng = np.random.default_rng(seed)
    obs = rng.standard_normal((ns, lanes)).astype(np.float32)
    tr.push_state(obs); ref.push_state(obs)
    for _ in range(frames):
        a = rng.integers(1, 3, lanes).astype(np.int32); r = rng.standard_normal(lanes).astype(np.float32)
        t = (rng.random(lanes) < 0.1).astype(np.uint8); obs = rng.standard_normal((ns, lanes)).astype(np.float32)
        tr.push(a, r, t, obs); ref.push(a, r, t, obs)
        if t.any():
            s0 = rng.standard_normal((ns, lanes)).astype(np.float32)
            tr.push_episode_start(s0, pending_only=True); ref.push_episode_start(s0, pending_only=True)
    return tr, ref, slots


UPDATE_CASES = [(128, True, False, True), (64, False, False, False), (128, True, True, True), (64, True, True, True), (128, False, False, False)]


@pytest.mark.parametrize("hidden,huber,double_dqn,prioritized", UPDATE_CASES)
def test_dqn_update_parity_n3(pkg, ctx, hidden, huber, double_dqn, prioritized):
    """test_dqn_update_parity's pattern with n = 3: sample + TD update with per-sample discounts + priority write-back"""
    ns, na, B, lanes, n, gamma = 4, 2, 1024, 32, 3, 0.99
    tr, ref, slots = _fill_both(pkg, ctx, ns, lanes, 64, 80, prioritized, B, 5, n=n, gamma=gamma)
    desc = O.ac_desc(ns, hidden, na)
    p0 = O.glorot_params(desc, 2, q_net=True) + 0.05 * np.random.default_rng(1).standard_normal(O.q_nparams(desc)).astype(np.float32)
    net = pkg.Network(ctx, ns, hidden, na, p0, kind=pkg.KIND_Q)
    net.set(pkg.learners.NET_TARGET, p0 * np.float32(0.9))
    cfg = pkg.dqn_config(gamma=gamma, huber=huber, double_dqn=double_dqn, target_update_freq=3, max_grad_norm=10.0, per_beta=0.4)
    learner = pkg.DQNLearner(ctx, net, tr, cfg)
    p = p0.copy(); pt = p0 * np.float32(0.9)
    m = np.zeros_like(p); v = np.zeros_like(p); bt = np.array([0.9, 0.999], np.float32)
    s = slots.copy()
    for it in range(4):
        stats = learner.update(want_stats=True)
        b = tr.batch()
        rb = ref.sample(s, B, prioritized=prioritized, beta=0.4)   # same draw as the oracle's 1-step sampler
        assert np.array_equal(b["key"], rb["key"]) and np.array_equal(b["state"], rb["state"])
        _check_against_restatement(tr, b, n, gamma)
        assert (b["horizon"] < n).any() and (b["horizon"] == n).any()
        w = b["weight"] if prioritized else None
        g, loss, td = Q.oracle_dqn_loss_grad(desc, p, pt, b, w, huber, double_dqn)
        gc, gn = O.clip_by_global_norm(g.astype(np.float32), 10.0)
        O.adam_step(p, gc, m, v, bt)
        tol = 2e-5 * (1 + it)
        assert stats["loss"] == pytest.approx(loss, rel=tol)
        assert stats["grad_norm"] == pytest.approx(gn, rel=10 * tol)
        np.testing.assert_allclose(learner.last_td(), td, rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(net.get(), p, rtol=0, atol=5e-6)
        if prioritized:
            newp = (np.abs(td) + np.float32(1e-6)) ** np.float32(0.6)
            ref.update_priority(b["key"], newp.astype(np.float32))
            assert tr.total_priority() == pytest.approx(ref.total_priority(), rel=1e-5)
            # the device tree holds its own priorities (from its TD errors): keep the oracle's sampler on the device's tree
            ref.update_priority(b["key"], _device_priorities(tr, b["key"]))
        if (it + 1) % 3 == 0:
            pt = p.copy()
            np.testing.assert_allclose(net.get(pkg.learners.NET_TARGET), net.get(), rtol=0, atol=0)
    tr.close(); net.close()


def _device_priorities(tr, keys):
    tree = tr.export_state()["tree"]
    return tree[tree.size // 2 + keys].astype(np.float32)


def test_n1_is_the_batch_sampler_bit_for_bit(pkg, ctx):
    ns, na, B, lanes = 4, 2, 1024, 32
    runs = []
    for setting in (None, (1, 0.9)):
        tr, _, _ = _fill_both(pkg, ctx, ns, lanes, 64, 80, True, B, 11)
        if setting:
            tr.set_nstep(*setting)
        desc = O.ac_desc(ns, 64, na)
        net = pkg.Network(ctx, ns, 64, na, O.glorot_params(desc, 2, q_net=True), kind=pkg.KIND_Q)
        learner = pkg.DQNLearner(ctx, net, tr, pkg.dqn_config(double_dqn=True, target_update_freq=2))
        out = []
        for _ in range(3):
            learner.update()
            out.append((tr.batch(), learner.last_td(), net.get(), net.get(pkg.learners.NET_TARGET), tr.export_state()["tree"]))
        runs.append(out)
        tr.close(); net.close()
    for (ba, tda, pa, ta, tra), (bb, tdb, pb, tb, trb) in zip(*runs):
        for f in DRAW_FIELDS + ("reward", "terminal", "next_state"):
            assert np.array_equal(ba[f], bb[f]), f
        assert np.all(ba["discount"] == np.float32(0.99)) and np.all(bb["discount"] == np.float32(0.9))
        assert np.all(ba["horizon"] == 1) and np.all(bb["horizon"] == 1)
        for x, y in ((tda, tdb), (pa, pb), (ta, tb), (tra, trb)):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


# ---- the device agent loop ------------------------------------------------------------------------------------------------------
def _setup(pkg, ctx, seed, n, lanes=127, hidden=64, cap=24, B=256, prioritized=True, ratio=1.0, threshold=3, target_freq=4,
           double_dqn=False):
    env = _env(pkg, ctx, "CartPole", lanes, seed)
    net = pkg.Network(ctx, 4, hidden, 2, O.glorot_params(O.ac_desc(4, hidden, 2), seed + 1, q_net=True), kind=pkg.KIND_Q)
    traj = pkg.Trajectory(ctx, 4, cap, lanes=lanes, batch_size=B, sampler_rng=O.splitmix_states_fast(B, seed + 2), prioritized=prioritized,
                          n_step=n, gamma=0.99)
    traj.controller = pkg.InsertSampleRatioController(ratio=ratio, threshold=threshold)
    learner = pkg.DQNLearner(ctx, net, traj, pkg.dqn_config(gamma=0.99, double_dqn=double_dqn, target_update_freq=target_freq))
    ex = pkg.EpsilonGreedyExplorer(0.05, eps_init=1.0, warmup_steps=2 * lanes, decay_steps=10 * lanes)
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


def _assert_same(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


@pytest.mark.parametrize("ratio,hidden,prioritized", [(1.0, 64, True), (0.25, 64, True), (1.0, 128, False), (0.25, 128, True)])
def test_device_loop_equals_stage_protocol_n3(pkg, ctx, ratio, hidden, prioritized):
    fast, stage = _setup(pkg, ctx, 70, 3, hidden=hidden, ratio=ratio, prioritized=prioritized), \
        _setup(pkg, ctx, 70, 3, hidden=hidden, ratio=ratio, prioritized=prioritized)
    stage["agent"].fusable = False
    for steps in (21, 9):                                     # target syncs (every 4 updates) fall inside both windows
        for s in (fast, stage):
            pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(steps), pkg.EmptyHook())
        assert fast["agent"]._replay is not None and stage["agent"]._replay is None
        _assert_same(_state(pkg, fast), _state(pkg, stage))
    assert fast["net"].step_count() >= 6
    if ratio >= 1.0:
        assert fast["agent"].graph_active()
        assert np.array_equal(fast["learner"].last_td(), stage["learner"].last_td())
    # a new n between runs: the captured units are re-captured, and the two paths still agree
    for s in (fast, stage):
        s["traj"].set_nstep(5, 0.99)
        pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(13), pkg.EmptyHook())
    _assert_same(_state(pkg, fast), _state(pkg, stage))
    if ratio >= 1.0:
        assert fast["agent"].graph_active()
        assert np.array_equal(fast["learner"].last_td(), stage["learner"].last_td())
    _close(fast); _close(stage)


# ---- refusals ----------------------------------------------------------------------------------------------------------------
def _everything(pkg, s):
    st = _state(pkg, s)
    st["batch"] = s["traj"].batch()
    return st


def _assert_untouched(a, b):
    for k in a:
        if k == "batch":
            for f in a[k]:
                assert np.array_equal(a[k][f], b[k][f]), f
        else:
            assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


def test_refusals_leave_everything_untouched(pkg, ctx):
    lib = ctx.lib
    s = _setup(pkg, ctx, 11, 3, lanes=64, cap=16)
    pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(6), pkg.EmptyHook())
    traj, net, env = s["traj"], s["net"], s["env"]
    before = _everything(pkg, s)
    for n, g in ((0, 0.9), (-1, 0.9), (33, 0.9), (17, 0.9), (3, float("nan")), (3, float("inf")), (3, -0.01), (3, 1.01)):
        assert lib.b200rl_traj_set_nstep(traj.h, n, C.c_float(g)) == pkg._lib.ERR_INVALID, (n, g)
    _assert_untouched(before, _everything(pkg, s))
    # the setting itself is unchanged: the next sample is an n = 3 window batch
    b = traj.sample()
    _check_against_restatement(traj, b, 3, 0.99)
    assert b["horizon"].max() == 3
    before = _everything(pkg, s)
    # a learner whose gamma is not the sampler's
    bad = pkg.dqn_config(gamma=0.9)
    assert lib.b200rl_dqn_update(net.h, traj.h, C.byref(bad), None) == pkg._lib.ERR_INVALID
    h = C.c_void_p()
    assert lib.b200rl_replay_create(ctx.h, net.h, env.h, traj.h, C.byref(bad), C.byref(h)) == pkg._lib.ERR_INVALID
    _assert_untouched(before, _everything(pkg, s))
    # run refuses too once the trajectory's gamma moves under a live handle
    r = s["agent"]._replay
    assert r is not None
    traj.set_nstep(3, 0.95)
    ex = s["policy"].explorer.as_struct()
    ctl = pkg._lib.InsertSampleRatio(1.0, 1, 5, 3)
    assert lib.b200rl_replay_run(r, C.c_void_p(s["policy"]._d_rng), C.byref(ex), C.byref(ctl), 4, None) == pkg._lib.ERR_INVALID
    assert (ctl.n_inserted, ctl.n_sampled) == (5, 3)
    _assert_untouched(before, _everything(pkg, s))
    with pytest.raises(Exception):
        pkg.Trajectory(ctx, 4, 8, lanes=4, batch_size=16, sampler_rng=O.splitmix_states_fast(16, 1), n_step=9)
    _close(s)
