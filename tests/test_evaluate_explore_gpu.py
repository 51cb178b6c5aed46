"""Evaluation of a QBasedPolicy with its explorer (b200rl_evaluate_explore, evaluate(QBasedPolicy, ...)):

1. the fused kernel (H = 64), the staged launches (H = 128, and H = 64 with the tensor cores off) and the stage protocol
   env.reset_(True), n x {QBasedPolicy.plan_device, env.act_} give the same records, env fields, explorer streams and explorer
   step, bit for bit, for every device explorer and GreedyExplorer;
2. a fused call is the reset plus one launch;
3. ϵ = 0 plans like GreedyExplorer and draws exactly once per column per step;
4. evaluating with a second QBasedPolicy between two training windows leaves the training run untouched;
5. refusals leave env, streams, explorer step and network untouched."""
import ctypes as C
import types

import numpy as np
import pytest

import explorers_ref as X
import oracle_lib as O
from test_evaluate_gpu import RecordHook, _compare, _snapshot, same
from test_explorers_gpu import _close, _setup, _state, _assert_same

pytestmark = pytest.mark.gpu

_NA = {"CartPole": 2, "MountainCar": 3, "Pendulum": 3}
_NS = {"CartPole": 4, "MountainCar": 2, "Pendulum": 3}


def _env(pkg, ctx, kind, n, seed, max_timeout=0):
    kw = dict(params=pkg.pendulum_params(continuous=False, n_actions=3)) if kind == "Pendulum" else {}
    env = pkg.B200VecEnv(ctx, kind, n, O.splitmix_states_fast(n, seed), auto_reset=True, **kw)
    if max_timeout:
        env.set_max_timeout(max_timeout)
    return env


def _qnet(pkg, ctx, kind, hidden, act, dueling, seed=21):
    ns, na = _NS[kind], _NA[kind]
    if dueling:
        import dueling_ref as D
        p = D.glorot_params(ns, hidden, na, seed)
        return pkg.Network(ctx, ns, hidden, na, p * np.float32(2.0), act=act, kind=pkg.KIND_DUELING)
    p = O.glorot_params(O.ac_desc(ns, hidden, na, act), seed, q_net=True) * np.float32(2.0)
    return pkg.Network(ctx, ns, hidden, na, p, act=act, kind=pkg.KIND_Q)


def _explorer(pkg, name, total):
    """`total` = N n_steps columns: the ϵ-greedy schedules cross their warm-up and decay inside the window"""
    return {
        "linear": lambda: pkg.EpsilonGreedyExplorer(0.05, kind="linear", eps_init=0.9, warmup_steps=total // 4, decay_steps=total // 3),
        "exp": lambda: pkg.EpsilonGreedyExplorer(0.1, kind="exp", eps_init=1.0, warmup_steps=total // 5, decay_steps=max(1, total // 6), step=3),
        "tie": lambda: pkg.EpsilonGreedyExplorer(0.3, is_break_tie=True, warmup_steps=total // 4, decay_steps=total // 2),
        "speedy": lambda: pkg.EpsilonSpeedyExplorer(4.0 / total, step=2),
        "weighted": pkg.WeightedSoftmaxExplorer,
        "gumbel": pkg.GumbelSoftmaxExplorer,
        "greedy": pkg.GreedyExplorer,
    }[name]()


def _policy(pkg, ctx, net, ex, n, seed=808):
    return pkg.QBasedPolicy(ctx, types.SimpleNamespace(net=net), ex, O.splitmix_states_fast(n, seed), n)


def _run(pkg, ctx, path, kind, n, hidden, act, dueling, ex_name, n_steps, K, max_timeout):
    """one evaluation window on fresh objects with fixed seeds; path "api" = evaluate(QBasedPolicy, ...), "stage" = the stage
    protocol"""
    env = _env(pkg, ctx, kind, n, 9, max_timeout)
    net = _qnet(pkg, ctx, kind, hidden, act, dueling)
    ex = _explorer(pkg, ex_name, n * n_steps)
    policy = _policy(pkg, ctx, net, ex, n)
    l0 = ctx.launch_count()
    if path == "api":
        r = pkg.evaluate(policy, env, n_steps, max_episodes=K)
    else:
        env.reset_(True)
        hook = RecordHook(n, K)
        hook.push("PreExperimentStage", policy, env)
        for _ in range(n_steps):
            env.act_(int(policy.plan_device(env)))
            hook.push("PostActStage", policy, env)
        r = dict(returns=hook.returns, lengths=hook.lengths, counts=hook.counts)
    launches = ctx.launch_count() - l0
    out = dict(r=r, env=_snapshot(env), xrng=policy.explorer_rng(), step=getattr(ex, "step", None), launches=launches,
               params=net.get(), target=net.get(pkg.learners.NET_TARGET), nstep=net.step_count())
    policy.close(); net.close(); env.close()
    return out


def _assert_equal_runs(a, b):
    for k in ("returns", "lengths", "counts"):
        assert same(a["r"][k], b["r"][k]), k
    _compare(a["env"], b["env"])
    assert same(a["xrng"], b["xrng"]), "explorer streams"
    assert a["step"] == b["step"]
    assert same(a["params"], b["params"]) and same(a["target"], b["target"]) and a["nstep"] == b["nstep"]


# (env, act, dueling, N, explorer, n_steps, K, MaxTimeoutEnv)
CASES = [
    ("CartPole", 0, False, 1000, "linear", 120, 3, 23),
    ("CartPole", 1, False, 127, "exp", 150, 1, 0),
    ("MountainCar", 0, True, 127, "tie", 150, 3, 40),
    ("Pendulum", 1, True, 1000, "speedy", 120, 1, 50),
    ("CartPole", 0, True, 1, "weighted", 200, 3, 0),
    ("MountainCar", 1, False, 1000, "gumbel", 120, 0, 30),
    ("Pendulum", 0, False, 127, "greedy", 150, 3, 40),
    ("CartPole", 1, True, 127, "greedy", 150, 1, 17),
    ("CartPole", 0, False, 65537, "gumbel", 40, 1, 0),
    ("MountainCar", 0, True, 65537, "linear", 40, 3, 15),
    ("Pendulum", 1, False, 1, "speedy", 200, 1, 0),
    ("CartPole", 0, False, 127, "weighted", 150, 0, 0),
]


@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}-{'relu' if c[1] == 0 else 'tanh'}-{'duel' if c[2] else 'q'}-N{c[3]}-{c[4]}-K{c[6]}"
                                             for c in CASES])
def test_fused_staged_and_stage_protocol_are_bit_identical(pkg, ctx, case):
    kind, act, dueling, n, ex_name, n_steps, K, mt = case
    args = (kind, n, 64, act, dueling, ex_name, n_steps, K, mt)
    stage = _run(pkg, ctx, "stage", *args)
    fused = _run(pkg, ctx, "api", *args)
    assert fused["launches"] == 2, fused["launches"]              # reset + one evaluation launch
    _assert_equal_runs(fused, stage)
    try:
        pkg._lib.check(ctx.lib.b200rl_set_tensor_cores(0))
        staged = _run(pkg, ctx, "api", *args)
    finally:
        pkg._lib.check(ctx.lib.b200rl_set_tensor_cores(1))
    assert staged["launches"] > n_steps
    _assert_equal_runs(staged, stage)
    assert fused["env"]["ep"]["env_steps"] == n * n_steps
    if ex_name != "greedy":
        assert not np.array_equal(fused["xrng"], O.splitmix_states_fast(n, 808))
        if ex_name in ("linear", "exp", "tie", "speedy"):
            start = {"exp": 3, "speedy": 2}.get(ex_name, 1)
            assert fused["step"] == start + n * n_steps
    else:
        assert np.array_equal(fused["xrng"], O.splitmix_states_fast(n, 808))   # GreedyExplorer draws nothing
    if K and n >= 127:
        assert (fused["r"]["counts"] > 0).any()


@pytest.mark.parametrize("case", [CASES[0], CASES[3], CASES[6], CASES[8]], ids=["linear", "speedy", "greedy", "gumbel-65537"])
def test_staged_h128_is_bit_identical_to_the_stage_protocol(pkg, ctx, case):
    kind, act, dueling, n, ex_name, n_steps, K, mt = case
    args = (kind, n, 128, act, dueling, ex_name, min(n_steps, 60), K, mt)
    stage, staged = _run(pkg, ctx, "stage", *args), _run(pkg, ctx, "api", *args)
    assert staged["launches"] > args[6]
    _assert_equal_runs(staged, stage)


def _xo_advance(states, k):
    out = states.copy()
    for row in out:
        s = [int(w) for w in row]
        for _ in range(k):
            X.xo_next(s)
        row[:] = np.array(s, np.uint64)
    return out


def test_epsilon_zero_plans_like_greedy_with_one_draw_per_column(pkg, ctx):
    n, n_steps = 300, 90
    outs = {}
    for name in ("eps0", "greedy"):
        env = _env(pkg, ctx, "MountainCar", n, 4)
        net = _qnet(pkg, ctx, "MountainCar", 64, 1, False)
        ex = pkg.EpsilonGreedyExplorer(0.0, eps_init=0.0) if name == "eps0" else pkg.GreedyExplorer()
        policy = _policy(pkg, ctx, net, ex, n)
        r = pkg.evaluate(policy, env, n_steps, max_episodes=2)
        outs[name] = dict(r=r, env=_snapshot(env), xrng=policy.explorer_rng())
        policy.close(); net.close(); env.close()
    a, b = outs["eps0"], outs["greedy"]
    for k in ("returns", "lengths", "counts"):
        assert same(a["r"][k], b["r"][k]), k
    _compare(a["env"], b["env"])
    seeds = O.splitmix_states_fast(n, 808)
    assert np.array_equal(b["xrng"], seeds)
    assert np.array_equal(a["xrng"], _xo_advance(seeds, n_steps))


def test_evaluation_between_training_windows_leaves_training_untouched(pkg, ctx):
    outs = []
    for with_eval in (True, False):
        s = _setup(pkg, ctx, 71, lanes=127, explorer="speedy", threshold=3)
        pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(30), pkg.EmptyHook())
        if with_eval:
            ev_env = _env(pkg, ctx, "CartPole", 2000, 72)
            ev = pkg.QBasedPolicy(ctx, s["learner"], pkg.EpsilonGreedyExplorer(0.05), O.splitmix_states_fast(2000, 73), 2000)
            r = pkg.evaluate(ev, ev_env, 150, max_episodes=1)
            assert (r["counts"] > 0).any() and ev.explorer.step == 1 + 2000 * 150
            ev.close(); ev_env.close()
        pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(20), pkg.EmptyHook())
        assert s["agent"]._replay is not None
        outs.append((_state(pkg, s), s["policy"].explorer.step, s["traj"].controller.n_sampled))
        _close(s)
    (a, sa, na), (b, sb, nb) = outs
    _assert_same(a, b)
    assert sa == sb and na == nb and na > 0


def test_refusals_leave_everything_untouched(pkg, ctx):
    L, lib = pkg._lib, ctx.lib
    n = 64
    cp = _env(pkg, ctx, "CartPole", n, 1)
    mc = _env(pkg, ctx, "MountainCar", n, 1)
    f64 = pkg.B200VecEnv(ctx, "CartPole", n, O.splitmix_states_fast(n, 1), T=np.float64, auto_reset=True)
    acro = pkg.B200VecEnv(ctx, "Acrobot", n, O.splitmix_states_fast(n, 1), T=np.float64, auto_reset=True)
    ccp = pkg.B200VecEnv(ctx, "ContinuousCartPole", n, O.splitmix_states_fast(n, 1), auto_reset=True)
    qnet = _qnet(pkg, ctx, "CartPole", 64, 0, False)
    q3 = pkg.Network(ctx, 4, 64, 3, O.glorot_params(O.ac_desc(4, 64, 3, 0), 2, q_net=True), kind=pkg.KIND_Q)
    acnet = pkg.Network(ctx, 4, 64, 2, O.glorot_params(O.ac_desc(4, 64, 2, 0), 3), kind=pkg.KIND_CATEGORICAL)
    policy = _policy(pkg, ctx, qnet, pkg.EpsilonSpeedyExplorer(0.01, step=7), n)
    rng = C.c_void_p(policy._d_rng)

    def snap(env):
        return (pkg.checkpoint.checkpoint(env=env), policy.explorer_rng(), qnet.get(), qnet.get(pkg.learners.NET_TARGET),
                qnet.step_count())

    def call(net, env, ex, rng=rng, n_steps=10, K=1):
        ret = np.zeros((max(K, 1), env.n), np.float32, order="F"); cnt = np.zeros(env.n, np.int32)
        step0 = None if ex is None else ex.step
        before = snap(env)
        st = lib.b200rl_evaluate_explore(net.h, env.h, n_steps, K, None if ex is None else C.byref(ex), rng, L.ptr(ret), None,
                                         L.ptr(cnt), 0)
        if st != L.OK:
            after = snap(env)
            for k in before[0]:
                assert same(before[0][k], after[0][k]), k
            for x, y in zip(before[1:4], after[1:4]):
                assert same(x, y)
            assert before[4] == after[4] and not cnt.any() and not ret.any()
            assert ex is None or ex.step == step0
        return st

    good = policy.explorer.as_struct
    assert call(qnet, f64, good()) == L.ERR_UNSUPPORTED
    assert call(qnet, acro, good()) == L.ERR_UNSUPPORTED
    assert call(qnet, ccp, good()) == L.ERR_UNSUPPORTED
    assert call(acnet, cp, good()) == L.ERR_INVALID                 # not a Q-network
    assert call(qnet, mc, good()) == L.ERR_INVALID                  # 4 inputs, 2 observations
    assert call(q3, cp, good()) == L.ERR_INVALID                    # 3 Q-values, 2 actions
    assert call(qnet, cp, good(), n_steps=0) == L.ERR_INVALID
    assert call(qnet, cp, good(), K=-1) == L.ERR_INVALID
    for ex in (pkg.EpsilonSpeedyExplorer(0.1), pkg.WeightedSoftmaxExplorer(), pkg.GumbelSoftmaxExplorer(), pkg.EpsilonGreedyExplorer(0.1)):
        assert call(qnet, cp, ex.as_struct(), rng=None) == L.ERR_INVALID        # no explorer streams
    bads = []
    for kind, beta in ((5, 0.0), (-1, 0.0), (2, float("nan")), (2, float("inf")), (2, float("-inf")), (3, 0.5), (4, 1.0)):
        e = good()
        e.kind, e.beta = kind, beta
        bads.append(e)
    for field, v in (("eps_stable", 0.1), ("eps_init", 1.0), ("warmup_steps", 3), ("decay_steps", 5), ("is_break_tie", 1)):
        for kind in (2, 3, 4):                                       # an ϵ-greedy field on a kind that does not read it
            e = good()
            e.kind = kind
            if kind != 2:
                e.beta = 0.0
            setattr(e, field, v)
            bads.append(e)
    for kw in (dict(eps_stable=1.5), dict(eps_init=-0.1), dict(warmup_steps=-1), dict(decay_steps=-2)):   # a bad ϵ-greedy schedule
        e = pkg.EpsilonGreedyExplorer(0.1).as_struct()
        for f, v in kw.items():
            setattr(e, f, v)
        bads.append(e)
    for e in bads:
        assert call(qnet, cp, e) == L.ERR_INVALID
    assert call(qnet, cp, None, rng=None, n_steps=5, K=0) == L.OK     # GreedyExplorer needs no streams; K = 0: counts only
    assert call(qnet, cp, good(), n_steps=5) == L.OK
    with pytest.raises(TypeError):
        pkg.evaluate(_policy(pkg, ctx, qnet, object(), n), cp, 5)
    policy.close()
    for h in (cp, mc, f64, acro, ccp, qnet, q3, acnet):
        h.close()
