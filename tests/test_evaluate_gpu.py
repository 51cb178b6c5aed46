"""Evaluation of a trained policy (b200rl_net_act_greedy, b200rl_evaluate, EvaluationPolicy, evaluate):

1. the greedy plan against the oracle's head outputs and arg-max;
2. the fused evaluation kernel against the stage protocol run(EvaluationPolicy, env, StopAfterNSteps(n), hook), bit for bit;
3. the staged path inside b200rl_evaluate (H = 128, tensor cores off) against the same protocol;
4. evaluating between training iterations leaves the training run untouched;
5. a known answer: a linear CartPole controller written as a relu network balances the pole when planned greedily;
6. refusals leave the env untouched."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from test_rollout_gpu import CASES

pytestmark = pytest.mark.gpu

REL = 1e-5
N_IN = {"CartPole": 4, "ContinuousCartPole": 4, "Pendulum": 3, "MountainCar": 2, "ContinuousMountainCar": 2}


def rel_err(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)


def same(x, y):   # bitwise, whatever the memory order
    x, y = np.asarray(x), np.asarray(y)
    return x.shape == y.shape and x.dtype == y.dtype and x.tobytes(order="A") == y.tobytes(order="A")


def _env(pkg, ctx, kind, n, seed, **envkw):
    return pkg.B200VecEnv(ctx, kind, n, O.splitmix_states_fast(n, seed), auto_reset=True, **envkw)


def _net(pkg, ctx, env, kind, act, hidden=64, q=False, seed=77):
    n_in = N_IN[kind]
    if q:
        n_out, net_kind = len(env.action_space()), pkg.KIND_Q
    elif env.continuous:
        n_out, net_kind = 1, pkg.KIND_GAUSSIAN
    else:
        n_out, net_kind = len(env.action_space()), pkg.KIND_CATEGORICAL
    desc = O.ac_desc(n_in, hidden, n_out, act, net_kind == pkg.KIND_GAUSSIAN)
    params = O.glorot_params(desc, seed, q_net=q)
    params = params + 0.05 * np.random.default_rng(3).standard_normal(params.size).astype(np.float32)
    return pkg.Network(ctx, n_in, hidden, n_out, params, act=act, kind=net_kind)


class RecordHook:
    """Stage-protocol restatement of the evaluation records: per-env Float32 return / length accumulators, the first K
    episodes of each env, and how many ended."""
    per_step = True

    def __init__(self, n, K):
        self.n, self.K = n, K

    def push(self, stage, policy, env):
        if stage == "PreExperimentStage":
            self.acc = np.zeros(self.n, np.float32)
            self.len = np.zeros(self.n, np.int32)
            self.counts = np.zeros(self.n, np.int32)
            self.returns = np.full((self.K, self.n), np.nan, np.float32, order="F")
            self.lengths = np.full((self.K, self.n), -1, np.int32, order="F")
        if stage != "PostActStage":
            return
        self.acc = self.acc + env.reward()                 # float32 + float32: the same rounding as the device accumulator
        self.len += 1
        idx = np.nonzero(env.is_terminated())[0]
        keep = idx[self.counts[idx] < self.K]
        self.returns[self.counts[keep], keep] = self.acc[keep]
        self.lengths[self.counts[keep], keep] = self.len[keep]
        self.counts[idx] += 1
        self.acc[idx] = 0
        self.len[idx] = 0


def _snapshot(env):
    return dict(state=env.internal_state(), obs=env.state(), t=env.t(), flags=env.flags(), erng=env.rng_state(), rew=env.reward(),
                act=env.last_action(), ep_ret=env._get(8, (env.n,), np.float32), ep=env.episode_stats())


def _compare(a, b):
    for k in ("state", "obs", "t", "flags", "erng", "rew", "act", "ep_ret"):
        assert same(a[k], b[k]), k
    ea, eb = a["ep"], b["ep"]
    assert ea["episodes"] == eb["episodes"] and ea["length_sum"] == eb["length_sum"] and ea["env_steps"] == eb["env_steps"]
    # (the FP64 sum of Float32 returns is reduced per CTA in the fused kernel, per 256 envs in the step kernel: last bits)
    assert abs(ea["return_sum"] - eb["return_sum"]) <= 1e-6 * max(1.0, abs(eb["return_sum"]))


def _fused_vs_stage(pkg, ctx, make_env, make_net, mode, n_steps, K, expect_fused):
    outs = []
    for fused in (True, False):
        env, net = make_env(), None
        net = make_net(env)
        n = env.n
        seeds = O.splitmix_states_fast(n, 5150)
        if fused:
            rng = seeds.copy() if mode == "sample" else None
            l0 = ctx.launch_count()
            r = pkg.evaluate(net, env, n_steps, max_episodes=K, mode=mode, rng=rng)
            launches = ctx.launch_count() - l0
            if expect_fused:
                assert launches == 2, launches         # reset + one evaluation launch
            else:
                assert launches > n_steps, launches     # staged: several launches per step
            prng = rng
        else:
            policy = pkg.EvaluationPolicy(net, n, mode=mode, rng=seeds if mode == "sample" else None)
            hook = RecordHook(n, K)
            pkg.run(policy, env, pkg.StopAfterNSteps(n_steps), hook)
            r = dict(returns=hook.returns, lengths=hook.lengths, counts=hook.counts)
            prng = policy.rng_state() if mode == "sample" else None
            policy.close()
        outs.append(dict(r=r, env=_snapshot(env), prng=prng))
        net.close(); env.close()
    a, b = outs
    for k in ("returns", "lengths", "counts"):
        assert same(a["r"][k], b["r"][k]), k
    _compare(a["env"], b["env"])
    if mode == "sample":
        assert same(a["prng"], b["prng"]), "policy streams"
        assert not np.array_equal(a["prng"], O.splitmix_states_fast(a["prng"].shape[0], 5150))
    return a


@pytest.mark.parametrize("act", [0, 1], ids=["relu", "tanh"])
@pytest.mark.parametrize("mode", ["greedy", "sample"])
@pytest.mark.parametrize("kind,envkw,algo,n", CASES)
def test_fused_evaluation_is_bit_identical_to_the_stage_protocol(pkg, ctx, kind, envkw, algo, n, mode, act):
    def make_env():
        env = _env(pkg, ctx, kind, n, 9, **envkw)
        if kind == "CartPole" and n == 1000:
            env.set_max_timeout(23)                  # MaxTimeoutEnv inside the fused kernel too
        return env
    a = _fused_vs_stage(pkg, ctx, make_env, lambda env: _net(pkg, ctx, env, kind, act), mode, 230, 2, expect_fused=True)
    assert a["env"]["ep"]["env_steps"] == 230 * n
    assert (a["r"]["counts"] > 0).any()
    c = a["r"]["counts"]
    assert np.all(np.isnan(a["r"]["returns"][1, c < 2])) and np.all(a["r"]["lengths"][1, c < 2] == -1)   # slots nobody reached


def test_fused_evaluation_has_no_env_count_limit(pkg, ctx):
    """200 000 envs = 1 563 tiles: more than the CTAs of the rollout kernel can keep resident; every CTA evaluates several groups."""
    a = _fused_vs_stage(pkg, ctx, lambda: _env(pkg, ctx, "CartPole", 200_000, 31), lambda env: _net(pkg, ctx, env, "CartPole", 0),
                        "greedy", 60, 1, expect_fused=True)
    assert (a["r"]["counts"] > 0).sum() > 1000


def test_q_network_h64_evaluates_fused(pkg, ctx):
    _fused_vs_stage(pkg, ctx, lambda: _env(pkg, ctx, "MountainCar", 3000, 4), lambda env: _net(pkg, ctx, env, "MountainCar", 1, q=True),
                    "greedy", 120, 1, expect_fused=True)


@pytest.mark.parametrize("case", ["q128-greedy", "ac64-no-tc-greedy", "ac64-no-tc-sample", "gauss64-no-tc-greedy", "gauss128-sample"])
def test_staged_evaluation_is_bit_identical_to_the_stage_protocol(pkg, ctx, case):
    kind, hidden, q, tc, mode = {
        "q128-greedy": ("CartPole", 128, True, 1, "greedy"),
        "ac64-no-tc-greedy": ("CartPole", 64, False, 0, "greedy"),
        "ac64-no-tc-sample": ("MountainCar", 64, False, 0, "sample"),
        "gauss64-no-tc-greedy": ("Pendulum", 64, False, 0, "greedy"),
        "gauss128-sample": ("ContinuousCartPole", 128, False, 1, "sample"),
    }[case]
    envkw = dict(continuous=True) if kind == "Pendulum" else {}
    try:
        pkg._lib.check(ctx.lib.b200rl_set_tensor_cores(tc))
        _fused_vs_stage(pkg, ctx, lambda: _env(pkg, ctx, kind, 1500, 12, **envkw), lambda env: _net(pkg, ctx, env, kind, 0, hidden, q),
                        mode, 220, 3, expect_fused=False)
    finally:
        pkg._lib.check(ctx.lib.b200rl_set_tensor_cores(1))


@pytest.mark.parametrize("case", [("cat2", "CartPole", 0), ("cat3", "MountainCar", 0), ("gauss", "Pendulum", 0), ("q64", "CartPole", 64),
                                  ("q128", "MountainCar", 128)])
@pytest.mark.parametrize("act", [0, 1], ids=["relu", "tanh"])
def test_greedy_plan_matches_the_oracle(pkg, ctx, case, act):
    name, kind, qh = case
    n_in = N_IN[kind]
    n = 3000
    obs = np.asfortranarray(np.random.default_rng(7).standard_normal((n_in, n)).astype(np.float32))
    d_obs = ctx.malloc(obs.nbytes); ctx.h2d(d_obs, obs)
    if name == "gauss":
        desc = O.ac_desc(n_in, 64, 1, act, True); kindn, n_out = pkg.KIND_GAUSSIAN, 1
    else:
        n_out = 2 if kind == "CartPole" else 3
        desc = O.ac_desc(n_in, qh or 64, n_out, act); kindn = pkg.KIND_Q if qh else pkg.KIND_CATEGORICAL
    params = O.glorot_params(desc, 19, q_net=bool(qh)) + 0.05 * np.random.default_rng(2).standard_normal(
        O.q_nparams(desc) if qh else O.ac_nparams(desc)).astype(np.float32)
    net = pkg.Network(ctx, n_in, qh or 64, n_out, params, act=act, kind=kindn)
    action = np.empty(n, np.float32 if name == "gauss" else np.int32)
    pkg._lib.check(ctx.lib.b200rl_net_act_greedy(net.h, pkg._lib.ptr(obs), n, pkg._lib.ptr(action), 0))
    d_act = ctx.malloc(n * 4)                                        # device in / out: the same actions
    pkg._lib.check(ctx.lib.b200rl_net_act_greedy(net.h, C.c_void_p(d_obs), n, C.c_void_p(d_act), 1))
    assert same(ctx.d2h(np.empty_like(action), d_act), action)
    seeds = O.splitmix_states_fast(n, 3)
    if qh:
        heads, ref = net.values(obs), O.q_values(desc, params, obs)
    else:
        d_rng = ctx.malloc(n * 32); ctx.h2d(d_rng, seeds)
        heads = net.act(obs, d_rng)["heads"]
        ctx.free(d_rng)
        ref = O.act_gaussian(desc, O.hyper_array(), params, obs, seeds)["mu"][None, :] if name == "gauss" else O.act_discrete(desc, params, obs, seeds)["logits"]
    if name == "gauss":
        assert rel_err(heads[0], ref[0]) < REL
        assert same(action, heads[0])                             # mu itself, bit for bit, as b200rl_net_act reports it
    else:
        assert rel_err(heads, ref) < REL
        assert np.array_equal(action, heads.argmax(0) + 1)           # the device's own head outputs (no NaN / ties here)
        top2 = np.sort(ref, axis=0)[-2:]
        safe = (top2[1] - top2[0]) > 1e-4 * (1 + np.abs(ref).max(0))
        assert safe.mean() > 0.99 and np.array_equal(action[safe], ref.argmax(0)[safe] + 1)
    ctx.free(d_obs); ctx.free(d_act); net.close()


def test_evaluation_between_iterations_leaves_training_untouched(pkg, ctx):
    n, T = 2048, 8
    R = pkg.learners
    outs = []
    for with_eval in (True, False):
        env = _env(pkg, ctx, "CartPole", n, 41)
        net = _net(pkg, ctx, env, "CartPole", 0)
        agent = pkg.OnPolicyAgent(ctx, net, env, pkg.onpolicy_config(update_freq=T, n_epochs=2, n_microbatches=2), O.splitmix_states_fast(n, 42),
                                  host_actions=False)
        env.reset_(is_force=True)
        if with_eval:
            agent.iterate(2)
            ev_env = _env(pkg, ctx, "CartPole", 3000, 43)
            r = pkg.evaluate(net, ev_env, 250)
            assert (r["counts"] >= 1).all()
            r = pkg.evaluate(net, ev_env, 40, mode="sample", rng=O.splitmix_states_fast(3000, 44))
            ev_env.close()
            agent.iterate(3)
        else:
            agent.iterate(5)
        outs.append(dict(params=net.get(), m=net.get(R.NET_M), v=net.get(R.NET_V), bt=net.get(R.NET_BETA_T), step=net.step_count(),
                         prng=agent.rollout(R.ROLL_RNG), env=_snapshot(env), graph=agent.graph_active()))
        agent.close(); net.close(); env.close()
    a, b = outs
    for k in ("params", "m", "v", "bt", "prng"):
        assert same(a[k], b[k]), k
    assert a["step"] == b["step"] and a["graph"] and b["graph"]
    _compare(a["env"], b["env"])
    assert a["env"]["ep"]["return_sum"] == b["env"]["ep"]["return_sum"]


# ---- known answer: a linear CartPole controller as a relu network ---------------------------------------------------------
GAINS = np.float32([0.1, 0.5, 1.0, 1.0])   # push right when 0.1 x + 0.5 xdot + theta + thetadot > 0


def _time_limit_share(lengths, states, params):
    """share of first episodes that ended at the time limit (t > max_steps) inside the position and angle thresholds"""
    max_steps = int(params[10])
    ok = (lengths == max_steps + 1) & (np.abs(states[:, 0]) <= params[9]) & (np.abs(states[:, 2]) <= params[8])
    return ok.mean()


def test_linear_controller_gains_balance_the_oracle_cartpole(oracle):
    n = 4096
    env = O.OracleVecEnv(O.KIND_CARTPOLE, n, O.splitmix_states_fast(n, 5))
    env.reset(force=True)
    p = O.default_params(O.KIND_CARTPOLE)
    first_len = np.zeros(n, np.int32); first_state = np.zeros((n, 4), np.float32); done = np.zeros(n, bool)
    for _ in range(230):
        u = (env.get(O.F_OBS) * GAINS).sum(1, dtype=np.float32)
        env.step(np.where(u > 0, 2, 1).astype(np.int32), auto_reset=False)
        term = env.get(O.F_TERMINAL).astype(bool)
        new = term & ~done
        first_len[new] = env.get(O.F_T)[new]; first_state[new] = env.get(O.F_STATE)[new]
        done |= term
    assert done.all() and _time_limit_share(first_len, first_state, p) >= 0.95


def _controller_params():
    """Actor: logit(2) - logit(1) = relu(u) - relu(-u) = u with u = GAINS . obs; critic zero."""
    H = 64
    W1 = np.zeros((H, 4), np.float32); W1[0] = GAINS; W1[1] = -GAINS
    W2 = np.zeros((H, H), np.float32); W2[0, 0] = 1; W2[1, 1] = 1
    W3 = np.zeros((2, H), np.float32); W3[1, 0] = 1; W3[1, 1] = -1
    actor = [W1.ravel(order="F"), np.zeros(H, np.float32), W2.ravel(order="F"), np.zeros(H, np.float32), W3.ravel(order="F"), np.zeros(2, np.float32)]
    critic_n = O.ac_nparams(O.ac_desc(4, H, 2)) - sum(a.size for a in actor)
    return np.concatenate(actor + [np.zeros(critic_n, np.float32)])


def test_greedy_evaluation_of_a_known_controller_reaches_the_time_limit(pkg, ctx):
    n = 4096
    params = _controller_params()
    net = pkg.Network(ctx, 4, 64, 2, params, act=0, kind=pkg.KIND_CATEGORICAL)
    env = _env(pkg, ctx, "CartPole", n, 5)
    r = pkg.evaluate(net, env, 230, max_episodes=1)
    p = O.default_params(O.KIND_CARTPOLE)
    assert (r["counts"] >= 1).all()
    # the time limit: t = max_steps + 1 at termination, every step rewarded 1 but the terminal one (CartPoleEnv.jl:84)
    at_limit = r["lengths"][0] == int(p[10]) + 1
    assert at_limit.mean() >= 0.95
    assert np.all(r["returns"][0][at_limit] == int(p[10]))
    # RandomPolicy on the same envs: almost never
    env2 = _env(pkg, ctx, "CartPole", n, 5)
    hook = RecordHook(n, 1)
    pkg.run(pkg.RandomPolicy(), env2, pkg.StopAfterNSteps(230), hook)
    assert (hook.lengths[0] == int(p[10]) + 1).mean() < 0.01
    # sampling the same network: the logit gap is |u| (small), so sampled episodes fail far more often than greedy ones
    env3 = _env(pkg, ctx, "CartPole", n, 5)
    rs = pkg.evaluate(net, env3, 230, mode="sample", rng=O.splitmix_states_fast(n, 6))
    assert (rs["lengths"][0] == int(p[10]) + 1).mean() < at_limit.mean() - 0.3
    net.close(); env.close(); env2.close(); env3.close()


# ---- refusals ------------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_env_untouched(pkg, ctx):
    L = pkg._lib
    n = 300

    def call(net, env, mode=0, n_steps=10, K=1, rng=None):
        cfg = L.EvalConfig(mode, n_steps, K)
        ret = np.zeros((max(K, 1), env.n), np.float32); cnt = np.zeros(env.n, np.int32)
        before = (env.internal_state(), env.rng_state(), env.t(), env.flags(), env.episode_stats())
        st = ctx.lib.b200rl_evaluate(net.h, env.h, C.byref(cfg), None if rng is None else C.c_void_p(rng), L.ptr(ret), None, L.ptr(cnt), 0)
        after = (env.internal_state(), env.rng_state(), env.t(), env.flags(), env.episode_stats())
        if st != L.OK:
            for x, y in zip(before[:4], after[:4]):
                assert same(x, y)
            assert before[4] == after[4] and not cnt.any()
        return st

    cp = _env(pkg, ctx, "CartPole", n, 1)
    net = _net(pkg, ctx, cp, "CartPole", 0)
    qnet = _net(pkg, ctx, cp, "CartPole", 0, q=True)
    d_rng = ctx.malloc(n * 32); ctx.h2d(d_rng, O.splitmix_states_fast(n, 2))
    f64 = pkg.B200VecEnv(ctx, "CartPole", n, O.splitmix_states_fast(n, 1), T=np.float64, auto_reset=True)
    acro = pkg.B200VecEnv(ctx, "Acrobot", n, O.splitmix_states_fast(n, 1), T=np.float64, auto_reset=True)
    mc = _env(pkg, ctx, "MountainCar", n, 1)
    pend = _env(pkg, ctx, "Pendulum", n, 1, continuous=True)
    pend5 = _env(pkg, ctx, "Pendulum", n, 1, continuous=False, n_actions=5)
    net3 = pkg.Network(ctx, 3, 64, 3, O.glorot_params(O.ac_desc(3, 64, 3), 1), kind=pkg.KIND_CATEGORICAL)
    assert call(net, f64) == L.ERR_UNSUPPORTED
    assert call(net, acro) == L.ERR_UNSUPPORTED
    assert call(qnet, cp, mode=1, rng=d_rng) == L.ERR_UNSUPPORTED
    assert call(net, mc) == L.ERR_INVALID                  # 4 inputs, 2 observations
    assert call(net3, pend5) == L.ERR_INVALID              # 3 logits, 5 actions
    assert call(net3, pend) == L.ERR_INVALID               # categorical head, continuous actions
    assert call(net, cp, n_steps=0) == L.ERR_INVALID
    assert call(net, cp, K=-1) == L.ERR_INVALID
    assert call(net, cp, mode=1) == L.ERR_INVALID          # no streams
    assert call(net, cp, mode=2) == L.ERR_INVALID
    assert call(net, cp, n_steps=5, K=0) == L.OK           # K = 0: counts only
    with pytest.raises(ValueError):
        pkg.EvaluationPolicy(net, n, mode="sample")
    ctx.free(d_rng)
    for h in (net, qnet, net3, cp, f64, acro, mc, pend, pend5):
        h.close()
