"""Float64 envs behind StateTransformedEnv(env; state_mapping = s -> Float32.(s)) (B200VecEnv.set_state_float32) on the device.

The wrapper leaves the dynamics alone: a wrapped and an unwrapped Float64 env driven with the same actions stay bit-identical in
every field, and the Float32 mirror the learners read is np.float32 of the Float64 observation after every kind of write.  The
learners then run on the mirror: the fused PPO / A2C rollout (graph-replayed iterate), the staged plan! / act! launches, the
host-action stage protocol, the device DQN loop and the evaluation kernels must all agree bit for bit, and the rollout's states and
rewards must be Float32 of the oracle's Float64 trajectory under the recorded actions."""
import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu

_OKIND = {"CartPole": O.KIND_CARTPOLE, "Pendulum": O.KIND_PENDULUM, "MountainCar": O.KIND_MOUNTAINCAR,
          "ContinuousMountainCar": O.KIND_MOUNTAINCAR_CONT}
_NIN = {"CartPole": 4, "Pendulum": 3, "MountainCar": 2, "ContinuousMountainCar": 2}
ENVS = [("CartPole", {}), ("Pendulum", dict(continuous=True)), ("Pendulum", dict(continuous=False, n_actions=3)),
        ("MountainCar", {}), ("ContinuousMountainCar", {})]


def _bits(x):
    x = np.asarray(x)
    return x.dtype, x.shape, x.tobytes(order="A")


def _env(pkg, ctx, kind, n, seed, wrapped=True, **kw):
    env = pkg.B200VecEnv(ctx, kind, n, O.splitmix_states_fast(n, seed), T=np.float64, auto_reset=True, **kw)
    if wrapped:
        env.set_state_float32()
    return env


FIELD_OBS = 1   # include/b200rl.h: state(env) in the env's own T


def _obs64(env):
    return env._get(FIELD_OBS, env.state().shape, np.float64)


def _fields(env):
    return dict(state=env.internal_state(), obs=_obs64(env), rew=env.reward(), flags=env.flags(), t=env.t(), rng=env.rng_state(),
                act=env.last_action(), ep=env.episode_stats())


def _same_fields(a, b):
    """every env field bit for bit; of the episode statistics the counts exactly and the return sum (Float32 per-warp partial sums,
    grouped by launch shape) to 1e-6"""
    for f in a:
        if f == "ep":
            assert (a[f]["episodes"], a[f]["length_sum"], a[f]["env_steps"]) == (b[f]["episodes"], b[f]["length_sum"], b[f]["env_steps"])
            assert abs(a[f]["return_sum"] - b[f]["return_sum"]) <= 1e-6 * max(1.0, abs(b[f]["return_sum"]))
        else:
            assert _bits(a[f]) == _bits(b[f]), f


def _mirror_ok(env):
    return _bits(env.state()) == _bits(_obs64(env).astype(np.float32))


@pytest.mark.parametrize("kind,kw", ENVS, ids=[f"{k}-{'-'.join(map(str, v.values()))}" for k, v in ENVS])
def test_wrapper_leaves_the_dynamics_alone_and_the_mirror_follows(pkg, ctx, kind, kw):
    n, steps = 1031, 450
    a, b = _env(pkg, ctx, kind, n, 5, **kw), _env(pkg, ctx, kind, n, 5, wrapped=False, **kw)
    assert a.state().dtype == np.float32 and b.state().dtype == np.float64 and _mirror_ok(a)
    with pytest.raises(pkg.B200RLError):                       # no Float32 view without the wrapper
        b.device_ptr(pkg._lib.FIELD_OBS_F32)
    r = np.random.default_rng(1)
    for k in range(steps):
        if a.continuous:
            lo, hi = a.action_space()
            act = r.uniform(lo, hi, n)
        else:
            act = r.integers(1, len(a.action_space()) + 1, n).astype(np.int32)
        a.act_(act); b.act_(act)
        if k == 200:
            b.set_state_float32()                                # turned on mid-run
            assert _mirror_ok(b)
        if k % 50 == 0 or k > steps - 3:
            fa, fb = _fields(a), _fields(b)
            for f in fa:
                assert (fa[f] == fb[f]) if f == "ep" else _bits(fa[f]) == _bits(fb[f]), (k, f)
            assert _mirror_ok(a), k
    assert a.episode_stats()["episodes"] > 0
    a.reset_(is_force=True); assert _mirror_ok(a)
    st = a.internal_state() * 1.5 + 0.25
    a.set_field(pkg._lib.FIELD_STATE, st); assert _mirror_ok(a)
    c = a.copy(); assert _mirror_ok(c) and _bits(c.state()) == _bits(a.state()) and c.state_f32
    c.act_(act); a.act_(act)
    assert _bits(c.state()) == _bits(a.state()) and _mirror_ok(c)
    a.set_state_float32(False)
    assert a.state().dtype == np.float64
    for e in (a, b, c):
        e.close()


def test_refusals(pkg, ctx):
    L = pkg._lib
    raw = _env(pkg, ctx, "Pendulum", 64, 1, wrapped=False, continuous=True)
    desc = O.ac_desc(3, 64, 1, 0, True)
    net = pkg.Network(ctx, 3, 64, 1, O.glorot_params(desc, 1), kind=pkg.KIND_GAUSSIAN)
    with pytest.raises(pkg.B200RLError) as ei:
        pkg.OnPolicyAgent(ctx, net, raw, pkg.onpolicy_config(update_freq=4, n_epochs=1, n_microbatches=1), O.splitmix_states_fast(64, 2))
    assert ei.value.status == L.ERR_UNSUPPORTED and "Float32" in str(ei.value)
    raw.set_state_float32()                                     # wrapped: accepted ...
    agent = pkg.OnPolicyAgent(ctx, net, raw, pkg.onpolicy_config(update_freq=4, n_epochs=1, n_microbatches=1), O.splitmix_states_fast(64, 2),
                              host_actions=False)
    agent.collect(2)
    raw.set_state_float32(False)                                # ... and refused again once the wrapper is gone
    with pytest.raises(pkg.B200RLError) as ei:
        agent.collect(1)
    assert ei.value.status == L.ERR_UNSUPPORTED
    agent.close(); net.close(); raw.close()
    acro = pkg.B200VecEnv(ctx, "Acrobot", 16, O.splitmix_states_fast(16, 3), T=np.float64)
    before = acro.state()
    assert ctx.lib.b200rl_env_set_state_f32(acro.h, 1) == L.ERR_UNSUPPORTED
    assert _bits(acro.state()) == _bits(before) and acro.state().dtype == np.float64
    acro.close()
    f32 = pkg.B200VecEnv(ctx, "CartPole", 16, O.splitmix_states_fast(16, 4))
    f32.set_state_float32()                                     # the identity on a Float32 env
    assert f32.device_ptr(L.FIELD_OBS_F32) == f32.device_ptr(L.FIELD_OBS)
    f32.close()


# ---------------------------------------------------------------------------------------------------------------- PPO / A2C
def _onpolicy(pkg, ctx, kind, kw, n, T, algo, hidden=64, host_actions=False, max_timeout=0):
    env = _env(pkg, ctx, kind, n, 9, **kw)
    if max_timeout:
        env.set_max_timeout(max_timeout)
    n_in = _NIN[kind]
    n_out, net_kind = (1, pkg.KIND_GAUSSIAN) if env.continuous else (len(env.action_space()), pkg.KIND_CATEGORICAL)
    desc = O.ac_desc(n_in, hidden, n_out, 0, env.continuous)
    params = O.glorot_params(desc, 77) + 0.05 * np.random.default_rng(3).standard_normal(O.ac_nparams(desc)).astype(np.float32)
    net = pkg.Network(ctx, n_in, hidden, n_out, params, act=0, kind=net_kind)
    cfg = pkg.onpolicy_config(update_freq=T, n_epochs=2, n_microbatches=2, algo=algo)
    agent = pkg.OnPolicyAgent(ctx, net, env, cfg, O.splitmix_states_fast(n, 10), host_actions=host_actions)
    env.reset_(is_force=True)
    return env, net, agent


def _snap(pkg, env, net, agent):
    R = pkg.learners
    out = {f"roll{f}": agent.rollout(f) for f in (R.ROLL_STATE, R.ROLL_ACTION, R.ROLL_LOGP, R.ROLL_REWARD, R.ROLL_TERMINAL, R.ROLL_VALUE, R.ROLL_RNG)}
    out.update(params=net.get(), m=net.get(R.NET_M), v=net.get(R.NET_V), bt=net.get(R.NET_BETA_T), state=env.internal_state(),
               obs=env.state(), erng=env.rng_state(), t=env.t(), flags=env.flags())
    return out


ONP = [("CartPole", {}, "ppo", 127, 64), ("Pendulum", dict(continuous=True), "a2c", 127, 64),
       ("Pendulum", dict(continuous=False, n_actions=3), "ppo", 1, 64), ("MountainCar", {}, "ppo", 127, 128),
       ("ContinuousMountainCar", {}, "a2c", 65537, 64), ("CartPole", {}, "a2c", 127, 128)]


@pytest.mark.parametrize("kind,kw,algo,n,hidden", ONP)
def test_onpolicy_paths_agree_and_follow_the_oracle(pkg, ctx, kind, kw, algo, n, hidden):
    """On the tensor cores: iterate (fused rollout, graph replay) == collect + update == the host-action stage protocol.  With
    them off (CUDA-core forward and backward, staged plan! / act! launches): collect + update == the stage protocol.  (The two
    compute paths round differently, Float32 envs alike, so each is compared with itself.)  The rollout's states and rewards are
    Float32 of the oracle's Float64 trajectory under the recorded actions."""
    T, iters = 8, 3
    mt = 5 if (kind == "CartPole" and algo == "a2c") else 0       # MaxTimeoutEnv inside the wrapped env
    snaps = []
    for path, tc in (("iterate", 1), ("collect", 1), ("stage", 1), ("collect", 0), ("stage", 0)):
        env, net, agent = _onpolicy(pkg, ctx, kind, kw, n, T, algo, hidden, host_actions=path == "stage", max_timeout=mt)
        ctx.lib.b200rl_set_tensor_cores(tc)
        try:
            if path == "iterate":
                agent.iterate(iters)
                assert agent.graph_active() or hidden != 64
            elif path == "collect":
                for _ in range(iters):
                    agent.collect(3); agent.collect(T - 3); agent.update()     # a rollout filled in two stretches
            else:
                for _ in range(iters * T):
                    a = agent.plan(env)
                    env.act_(a)
                    agent.push(pkg.core.PostActStage, env)
                    agent.optimise(pkg.core.PostActStage)
        finally:
            ctx.lib.b200rl_set_tensor_cores(1)
        snaps.append(_snap(pkg, env, net, agent))
        agent.close(); net.close(); env.close()
    for a, b in ((snaps[0], snaps[1]), (snaps[0], snaps[2]), (snaps[3], snaps[4])):
        for k in a:
            assert _bits(a[k]) == _bits(b[k]), k
    # one fused rollout against the oracle's Float64 trajectory under the recorded actions
    env, net, agent = _onpolicy(pkg, ctx, kind, kw, n, T, algo, hidden, max_timeout=mt)
    agent.collect(T)
    R = pkg.learners
    S, A, RW, TM = (agent.rollout(f) for f in (R.ROLL_STATE, R.ROLL_ACTION, R.ROLL_REWARD, R.ROLL_TERMINAL))
    params = None
    if kind == "Pendulum":
        params = O.default_params(O.KIND_PENDULUM, "f64").copy()
        params[7], params[8] = 3, float(kw["continuous"])
    ref = O.OracleVecEnv(_OKIND[kind], n, O.splitmix_states_fast(n, 9), dtype="f64", params=params)
    if mt:
        ref.set_max_timeout(mt)
    ref.reset(force=True)
    lo, hi = (-2.0, 2.0) if kind == "Pendulum" else (-1.0, 1.0)
    for t in range(T):
        assert _bits(np.ascontiguousarray(S[:, :, t].T)) == _bits(ref.get(O.F_OBS).astype(np.float32)), t
        act = np.clip(A[:, t], np.float32(lo), np.float32(hi)).astype(np.float64) if env.continuous else A[:, t]
        assert ref.step(act, auto_reset=True) == 0
        assert _bits(RW[:, t]) == _bits(ref.get(O.F_REWARD).astype(np.float32)), t
        assert np.array_equal(TM[:, t], ref.get(O.F_TERMINAL) & 1), t
    agent.close(); net.close(); env.close()


def test_iterate_recaptures_when_the_wrapper_is_toggled(pkg, ctx):
    T = 8
    outs = []
    for graph in (True, False):
        env, net, agent = _onpolicy(pkg, ctx, "CartPole", {}, 300, T, "ppo")
        for phase in range(2):
            if graph:
                agent.iterate(2)
            else:
                for _ in range(2):
                    agent.collect(T); agent.update()
            if phase == 0:
                env.set_state_float32(False)
                with pytest.raises(pkg.B200RLError):
                    agent.iterate(1) if graph else agent.collect(T)
                env.set_state_float32(True)
        if graph:
            assert agent.graph_active()
        outs.append(_snap(pkg, env, net, agent))
        agent.close(); net.close(); env.close()
    for k in outs[0]:
        assert _bits(outs[0][k]) == _bits(outs[1][k]), k


def test_onpolicy_checkpoint_resumes_bit_for_bit(pkg, ctx):
    T = 8
    env, net, agent = _onpolicy(pkg, ctx, "Pendulum", dict(continuous=True), 257, T, "ppo")
    agent.iterate(1); agent.collect(3)
    ck = pkg.checkpoint.checkpoint(env=env, net=net, agent=agent)
    agent.collect(T - 3); agent.update(); agent.iterate(1)
    want = _snap(pkg, env, net, agent)
    env2 = pkg.B200VecEnv(ctx, "Pendulum", 257, O.splitmix_states_fast(257, 999), T=np.float64, auto_reset=True, continuous=True)
    env2.set_state_float32()
    desc = O.ac_desc(3, 64, 1, 0, True)
    net2 = pkg.Network(ctx, 3, 64, 1, O.glorot_params(desc, 5), act=0, kind=pkg.KIND_GAUSSIAN)
    agent2 = pkg.OnPolicyAgent(ctx, net2, env2, pkg.onpolicy_config(update_freq=T, n_epochs=2, n_microbatches=2), O.splitmix_states_fast(257, 998),
                               host_actions=False)
    pkg.checkpoint.restore(ck, env=env2, net=net2, agent=agent2)
    agent2.collect(T - 3); agent2.update(); agent2.iterate(1)
    got = _snap(pkg, env2, net2, agent2)
    for k in want:
        assert _bits(want[k]) == _bits(got[k]), k
    for o in (agent, net, env, agent2, net2, env2):
        o.close()


# ---------------------------------------------------------------------------------------------------------------------- DQN
_NA = {"CartPole": 2, "MountainCar": 3, "Pendulum": 3}


def _dqn(pkg, ctx, seed, env_kind="CartPole", lanes=127, hidden=64, prioritized=True, explorer="linear", n_step=1, dueling=False):
    kw = dict(continuous=False, n_actions=3) if env_kind == "Pendulum" else {}
    env = _env(pkg, ctx, env_kind, lanes, seed, **kw)
    ns, na = _NIN[env_kind], _NA[env_kind]
    kind = pkg.KIND_DUELING if dueling else pkg.KIND_Q
    n_par = pkg.Network.count_params(ctx, ns, hidden, na, act=0, kind=kind)
    p = (0.3 * np.random.default_rng(seed + 1).standard_normal(n_par)).astype(np.float32)
    net = pkg.Network(ctx, ns, hidden, na, p, act=0, kind=kind)
    traj = pkg.Trajectory(ctx, ns, 16, lanes=lanes, batch_size=256, sampler_rng=O.splitmix_states_fast(256, seed + 2), prioritized=prioritized)
    if n_step > 1:
        traj.set_nstep(n_step, 0.99)
    traj.controller = pkg.InsertSampleRatioController(ratio=1.0, threshold=3)
    learner = pkg.DQNLearner(ctx, net, traj, pkg.dqn_config(target_update_freq=5))
    ex = (pkg.WeightedSoftmaxExplorer() if explorer == "softmax" else
          pkg.EpsilonGreedyExplorer(0.05, eps_init=1.0, warmup_steps=2 * lanes, decay_steps=10 * lanes))
    policy = pkg.QBasedPolicy(ctx, learner, ex, O.splitmix_states_fast(lanes, seed + 3), lanes)
    return dict(env=env, net=net, traj=traj, policy=policy, agent=pkg.Agent(policy, traj))


DQN = [dict(env_kind="CartPole"), dict(env_kind="MountainCar", hidden=128, prioritized=False),
       dict(env_kind="Pendulum", n_step=3), dict(env_kind="CartPole", dueling=True, explorer="softmax"),
       dict(env_kind="MountainCar", dueling=True, hidden=128)]


@pytest.mark.parametrize("kw", DQN, ids=lambda d: "-".join(f"{k}={v}" for k, v in d.items()))
def test_replay_loop_equals_the_stage_protocol(pkg, ctx, kw):
    steps = 40
    fast, stage = _dqn(pkg, ctx, 100, **kw), _dqn(pkg, ctx, 100, **kw)
    stage["agent"].fusable = False
    for n in (steps, 7):
        pkg.run(fast["agent"], fast["env"], pkg.StopAfterNSteps(n), pkg.EmptyHook())
        pkg.run(stage["agent"], stage["env"], pkg.StopAfterNSteps(n), pkg.EmptyHook())
        if n == steps:
            fast["env"].set_state_float32(False); fast["env"].set_state_float32(True)   # toggled: the graphs are re-keyed
    assert fast["agent"]._replay is not None and stage["agent"]._replay is None
    a = pkg.checkpoint.checkpoint_replay(fast["env"], fast["net"], fast["agent"])
    b = pkg.checkpoint.checkpoint_replay(stage["env"], stage["net"], stage["agent"])
    for k in a:
        if k == "env/episode_stats":
            assert np.array_equal(a[k][[0, 2, 3]], b[k][[0, 2, 3]]) and abs(a[k][1] - b[k][1]) <= 1e-9 * max(1.0, abs(b[k][1]))
            continue
        assert _bits(a[k]) == _bits(b[k]), k
    st = a["traj/state"]
    assert st.dtype == np.float32 and np.isfinite(st).all()
    for s in (fast, stage):
        s["agent"].close()
        for k in ("policy", "traj", "net", "env"):
            s[k].close()


def test_raw_float64_env_keeps_the_replay_loop_off(pkg, ctx):
    s = _dqn(pkg, ctx, 7)
    s["env"].set_state_float32(False)
    assert not s["agent"].replay_supported(s["env"])
    with pytest.raises(pkg.B200RLError):
        s["traj"].push_env(s["env"])
    s["agent"].close()
    for k in ("policy", "traj", "net", "env"):
        s[k].close()


# --------------------------------------------------------------------------------------------------------------- evaluation
class Float32RecordHook:
    """the evaluation records as the stage protocol sees them: per env the Float32 sum of Float32(reward) in step order and the
    length, for the first K episodes, and how many ended"""
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
        self.acc = self.acc + env.reward().astype(np.float32)
        self.len += 1
        idx = np.nonzero(env.is_terminated())[0]
        keep = idx[self.counts[idx] < self.K]
        self.returns[self.counts[keep], keep] = self.acc[keep]
        self.lengths[self.counts[keep], keep] = self.len[keep]
        self.counts[idx] += 1
        self.acc[idx] = 0
        self.len[idx] = 0

    def records(self):
        return dict(returns=self.returns, lengths=self.lengths, counts=self.counts)


def _same_records(a, b):
    for k in ("returns", "lengths", "counts"):
        assert _bits(a[k]) == _bits(b[k]), k


@pytest.mark.parametrize("kind,kw,mode", [("CartPole", {}, "greedy"), ("Pendulum", dict(continuous=True), "sample"),
                                          ("ContinuousMountainCar", {}, "greedy"), ("MountainCar", {}, "sample")])
def test_evaluate_fused_staged_and_run_agree(pkg, ctx, kind, kw, mode):
    """fused == run(EvaluationPolicy) on the tensor-core path; the staged launches == run(EvaluationPolicy) with tensor cores off"""
    n, steps = 300, 260
    outs = []
    for path, tc in (("fused", 1), ("run", 1), ("staged", 0), ("run", 0)):
        ctx.lib.b200rl_set_tensor_cores(tc)
        env = _env(pkg, ctx, kind, n, 21, **kw)
        n_in = _NIN[kind]
        n_out, nk = (1, pkg.KIND_GAUSSIAN) if env.continuous else (len(env.action_space()), pkg.KIND_CATEGORICAL)
        desc = O.ac_desc(n_in, 64, n_out, 1, env.continuous)
        net = pkg.Network(ctx, n_in, 64, n_out, O.glorot_params(desc, 4), act=1, kind=nk)
        rng = O.splitmix_states_fast(n, 22).copy() if mode == "sample" else None
        try:
            if path == "run":
                pol = pkg.EvaluationPolicy(net, n, mode=mode, rng=rng)
                hook = Float32RecordHook(n, 2)
                pkg.run(pol, env, pkg.StopAfterNSteps(steps), hook)
                rec = hook.records()
                prng = pol.rng_state() if mode == "sample" else None
                pol.close()
            else:
                rec = pkg.evaluate(net, env, steps, max_episodes=2, mode=mode, rng=rng)
                prng = rng
        finally:
            ctx.lib.b200rl_set_tensor_cores(1)
        outs.append(dict(rec=rec, f=_fields(env), prng=prng))
        net.close(); env.close()
    for a, o in ((outs[0], outs[1]), (outs[2], outs[3])):
        _same_records(a["rec"], o["rec"])
        _same_fields(a["f"], o["f"])
        if mode == "sample":
            assert _bits(a["prng"]) == _bits(o["prng"])
    assert (outs[0]["rec"]["counts"] > 0).any() or kind == "MountainCar"


@pytest.mark.parametrize("explorer", ["greedy", "linear"])
def test_evaluate_explore_fused_staged_and_run_agree(pkg, ctx, explorer):
    n, steps = 300, 230
    outs = []
    for path, tc in (("fused", 1), ("run", 1), ("staged", 0), ("run", 0)):
        ctx.lib.b200rl_set_tensor_cores(tc)
        env = _env(pkg, ctx, "Pendulum", n, 31, continuous=False, n_actions=3)
        net = pkg.Network(ctx, 3, 64, 3, (0.3 * np.random.default_rng(2).standard_normal(pkg.Network.count_params(ctx, 3, 64, 3, act=0, kind=pkg.KIND_Q))).astype(np.float32),
                          act=0, kind=pkg.KIND_Q)
        traj = pkg.Trajectory(ctx, 3, 8, lanes=n, batch_size=32, sampler_rng=O.splitmix_states_fast(32, 3))
        learner = pkg.DQNLearner(ctx, net, traj, pkg.dqn_config())
        ex = pkg.GreedyExplorer() if explorer == "greedy" else pkg.EpsilonGreedyExplorer(0.1, eps_init=1.0, warmup_steps=n, decay_steps=50 * n)
        pol = pkg.QBasedPolicy(ctx, learner, ex, O.splitmix_states_fast(n, 32), n)
        try:
            if path == "run":
                hook = Float32RecordHook(n, 2)
                pkg.run(pol, env, pkg.StopAfterNSteps(steps), hook)
                rec = hook.records()
            else:
                rec = pkg.evaluate(pol, env, steps, max_episodes=2)
        finally:
            ctx.lib.b200rl_set_tensor_cores(1)
        outs.append(dict(rec=rec, f=_fields(env), xrng=pol.explorer_rng(), step=getattr(ex, "step", 0)))
        pol.close(); traj.close(); net.close(); env.close()
    for a, o in ((outs[0], outs[1]), (outs[2], outs[3]), (outs[0], outs[2])):
        _same_records(a["rec"], o["rec"])
        _same_fields(a["f"], o["f"])
        assert _bits(a["xrng"]) == _bits(o["xrng"]) and a["step"] == o["step"]


# ------------------------------------------------------------------------------------------------------------- fused kernels
@pytest.mark.parametrize("kind,kw", ENVS, ids=[f"{k}-{'-'.join(map(str, v.values()))}" for k, v in ENVS])
def test_float64_envs_take_the_fused_kernels(pkg, ctx, kind, kw):
    """A wrapped Float64 env runs the Float64 instantiations of the fused kernels, not the staged fallback: the rollout, the
    evaluation (modes 0, 1 and, discrete, 2) and the DQN collect launch exactly what the same call on a Float32 env launches (one
    kernel per stretch), while the staged path would launch several kernels per env step."""
    n, T, steps = 300, 8, 20
    counts = {}
    for f64 in (False, True):
        env = pkg.B200VecEnv(ctx, kind, n, O.splitmix_states_fast(n, 3), T=np.float64 if f64 else np.float32, auto_reset=True, **kw)
        if f64:
            env.set_state_float32()
        n_in = _NIN[kind]
        n_out, nk = (1, pkg.KIND_GAUSSIAN) if env.continuous else (len(env.action_space()), pkg.KIND_CATEGORICAL)
        desc = O.ac_desc(n_in, 64, n_out, 0, env.continuous)
        net = pkg.Network(ctx, n_in, 64, n_out, O.glorot_params(desc, 4), act=0, kind=nk)
        agent = pkg.OnPolicyAgent(ctx, net, env, pkg.onpolicy_config(update_freq=T, n_epochs=1, n_microbatches=1), O.splitmix_states_fast(n, 4),
                                  host_actions=False)
        agent.collect(1)                                          # (first launch: module load, shared-memory attribute)
        c = {}
        l0 = ctx.launch_count(); agent.collect(T - 1); c["rollout"] = ctx.launch_count() - l0
        agent.close()
        for mode in ("greedy", "sample"):
            rng = O.splitmix_states_fast(n, 5).copy() if mode == "sample" else None
            pkg.evaluate(net, env, 4, mode=mode, rng=rng)
            l0 = ctx.launch_count(); pkg.evaluate(net, env, steps, mode=mode, rng=rng); c[mode] = ctx.launch_count() - l0
        net.close()
        if not env.continuous:
            s = _dqn(pkg, ctx, 11, env_kind="Pendulum" if kind == "Pendulum" else kind, lanes=n, prioritized=False)
            s["env"].close()
            s["env"] = env
            s["traj"].controller = pkg.InsertSampleRatioController(ratio=1.0, threshold=10 ** 6)   # collect only
            pkg.run(s["agent"], env, pkg.StopAfterNSteps(2), pkg.EmptyHook())
            assert s["agent"]._replay is not None
            l0 = ctx.launch_count(); s["agent"].run_replay(env, steps); c["replay"] = ctx.launch_count() - l0
            pkg.evaluate(s["policy"], env, 4)
            l0 = ctx.launch_count(); pkg.evaluate(s["policy"], env, steps); c["explore"] = ctx.launch_count() - l0
            s["agent"].close()
            for k in ("policy", "traj", "net"):
                s[k].close()
        env.close()
        counts[f64] = c
    assert counts[True] == counts[False], counts
    assert counts[True]["rollout"] == 1 and counts[True]["greedy"] == counts[True]["sample"] == 2, counts   # (evaluate: reset + 1)
    if "replay" in counts[True]:
        assert counts[True]["replay"] <= 2 and counts[True]["explore"] == 2, counts   # one collect window (+ the explorer step)
