"""GPU tests of the device episode log (b200rl_env_episode_log, DeviceEpisodeLog): the per-env episode lists it hands to the host
equal those of BatchStepsPerEpisode + TotalBatchRewardPerEpisode (lengths exactly, returns bit for bit against a Float32
step-order restatement and equal to the host hook where rewards are integers), under K1 (RandomPolicy and host actions, auto and
soft reset, MaxTimeoutEnv, Float32 and Float64 envs), the fused PPO / A2C iteration and the DQN replay loop (fused and staged
collect), on a sharded ctx, and without changing what those paths compute.  Evaluation is not logged, an overflowing window is an
error, a detached log leaves the run it would have been, and one env is recorded by one hook at a time.

Coverage of the K1 matrix: N = 1 and 127 run every env kind, dtype and reset mode; N = 65 537 runs CartPole and the Pendulum
variants with auto-reset and MaxTimeoutEnv only.  Without MaxTimeoutEnv only CartPole and ContinuousCartPole run: the other kinds'
episodes (200 steps, or MountainCar's goal) would not end inside the 150-step window, so they take a 45-step timeout instead."""
import threading

import numpy as np
import pytest

import oracle_lib as O
import test_replay_sharded_gpu as SH

pytestmark = pytest.mark.gpu


class F32Returns:
    """TotalBatchRewardPerEpisode restated in Float32 (the env's FIELD_EPISODE_RETURN accumulator): per step
    ret = Float32(ret + Float32(reward)), pushed on termination."""
    per_step = True

    def __init__(self, n):
        self.rewards = [[] for _ in range(n)]
        self.acc = np.zeros(n, np.float32)

    def push(self, stage, policy, env):
        if stage != "PostActStage":
            return
        self.acc = (self.acc + env.reward().astype(np.float32)).astype(np.float32)
        for i in np.nonzero(env.is_terminated())[0]:
            self.rewards[i].append(float(self.acc[i]))
            self.acc[i] = 0


class SeededActions:
    """host actions from a seeded generator (continuous envs, where RandomPolicy refuses an interval)"""
    fusable = False

    def __init__(self, env, seed):
        self.rng, self.lo, self.hi, self.n, self.dt = np.random.default_rng(seed), *env.action_space(), env.n, env.act_dtype

    def plan(self, env):
        return self.rng.uniform(self.lo, self.hi, self.n).astype(self.dt)

    def push(self, *a, **k):
        pass

    def optimise(self, *a):
        pass


def _host_hooks(pkg, n):
    return pkg.BatchStepsPerEpisode(n), pkg.TotalBatchRewardPerEpisode(n), F32Returns(n)


def _check_lists(log, steps, tot, f32, integer_rewards):
    assert sum(map(len, log.steps)) > 0
    assert log.steps == steps.steps
    assert log.rewards == f32.rewards                       # Float32 bit for bit (both are Python floats of float32 values)
    if integer_rewards:
        assert log.rewards == tot.rewards


K1_CASES = [("CartPole", np.float32, {}), ("CartPole", np.float64, {}), ("Pendulum", np.float32, dict(continuous=False, n_actions=5)),
            ("Pendulum", np.float64, dict(continuous=False, n_actions=3)), ("MountainCar", np.float32, {}), ("MountainCar", np.float64, {}),
            ("Acrobot", np.float64, {}), ("Pendulum", np.float32, dict(continuous=True)), ("Pendulum", np.float64, dict(continuous=True)),
            ("ContinuousCartPole", np.float32, {}), ("ContinuousMountainCar", np.float32, {}), ("ContinuousMountainCar", np.float64, {})]


@pytest.mark.parametrize("kind,T,kw", K1_CASES, ids=[f"{k}-{np.dtype(t).name}-{'c' if kw.get('continuous') else ''}" for k, t, kw in K1_CASES])
@pytest.mark.parametrize("auto_reset", [True, False])
@pytest.mark.parametrize("max_timeout", [0, 29])
@pytest.mark.parametrize("n", [1, 127, 65537])
def test_k1_lists_equal_the_host_hooks(pkg, ctx, kind, T, kw, auto_reset, max_timeout, n):
    if n == 65537 and (kind not in ("CartPole", "Pendulum") or max_timeout == 0 or not auto_reset):
        pytest.skip("the largest batch runs two kinds, the others run at 1 and 127 envs")
    if kind not in ("CartPole", "ContinuousCartPole") and max_timeout == 0:
        max_timeout = 45                        # episodes that end inside the window
    steps, cap = 150, 32
    env = pkg.B200VecEnv(ctx, kind, n, O.splitmix_states_fast(n, 31), T=T, auto_reset=auto_reset, **kw)
    if max_timeout:
        env.set_max_timeout(max_timeout)
    policy = SeededActions(env, 5) if env.continuous else pkg.RandomPolicy()
    log = pkg.DeviceEpisodeLog(n, capacity=cap)
    steps_h, tot_h, f32_h = _host_hooks(pkg, n)
    pkg.run(policy, env, pkg.StopAfterNSteps(steps), steps_h + tot_h + f32_h + log)
    _check_lists(log, steps_h, tot_h, f32_h, integer_rewards=kind not in ("Pendulum",))
    assert log[0] == (log.rewards, log.steps)
    env.close()


def _ppo(pkg, ctx, kind, n, T, seed, algo, **envkw):
    env = pkg.B200VecEnv(ctx, kind, n, O.splitmix_states_fast(n, seed), auto_reset=True, **envkw)
    n_in, cont = {"CartPole": 4, "Pendulum": 3}[kind], env.continuous
    n_out = 1 if cont else len(env.action_space())
    desc = O.ac_desc(n_in, 64, n_out, 0, cont)
    net = pkg.Network(ctx, n_in, 64, n_out, O.glorot_params(desc, 77), act=0, kind=pkg.KIND_GAUSSIAN if cont else pkg.KIND_CATEGORICAL)
    cfg = pkg.onpolicy_config(update_freq=T, n_epochs=2, n_microbatches=2, algo=algo)
    agent = pkg.OnPolicyAgent(ctx, net, env, cfg, O.splitmix_states_fast(n, seed + 1), host_actions=False)
    return env, net, agent


def _ppo_state(pkg, env, net, agent):
    R = pkg.learners
    ck = {k: np.array(v, copy=True) for k, v in pkg.checkpoint.checkpoint(env, net, agent).items()}
    for f in (R.ROLL_ACTION, R.ROLL_LOGP, R.ROLL_REWARD, R.ROLL_TERMINAL, R.ROLL_RNG, R.ROLL_VALUE, R.ROLL_STATE):
        ck[f"rollout/{f}"] = np.array(agent.rollout(f), copy=True)
    return ck


def _same(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        x, y = np.ascontiguousarray(a[k]), np.ascontiguousarray(b[k])
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), k


@pytest.mark.parametrize("kind,envkw,algo", [("CartPole", {}, "ppo"), ("Pendulum", dict(continuous=True), "a2c")])
def test_fused_onpolicy_run_logs_what_the_stage_protocol_sees(pkg, ctx, kind, envkw, algo):
    n, T, cap, iters = 300, 8, 32, 12           # windows of 4 iterations: iterate(4) three times
    out = {}
    for which in ("log", "stats", "stage"):
        env, net, agent = _ppo(pkg, ctx, kind, n, T, 9, algo, **envkw)
        env.set_max_timeout(23)               # (Pendulum episodes would otherwise outlast the run)
        if which == "stage":
            agent.fusable = False
            hooks = _host_hooks(pkg, n)
            pkg.run(agent, env, pkg.StopAfterNSteps(iters * T), hooks[0] + hooks[1] + hooks[2])
            out[which] = hooks
        else:
            hook = pkg.DeviceEpisodeLog(n, capacity=cap) if which == "log" else pkg.DeviceEpisodeStats()
            l0 = ctx.launch_count()
            pkg.run(agent, env, pkg.StopAfterNSteps(iters * T), hook)
            out[which] = dict(hook=hook, launches=ctx.launch_count() - l0, graph=agent.graph_active(),
                              state=_ppo_state(pkg, env, net, agent))
        agent.close(); net.close(); env.close()
    lg, st = out["log"], out["stats"]
    assert lg["graph"] and st["graph"]                                  # the fused path: whole iterations as CUDA graphs
    assert lg["launches"] == st["launches"] + 3 * (iters * T // cap + 1)   # + the three flush kernels per window and at the end
    _same(lg["state"], st["state"])                                     # the log changes nothing the run computes
    _check_lists(lg["hook"], *out["stage"], integer_rewards=kind == "CartPole")


def _dqn(pkg, ctx, seed, lanes, hidden, dueling, n_step, explorer):
    env = pkg.B200VecEnv(ctx, "CartPole", lanes, O.splitmix_states_fast(lanes, seed), auto_reset=True)
    env.set_max_timeout(40)
    kind = pkg.KIND_DUELING if dueling else pkg.KIND_Q
    p = np.random.default_rng(seed).uniform(-0.3, 0.3, pkg.Network.count_params(ctx, 4, hidden, 2, kind=kind)).astype(np.float32)
    net = pkg.Network(ctx, 4, hidden, 2, p, kind=kind)
    traj = pkg.Trajectory(ctx, 4, 16, lanes=lanes, batch_size=128, sampler_rng=O.splitmix_states_fast(128, seed + 2), prioritized=True,
                          n_step=n_step)
    traj.controller = pkg.InsertSampleRatioController(ratio=0.5, threshold=3)
    learner = pkg.DQNLearner(ctx, net, traj, pkg.dqn_config(target_update_freq=4))
    ex = pkg.EpsilonSpeedyExplorer(0.002) if explorer == "speedy" else pkg.EpsilonGreedyExplorer(
        0.05, kind="exp", eps_init=1.0, warmup_steps=lanes, decay_steps=10 * lanes)
    policy = pkg.QBasedPolicy(ctx, learner, ex, O.splitmix_states_fast(lanes, seed + 3), lanes)
    return dict(env=env, net=net, traj=traj, policy=policy, agent=pkg.Agent(policy, traj), learner=learner)


def _dqn_close(s):
    s["agent"].close()
    for k in ("policy", "traj", "net", "env"):
        s[k].close()


@pytest.mark.parametrize("hidden,dueling,n_step,explorer", [(64, True, 3, "speedy"), (128, False, 3, "exp"), (64, False, 1, "exp")])
def test_dqn_replay_loop_logs_what_the_stage_protocol_sees(pkg, ctx, hidden, dueling, n_step, explorer):
    lanes, steps, cap = 127, 100, 24
    out = {}
    for which in ("log", "stats", "stage"):
        s = _dqn(pkg, ctx, 100, lanes, hidden, dueling, n_step, explorer)
        if which == "stage":
            s["agent"].fusable = False
            hooks = _host_hooks(pkg, lanes)
            pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(steps), hooks[0] + hooks[1] + hooks[2])
            out[which] = hooks
        else:
            hook = pkg.DeviceEpisodeLog(lanes, capacity=cap) if which == "log" else pkg.DeviceEpisodeStats()
            pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(steps), hook)
            assert s["agent"]._replay is not None                         # the device loop ran
            ck = {k: np.array(v, copy=True) for k, v in pkg.checkpoint.checkpoint_replay(s["env"], s["net"], s["agent"]).items()}
            c = s["traj"].controller
            out[which] = dict(hook=hook, state=ck, ctl=(c.n_inserted, c.n_sampled), td=s["learner"].last_td())
        _dqn_close(s)
    lg, st = out["log"], out["stats"]
    _same(lg["state"], st["state"])                # env, Q-network, ring + sum tree, streams: windows of `cap` steps change nothing
    assert lg["ctl"] == st["ctl"] and np.array_equal(lg["td"], st["td"])
    _check_lists(lg["hook"], *out["stage"], integer_rewards=True)


class _Meet:
    """a hook that holds a rank at the experiment stages until the other rank gets there"""
    per_step = False

    def __init__(self, barrier):
        self.barrier = barrier

    def __add__(self, other):
        return _compose(self, other)

    def push(self, stage, policy, env):
        if stage in ("PreExperimentStage", "PostExperimentStage"):
            self.barrier.wait(timeout=60)


def _compose(*hooks):
    import __graft_entry__ as g
    core = g.load_package().core
    flat = []
    for h in hooks:
        flat.extend(h.hooks if isinstance(h, core.ComposedHook) else (h,))
    return core.ComposedHook(*flat)


def test_sharded_dqn_logs_global_indices_and_the_union(pkg):
    pairs = [SH._two_ranks(pkg)]
    one = pkg.Context(0)
    n, steps, case = 96, 40, dict(env="CartPole", threshold=1000)       # no update inside the window: each rank's lanes are the union's
    try:
        SH._warm(pkg, one, 2 * n, case)
        ranks = [SH._agent(pkg, c, 2 * n, case, steps=steps) for c in pairs[0]]
        union = SH._agent(pkg, one, 2 * n, case, steps=steps)
        for s in ranks + [union]:
            s["env"].set_max_timeout(15)
        hu = pkg.DeviceEpisodeLog(2 * n, capacity=16)
        pkg.run(union["agent"], union["env"], pkg.StopAfterNSteps(steps), hu)
        hooks = [pkg.DeviceEpisodeLog(n, capacity=16) for _ in ranks]
        # both ranks attach (allocate) before either starts exchanging, and detach (free) only once both have launched every
        # exchange: ranks sharing a device must not allocate or free while a peer's kernel waits for them
        meet = _Meet(threading.Barrier(2))
        SH._prepare(ranks)
        SH._in_threads([lambda s=s, h=h: pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(steps), meet + h + meet)
                        for s, h in zip(ranks, hooks)])
        assert [h._base for h in hooks] == [0, n]                      # records carry rank * N + i
        assert hooks[0].steps + hooks[1].steps == hu.steps and hooks[0].rewards + hooks[1].rewards == hu.rewards
        assert sum(map(len, hu.steps)) >= 2 * n
        # the global index through the ABI: rank 1's records name envs n .. 2n - 1
        env = ranks[1]["env"]
        env.episode_log(8)
        env.act_random_()
        for _ in range(20):
            env.act_random_()
        arr, addr = env.episode_log_buffer(8 * n)
        env.episode_log_flush(addr, 8 * n)
        rec = env.episode_log_read(arr, addr)
        env.ctx.host_free(addr)
        env.episode_log(0)
        assert len(rec) > 0 and rec["env"].min() >= n and rec["env"].max() < 2 * n
        for s in ranks + [union]:
            SH._close(s)
    finally:
        for c in pairs[0]:
            c.close()
        one.close()


def _flush_read(env, cap):
    arr, addr = env.episode_log_buffer(cap)
    try:
        env.episode_log_flush(addr, cap)
        return env.episode_log_read(arr, addr)
    finally:
        env.ctx.host_free(addr)


@pytest.mark.parametrize("hidden", [64, 128])
def test_evaluation_between_two_runs_is_not_logged(pkg, ctx, hidden):
    n = 257
    s = _dqn(pkg, ctx, 7, n, hidden, False, 1, "exp")
    env = s["env"]
    env.episode_log(16)
    for _ in range(10):
        env.act_random_()
    first = _flush_read(env, 16 * n)
    assert len(first) > 0
    ac = pkg.Network(ctx, 4, hidden, 2, O.glorot_params(O.ac_desc(4, hidden, 2), 3), kind=pkg.KIND_CATEGORICAL)
    counts = pkg.evaluate(ac, env, 60, max_episodes=4)["counts"]
    counts_x = pkg.evaluate(s["policy"], env, 60, max_episodes=4)["counts"]
    assert counts.sum() > n and counts_x.sum() > n                    # the evaluations did finish episodes ...
    assert len(_flush_read(env, 16 * n)) == 0                          # ... none of which reached the log
    env.reset_(is_force=True)
    for _ in range(10):
        env.act_random_()
    assert len(_flush_read(env, 16 * n)) > 0                           # and the log still records training steps
    env.episode_log(0)
    ac.close()
    _dqn_close(s)


def test_overflowing_window_is_an_error(pkg, ctx):
    n, K = 300, 4
    env = pkg.B200VecEnv(ctx, "CartPole", n, O.splitmix_states_fast(n, 2), auto_reset=True)
    env.set_max_timeout(3)                        # every env ends an episode every 3 steps
    env.episode_log(K)
    for _ in range(3 * K):
        env.act_random_()
    assert len(_flush_read(env, n * K)) == n * K  # exactly K per env fits
    for _ in range(3 * K + 3):
        env.act_random_()
    with pytest.raises(pkg.B200RLError) as e:
        _flush_read(env, n * K)
    assert e.value.status == pkg._lib.ERR_OVERFLOW and f"{n} of the {n} envs" in str(e.value)
    for _ in range(3):
        env.act_random_()
    assert len(_flush_read(env, n * K)) == n      # the next window starts clean
    env.episode_log(0)
    with pytest.raises(pkg.B200RLError):          # detached: nothing to flush
        _flush_read(env, n * K)
    env.close()


def test_detached_log_leaves_the_run_it_would_have_been(pkg, ctx):
    n, T = 200, 8
    out = []
    for with_log in (True, False):
        env, net, agent = _ppo(pkg, ctx, "CartPole", n, T, 4, "ppo")
        first = pkg.DeviceEpisodeLog(n, capacity=16) if with_log else pkg.DeviceEpisodeStats()
        pkg.run(agent, env, pkg.StopAfterNSteps(4 * T), first)            # the graph is captured with the log's pointers ...
        if with_log:
            first.close()                                                   # ... the log detached ...
        pkg.run(agent, env, pkg.StopAfterNSteps(4 * T), pkg.DeviceEpisodeStats())   # ... and recaptured without them
        assert agent.graph_active()
        out.append(_ppo_state(pkg, env, net, agent))
        agent.close(); net.close(); env.close()
    _same(*out)


def test_hooks_share_an_env_one_at_a_time(pkg, ctx):
    n = 64
    env = pkg.B200VecEnv(ctx, "CartPole", n, O.splitmix_states_fast(n, 6), auto_reset=True)
    env.set_max_timeout(3)                        # every env ends an episode every 3 steps (a pole needs longer to fall)
    a = pkg.DeviceEpisodeLog(n, capacity=16)
    pkg.run(pkg.RandomPolicy(), env, pkg.StopAfterNSteps(40), a)
    bufs = list(a._bufs)
    b = pkg.DeviceEpisodeLog(n, capacity=16)      # a second hook of the same size takes the idle hook's buffers over
    pkg.run(pkg.RandomPolicy(), env, pkg.StopAfterNSteps(40), b)
    assert b._bufs == bufs and a._bufs == []
    assert [len(x) for x in a.steps] == [len(x) for x in b.steps] == [13] * n
    c, d = pkg.DeviceEpisodeLog(n, capacity=16), pkg.DeviceEpisodeLog(n, capacity=16)
    with pytest.raises(RuntimeError):             # two hooks recording one env in the same run
        pkg.run(pkg.RandomPolicy(), env, pkg.StopAfterNSteps(5), c + d)
    c.close()
    e = pkg.DeviceEpisodeLog(n, capacity=2)       # an overflowing window ends the hook's recording ...
    e.push("PreExperimentStage", None, env)
    for _ in range(30):
        env.act_random_()
    e.flush()
    with pytest.raises(pkg.B200RLError):
        e.flush()
    f = pkg.DeviceEpisodeLog(n, capacity=16)      # ... so that another hook can record the env
    pkg.run(pkg.RandomPolicy(), env, pkg.StopAfterNSteps(20), f)
    assert [len(x) for x in f.steps] == [6] * n
    for h in (a, b, e, f):
        h.close()
    env.close()
