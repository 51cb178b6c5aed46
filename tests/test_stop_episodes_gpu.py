"""GPU tests of StopAfterNEpisodes on the fused PPO / A2C and DQN loops (b200rl_onpolicy_run_episodes, b200rl_replay_run_episodes).

Every case runs two twins built from the same seeds: one through the stage loop (a per-step hook forces it; it also records the
per-step episode counts and the BatchStepsPerEpisode lists), one through the fused path (DeviceEpisodeLog or EmptyHook).  Both
must stop after the same step with the same stop_condition.cur and leave the same state bit for bit: every env field, the rollout
columns, fill level and policy streams, parameters, Adam moments and step; for DQN the ring with its sum tree and sampler streams,
the target, the explorer streams and step and the controller counters.  The budget k is chosen from a probe twin's own per-step
counts, so that the stop lands on the first step, inside a rollout, on a rollout's last step, several rollouts in, inside a log
window or on its boundary, between two updates and on a target-sync update."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
import test_episode_log_gpu as EL
import test_replay_sharded_gpu as SH

pytestmark = pytest.mark.gpu


class StepCounts:
    """per-step episode counts (lanes terminal after each step) of a stage-loop run; per_step forces the stage loop"""
    per_step = True

    def __init__(self):
        self.counts = []

    def push(self, stage, policy, env):
        if stage == "PostActStage":
            self.counts.append(int(np.count_nonzero(env.is_terminated())))


def budget_for(counts, target, exact=True, where=lambda s: True):
    """k (from cur = 0) whose first crossing is at step s* = the first step >= target with a count for which where(s*) holds, and
    s*.  Fails when the probe has no such step (the case would not land where its name says)."""
    c = np.asarray(counts, np.int64)
    j = target - 1
    while j < len(c) and (c[j] == 0 or not where(j + 1)):
        j += 1
    assert j < len(c), "no step of the probe satisfies the case"
    csum = np.cumsum(c)
    if exact or c[j] < 2:
        return int(csum[j]), j + 1
    return int(csum[j]) - 1, j + 1       # the crossing overshoots k by one


# ---- on-policy ----------------------------------------------------------------------------------------------------------------
N_ON, T_ON = 96, 8
ON_CONFIGS = {
    "ppo-cartpole": dict(kind="CartPole", algo="ppo", envkw={}, timeout=0, f64=False),
    "a2c-pendulum": dict(kind="Pendulum", algo="a2c", envkw=dict(continuous=True), timeout=10, f64=False),   # ends at 10, 20, 30, ...
    "ppo-cartpole-f64": dict(kind="CartPole", algo="ppo", envkw=dict(T=np.float64), timeout=0, f64=True),   # Float64 behind set_state_float32
    "ppo-cartpole-timeout": dict(kind="CartPole", algo="ppo", envkw={}, timeout=6, f64=False),
}


def _onpolicy(pkg, ctx, cfg, n=N_ON, seed=21):
    env = pkg.B200VecEnv(ctx, cfg["kind"], n, O.splitmix_states_fast(n, seed), auto_reset=True, **cfg["envkw"])
    if cfg["f64"]:
        env.set_state_float32()
    if cfg["timeout"]:
        env.set_max_timeout(cfg["timeout"])
    n_in, cont = {"CartPole": 4, "Pendulum": 3}[cfg["kind"]], env.continuous
    n_out = 1 if cont else len(env.action_space())
    desc = O.ac_desc(n_in, 64, n_out, 0, cont)
    net = pkg.Network(ctx, n_in, 64, n_out, O.glorot_params(desc, 77), act=0, kind=pkg.KIND_GAUSSIAN if cont else pkg.KIND_CATEGORICAL)
    ocfg = pkg.onpolicy_config(update_freq=T_ON, n_epochs=2, n_microbatches=2, algo=cfg["algo"])
    agent = pkg.OnPolicyAgent(ctx, net, env, ocfg, O.splitmix_states_fast(n, seed + 1), host_actions=False)
    # the rollout columns a run has not written yet hold whatever the allocation held: zero them, so that the twins compare equal there
    for f in range(6):
        z = np.zeros_like(agent.rollout(f))
        pkg._lib.check(agent.lib.b200rl_onpolicy_set(agent.h, f, pkg._lib.ptr(z), z.nbytes))
    return env, net, agent


def _on_state(pkg, env, net, agent):
    st = EL._ppo_state(pkg, env, net, agent)
    st["fill"] = np.array(agent.fill(), np.int64)
    st["step"] = np.array([net.step_count()], np.int64)
    return st


def _on_run(pkg, ctx, cfg, warm, k, fused, hook_kind="log", cur=0, again=None, n=N_ON):
    """warm steps (StopAfterNSteps, fused), then StopAfterNEpisodes(k, cur) [then StopAfterNEpisodes(again)]"""
    env, net, agent = _onpolicy(pkg, ctx, cfg, n=n)
    if warm:
        pkg.run(agent, env, pkg.StopAfterNSteps(warm), pkg.EmptyHook())
    outs = []
    for kk, cc in [(k, cur)] + ([(again, 0)] if again is not None else []):
        stop = pkg.StopAfterNEpisodes(kk, cc)
        steps_before = env.episode_stats()["env_steps"] / n
        if fused:
            agent.fusable = True
            hook = pkg.DeviceEpisodeLog(n, capacity=20) if hook_kind == "log" else pkg.EmptyHook()
            pkg.run(agent, env, stop, hook)
            lists = hook.steps if hook_kind == "log" else None
        else:
            agent.fusable = False
            counts, lengths = StepCounts(), pkg.BatchStepsPerEpisode(n)
            pkg.run(agent, env, stop, pkg.core.ComposedHook(counts, lengths))
            lists = lengths.steps
        outs.append(dict(steps=round(env.episode_stats()["env_steps"] / n - steps_before), cur=stop.cur, lists=lists,
                         state=_on_state(pkg, env, net, agent), graph=agent.graph_active()))
    agent.close(); net.close(); env.close()
    return outs


def _on_probe(pkg, ctx, cfg, warm, steps, n=N_ON):
    env, net, agent = _onpolicy(pkg, ctx, cfg, n=n)
    if warm:
        pkg.run(agent, env, pkg.StopAfterNSteps(warm), pkg.EmptyHook())
    agent.fusable = False
    counts = StepCounts()
    pkg.run(agent, env, pkg.StopAfterNSteps(steps), counts)
    agent.close(); net.close(); env.close()
    return counts.counts


def _on_compare(pkg, ctx, cfg, warm, k, cur=0, again=None, hook_kind="log", n=N_ON):
    a = _on_run(pkg, ctx, cfg, warm, k, False, cur=cur, again=again, n=n)
    b = _on_run(pkg, ctx, cfg, warm, k, True, hook_kind=hook_kind, cur=cur, again=again, n=n)
    for x, y in zip(a, b):
        assert (x["steps"], x["cur"]) == (y["steps"], y["cur"])
        EL._same(x["state"], y["state"])
        if y["lists"] is not None:
            assert x["lists"] == y["lists"]
    return b


# (warm steps, target step, exact hit, where s* must land given t0 = warm % T) — T = 8: warm 0 enters with an empty rollout, warm 14
# with 6 of 8 columns (run() force-resets the env, so the fixed-length episodes restart with it).  DeviceEpisodeLog(capacity = 20) windows start with the run.
CAP = 20
ON_CASES = {
    "inside-rollout": (0, 3, True, lambda s, t0: (t0 + s) % T_ON != 0),
    "rollout-last-step": (0, 8, True, lambda s, t0: (t0 + s) % T_ON == 0),      # the update of the rollout must run
    "several-rollouts": (0, 27, False, lambda s, t0: (t0 + s) % T_ON != 0),
    "part-filled-inside": (14, 1, False, lambda s, t0: (t0 + s) % T_ON != 0),
    "part-filled-last-step": (14, 2, True, lambda s, t0: (t0 + s) % T_ON == 0),
    "log-window-boundary": (0, CAP, True, lambda s, t0: s % CAP == 0),
    "log-window-inside": (0, CAP + 1, True, lambda s, t0: s % CAP != 0),
}


@pytest.mark.parametrize("config", sorted(ON_CONFIGS))
@pytest.mark.parametrize("case", sorted(ON_CASES))
def test_onpolicy_stops_where_the_stage_loop_stops(pkg, ctx, config, case):
    cfg = ON_CONFIGS[config]
    warm, target, exact, where = ON_CASES[case]
    t0 = warm % T_ON
    counts = _on_probe(pkg, ctx, cfg, warm, 90)
    k, s_star = budget_for(counts, target, exact, where=lambda s: where(s, t0))
    res = _on_compare(pkg, ctx, cfg, warm, k)[0]
    assert res["steps"] == s_star and where(s_star, t0) and res["cur"] >= k
    assert res["state"]["fill"][0] == (t0 + s_star) % T_ON   # a rollout completed by s* was updated, one s* falls inside stays part-filled


@pytest.mark.parametrize("config", ["ppo-cartpole-timeout", "a2c-pendulum"])     # episodes of at most 6 / exactly 10 steps
@pytest.mark.parametrize("last_step", [False, True])
def test_onpolicy_long_run_through_unmarked_rollouts(pkg, ctx, config, last_step):
    """k - cur >> N T: many whole rollouts run unmarked (b200rl_onpolicy_iterate, no shadow) before the stretch that crosses; the
    crossing lands inside a rollout or on the last step of one"""
    cfg, n = ON_CONFIGS[config], 8
    counts = _on_probe(pkg, ctx, cfg, 0, 900, n=n)
    k, s_star = budget_for(counts, 800, exact=not last_step, where=lambda s: (s % T_ON == 0) == last_step)
    assert k > 8 * n * T_ON                                  # the rollouts stay unmarked until fewer than N T episodes remain
    for hook_kind in ("empty", "log"):
        res = _on_compare(pkg, ctx, cfg, 0, k, hook_kind=hook_kind, n=n)[0]
        assert res["steps"] == s_star and res["graph"]       # whole rollouts ran as the captured iterate graph
        assert res["state"]["fill"][0] == s_star % T_ON


@pytest.mark.parametrize("config", ["ppo-cartpole", "a2c-pendulum"])
def test_onpolicy_first_step_and_spent_budget(pkg, ctx, config):
    cfg = ON_CONFIGS[config]
    counts = _on_probe(pkg, ctx, cfg, 13, 4)
    if counts[0] > 0:
        (res,) = _on_compare(pkg, ctx, cfg, 13, counts[0])                   # the first step reaches the budget
        assert res["steps"] == 1
    (res,) = _on_compare(pkg, ctx, cfg, 13, 5, cur=5)                          # cur >= k on entry: exactly one step
    assert res["steps"] == 1
    (res,) = _on_compare(pkg, ctx, cfg, 13, 5, cur=9, hook_kind="empty")
    assert res["steps"] == 1


@pytest.mark.parametrize("config", ["ppo-cartpole", "ppo-cartpole-timeout"])
def test_onpolicy_second_run_continues(pkg, ctx, config):
    cfg = ON_CONFIGS[config]
    counts = _on_probe(pkg, ctx, cfg, 0, 40)
    k, _ = budget_for(counts, 5, exact=False)
    k2, _ = budget_for(counts[5:], 11, exact=True)
    for hook_kind in ("log", "empty"):
        a, b = _on_compare(pkg, ctx, cfg, 0, k, again=k2, hook_kind=hook_kind)
        assert a["steps"] >= 5 and b["steps"] >= 1


# ---- DQN ----------------------------------------------------------------------------------------------------------------------
LANES = 64


def _dqn(pkg, ctx, explorer, ratio=0.25, target_update_freq=3, lanes=LANES):
    s = EL._dqn(pkg, ctx, 300, lanes, 64, True, 3, "exp")      # (MaxTimeoutEnv 40; 6 for a few lanes: short episodes, large k)
    if lanes < LANES:
        s["env"].set_max_timeout(6)
    if explorer == "gumbel":
        s["policy"].explorer = pkg.GumbelSoftmaxExplorer()
    s["traj"].controller = pkg.InsertSampleRatioController(ratio=ratio, threshold=3)
    s["learner"].cfg = pkg.dqn_config(target_update_freq=target_update_freq)
    return s


def _dqn_state(pkg, s):
    st = {k: np.array(v, copy=True) for k, v in pkg.checkpoint.checkpoint_replay(s["env"], s["net"], s["agent"]).items()}
    c = s["traj"].controller
    st["ctl"] = np.array([c.n_inserted, c.n_sampled], np.int64)
    st["total_priority"] = np.array([s["traj"].total_priority()], np.float32)
    return st


def _dqn_run(pkg, ctx, explorer, warm, k, fused, again=None, hook_kind="log", lanes=LANES):
    s = _dqn(pkg, ctx, explorer, lanes=lanes)
    if warm:
        pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(warm), pkg.EmptyHook())
    outs = []
    for kk in [k] + ([again] if again is not None else []):
        stop = pkg.StopAfterNEpisodes(kk)
        steps_before = s["env"].episode_stats()["env_steps"] / lanes
        if fused:
            s["agent"].fusable = True
            hook = pkg.DeviceEpisodeLog(lanes, capacity=7) if hook_kind == "log" else pkg.EmptyHook()
            pkg.run(s["agent"], s["env"], stop, hook)
            assert s["agent"]._replay is not None
            lists = hook.steps if hook_kind == "log" else None
        else:
            s["agent"].fusable = False
            counts, lengths = StepCounts(), pkg.BatchStepsPerEpisode(lanes)
            pkg.run(s["agent"], s["env"], stop, pkg.core.ComposedHook(counts, lengths))
            lists = lengths.steps
        outs.append(dict(steps=round(s["env"].episode_stats()["env_steps"] / lanes - steps_before), cur=stop.cur, lists=lists,
                         state=_dqn_state(pkg, s)))
    EL._dqn_close(s)
    return outs


def _dqn_probe(pkg, ctx, explorer, warm, steps, lanes=LANES):
    s = _dqn(pkg, ctx, explorer, lanes=lanes)
    if warm:
        pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(warm), pkg.EmptyHook())
    s["agent"].fusable = False
    counts = StepCounts()
    pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(steps), counts)
    EL._dqn_close(s)
    return counts.counts


# (warm steps, target step, exact, where global step g = warm + s* must land).  Ratio 0.25, threshold 3: the updates run after global
# steps 3, 7, 11, ... and every third of them (after 11, 23, 35, ...) syncs the target.  The ring holds 16 frames per lane, so chunks
# are 8 steps; DeviceEpisodeLog(capacity = 7) windows cut them further.
DQN_CASES = {
    "first-chunk": (0, 2, True, lambda g: True),
    "between-updates": (20, 2, False, lambda g: (g - 3) % 4 != 0),
    "on-update": (20, 4, True, lambda g: (g - 3) % 4 == 0),
    "several-chunks": (20, 29, True, lambda g: True),
    "target-sync-update": (0, 12, True, lambda g: (g - 3) % 12 == 8),
}


@pytest.mark.parametrize("explorer", ["exp", "gumbel"])
@pytest.mark.parametrize("case", sorted(DQN_CASES))
def test_dqn_stops_where_the_stage_loop_stops(pkg, ctx, explorer, case):
    warm, target, exact, where = DQN_CASES[case]
    counts = _dqn_probe(pkg, ctx, explorer, warm, 90)
    k, s_star = budget_for(counts, target, exact, where=lambda s: where(warm + s))
    a = _dqn_run(pkg, ctx, explorer, warm, k, False)[0]
    b = _dqn_run(pkg, ctx, explorer, warm, k, True)[0]
    assert (a["steps"], a["cur"]) == (b["steps"], b["cur"]) == (s_star, a["cur"]) and a["cur"] >= k and where(warm + s_star)
    EL._same(a["state"], b["state"])
    assert a["lists"] == b["lists"]


@pytest.mark.parametrize("explorer", ["exp", "gumbel"])
def test_dqn_long_run_through_unmarked_chunks(pkg, ctx, explorer):
    """k - cur >> N · chunk: many chunks run unmarked (no shadow) before the one that crosses"""
    lanes = 8
    counts = _dqn_probe(pkg, ctx, explorer, 0, 500, lanes=lanes)
    k, s_star = budget_for(counts, 400, exact=False)
    assert k > 4 * lanes * 8                                 # the chunks stay unmarked until fewer than N · 8 episodes remain
    for hook_kind in ("empty", "log"):
        a = _dqn_run(pkg, ctx, explorer, 0, k, False, lanes=lanes)[0]
        b = _dqn_run(pkg, ctx, explorer, 0, k, True, hook_kind=hook_kind, lanes=lanes)[0]
        assert (a["steps"], a["cur"]) == (b["steps"], b["cur"]) and a["steps"] == s_star
        EL._same(a["state"], b["state"])


def test_dqn_spent_budget_and_second_run(pkg, ctx):
    counts = _dqn_probe(pkg, ctx, "exp", 10, 40)
    k, _ = budget_for(counts, 3, exact=False)
    k2, _ = budget_for(counts[3:], 13, exact=True)
    for hook_kind in ("log", "empty"):
        outs_a = _dqn_run(pkg, ctx, "exp", 10, k, False, again=k2)
        outs_b = _dqn_run(pkg, ctx, "exp", 10, k, True, again=k2, hook_kind=hook_kind)
        for a, b in zip(outs_a, outs_b):
            assert (a["steps"], a["cur"]) == (b["steps"], b["cur"])
            EL._same(a["state"], b["state"])
    a = _dqn_run(pkg, ctx, "exp", 10, 0, False)[0]
    b = _dqn_run(pkg, ctx, "exp", 10, 0, True)[0]
    assert a["steps"] == b["steps"] == 1
    EL._same(a["state"], b["state"])


# ---- sharded ctx --------------------------------------------------------------------------------------------------------------
def test_sharded_ctx_is_refused_with_nothing_touched(pkg):
    L = pkg._lib
    ctxs = SH._two_ranks(pkg)
    try:
        ctx = ctxs[0]
        env, net, agent = EL._ppo(pkg, ctx, "CartPole", 32, 8, 3, "ppo")
        before = _on_state(pkg, env, net, agent)
        steps, eps = C.c_int64(-1), C.c_int64(-1)
        st = ctx.lib.b200rl_onpolicy_run_episodes(agent.h, 100, 10, None, C.byref(steps), C.byref(eps))
        assert st == L.ERR_UNSUPPORTED and (steps.value, eps.value) == (-1, -1)
        EL._same(before, _on_state(pkg, env, net, agent))
        agent.close(); net.close(); env.close()

        s = EL._dqn(pkg, ctx, 5, 32, 64, False, 1, "exp")
        h = s["agent"]._handle(s["env"])
        assert h is not None
        before = _dqn_state(pkg, s)
        ex = s["policy"].explorer.as_struct()
        c = s["traj"].controller
        ctl = L.InsertSampleRatio(c.ratio, c.threshold, c.n_inserted, c.n_sampled)
        st = ctx.lib.b200rl_replay_run_episodes(h, C.c_void_p(s["policy"]._d_rng), C.byref(ex), C.byref(ctl), 100, 10, None,
                                                C.byref(steps), C.byref(eps))
        assert st == L.ERR_UNSUPPORTED and (steps.value, eps.value) == (-1, -1)
        assert (ctl.n_inserted, ctl.n_sampled, ex.step) == (c.n_inserted, c.n_sampled, s["policy"].explorer.step)
        EL._same(before, _dqn_state(pkg, s))
        EL._dqn_close(s)
    finally:
        for c in ctxs:
            c.close()
