"""Host logic of the drop-in surface (no GPU): the run loop / stages / hooks / stop conditions mirror
(reinforcementlearning.jl_b200/core.py), the explorer schedule mirror (explorers.py) and the trajectory controller,
driven with a stub batched env.  Expected values are the reference's own test vectors:
RLCore/test/core/stop_conditions.jl:3-50, test/core/hooks.jl:44-152,
test/policies/explorers/epsilon_greedy_explorer.jl:8-74."""
import json
import os

import numpy as np
import pytest

import oracle_lib as O

with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "control_reference_vectors.json")) as _f:
    GOLD = json.load(_f)


def make_stop(pkg, spec):
    name, *args = spec
    if name in ("StopIfAny", "StopIfAll"):
        return getattr(pkg, name)(*[make_stop(pkg, a) for a in args])
    return getattr(pkg, name)(*args)


class StubVecEnv:
    """N counters: sub-env i terminates every period[i] steps; auto_reset like the fused step kernel."""

    def __init__(self, periods, auto_reset=True):
        self.periods = np.asarray(periods, np.int64)
        self.n = len(self.periods)
        self.auto_reset = auto_reset
        self.t = np.zeros(self.n, np.int64)
        self.term = np.zeros(self.n, bool)
        self.log = []

    def reset_(self, is_force=True):
        self.log.append(("reset", bool(is_force)))
        if is_force:
            self.t[:] = 0
            self.term[:] = False
        else:
            self.t[self.term] = 0
            self.term[:] = False

    def act_random_(self):
        self.log.append(("act_random",))
        self._step()

    def act_(self, actions):
        self.log.append(("act", np.array(actions).copy()))
        self._step()

    def _step(self):
        self.t += 1
        self.term = self.t >= self.periods
        if self.auto_reset:
            self.t[self.term] = 0

    def is_terminated(self):
        return self.term.copy()

    def reward(self):
        return np.where(self.term, 0.0, 1.0)

    def check(self):
        self.log.append(("check",))

    def episode_stats(self, reset=False):
        return {"episodes": 0, "return_sum": 0.0, "length_sum": 0.0, "env_steps": 0}


@pytest.mark.parametrize("case", [c for c in GOLD["stop_conditions"] if "trues" in c], ids=lambda c: c["ref"])
def test_stop_condition_counts_golden(pkg, case):
    s = make_stop(pkg, case["condition"])
    assert sum(s.check(None, None) for _ in range(case["calls"])) == case["trues"]


def test_stop_after_n_episodes_batched(pkg):
    env = StubVecEnv([2, 3])
    s = pkg.StopAfterNEpisodes(2)
    env._step()
    assert s.check(None, env) is False                                  # nobody finished
    env._step()
    assert s.check(None, env) is False                                  # env 0 finished: 1 episode
    env._step()
    assert s.check(None, env) is True                                   # env 1 finished: 2 episodes


def test_stop_after_no_improvement(pkg):
    env = StubVecEnv([1])
    s = pkg.StopAfterNoImprovement(lambda: 1.0, 10)
    idle = StubVecEnv([100])
    idle._step()
    assert sum(s.check(None, idle) for _ in range(11)) == 0             # no finished episode: never evaluated
    env._step()
    assert sum(s.check(None, env) for _ in range(11)) == 1              # constant metric: patience runs out once
    vals = iter(range(1, 100))
    s2 = pkg.StopAfterNoImprovement(lambda: float(next(vals)), 10)
    assert sum(s2.check(None, env) for _ in range(11)) == 0             # improving metric never stops


def test_stop_signal(pkg):
    s = pkg.StopSignal()
    assert s.check(None, None) is False
    s.is_stop = True
    assert s.check(None, None) is True


def test_hook_composition_flattens(pkg):
    class Mock(pkg.AbstractHook):
        pass
    a, b, c, d = Mock(), Mock(), Mock(), Mock()
    assert (a + b).hooks == (a, b)
    assert (pkg.ComposedHook(a) + b).hooks == (a, b)
    assert (a + pkg.ComposedHook(b)).hooks == (a, b)
    assert (pkg.ComposedHook(a, b) + pkg.ComposedHook(c, d)).hooks == (a, b, c, d)
    assert (a + b)[1] is b
    (a + b).push("PreActStage", None, None)                              # default push is a no-op


def test_do_every_n_steps_and_do_on_exit(pkg):
    for n in (1, 2):
        calls = []
        h = pkg.DoEveryNSteps(lambda t, agent, env: calls.append(t), n=n)
        for t in range(1, 5):
            h.push("PostActStage", None, None)
            assert len(calls) == t // n                                   # hooks.jl test: env.pos == 1 + div(t, n)
        for stage in ("PreActStage", "PreExperimentStage", "PostExperimentStage"):
            h.push(stage, None, None)
        assert len(calls) == 4 // n
    seen = []
    pkg.DoOnExit(lambda agent, env: seen.append(1)).push("PostExperimentStage", None, None)
    assert seen == [1]


def test_batch_steps_and_rewards_per_episode(pkg):
    env = StubVecEnv([2, 3])
    steps, rewards = pkg.BatchStepsPerEpisode(2), pkg.TotalBatchRewardPerEpisode(2)
    for _ in range(6):
        env._step()
        steps.push("PostActStage", None, env)
        rewards.push("PostActStage", None, env)
    assert steps[()] == [[2, 2, 2], [3, 3]]
    assert rewards.rewards == [[1.0, 1.0, 1.0], [2.0, 2.0]]              # the terminating step pays 0


def test_run_loop_order_and_step_count(pkg):
    """run.jl:36-78 with the MultiThreadEnv control flow: forced reset, then per iteration
    PreAct -> plan! -> act! -> PostAct -> check!; StopAfterNSteps(n) => exactly n act! calls."""
    env = StubVecEnv([3, 5], auto_reset=False)
    stages = []

    class Rec(pkg.AbstractHook):
        def push(self, stage, policy, env):
            stages.append(stage)

    class Pol(pkg.AbstractPolicy):
        def __init__(self):
            self.events = []

        def plan(self, env):
            self.events.append("plan")
            return np.array([1, 2])

        def push(self, stage, env, action=None):
            self.events.append(("push", stage))

        def optimise(self, stage):
            self.events.append(("optimise", stage))

    pol = Pol()
    pkg.run(pol, env, pkg.StopAfterNSteps(4), Rec())
    acts = [e for e in env.log if e[0] == "act"]
    assert len(acts) == 4 and all(np.array_equal(a[1], [1, 2]) for a in acts)
    assert env.log[0] == ("reset", True)                                 # run.jl:46
    assert [e for e in env.log if e[0] == "reset"][1:] == [("reset", False)] * 4   # soft reset at the top of every iteration
    assert env.log[-1] == ("check",)
    assert stages == ["PreExperimentStage"] + ["PreActStage", "PostActStage"] * 4 + ["PostExperimentStage"]
    per_iter = [("push", "PreActStage"), ("optimise", "PreActStage"), "plan", ("push", "PostActStage"), ("optimise", "PostActStage")]
    # run.jl:46-49: the forced reset is followed by the PreEpisodeStage push (every lane starts an episode)
    assert pol.events == [("push", "PreExperimentStage"), ("push", "PreEpisodeStage")] + per_iter * 4 + [("push", "PostExperimentStage")]


def test_run_random_policy_is_fused_into_the_step(pkg):
    env = StubVecEnv([4, 4])
    hook = pkg.run(pkg.RandomPolicy(), env, pkg.StopAfterNEpisodes(4), pkg.BatchStepsPerEpisode(2))
    assert [e[0] for e in env.log].count("act_random") == 8             # 2 envs x 2 episodes of 4 steps each
    assert hook[()] == [[4, 4], [4, 4]]


# ---- explorers ---------------------------------------------------------------------------------
KW = dict(eps_init=0.9, warmup_steps=100, decay_steps=100)


@pytest.mark.parametrize("case", GOLD["explorer_schedule"], ids=lambda c: c["ref"])
def test_epsilon_schedule_golden(pkg, case):
    e = GOLD["explorer"]
    mine = pkg.EpsilonGreedyExplorer(e["eps_stable"], kind=case["kind"], eps_init=e["eps_init"], warmup_steps=e["warmup_steps"],
                                     decay_steps=e["decay_steps"])
    ex6 = O.explorer6(e["eps_stable"], e["eps_init"], e["warmup_steps"], e["decay_steps"], case["kind"])
    for got in (mine.get_eps(case["step"]), O.get_eps(ex6, case["step"])):
        if "atol" in case:
            assert got == pytest.approx(case["expected"], abs=case["atol"])
        else:
            assert got == pytest.approx(case["expected"], rel=1.5e-8)        # Julia's isapprox default
    assert pkg.EpsilonGreedyExplorer(0.3).get_eps() == 0.3                   # EpsilonGreedyExplorer(ϵ): no warm-up, no decay


def test_epsilon_schedule_host_mirror_equals_oracle_bitwise(pkg):
    for kind in ("linear", "exp"):
        mine = pkg.EpsilonGreedyExplorer(0.05, kind=kind, eps_init=0.95, warmup_steps=37, decay_steps=1234)
        ex6 = O.explorer6(0.05, 0.95, 37, 1234, kind)
        steps = list(range(1, 60)) + list(range(900, 1400, 7))
        assert [mine.get_eps(s) for s in steps] == [O.get_eps(ex6, s) for s in steps]


@pytest.mark.parametrize("case", GOLD["explorer_prob"], ids=lambda c: c["ref"])
def test_explorer_prob_golden(pkg, case):
    e = GOLD["explorer"]
    mine = pkg.EpsilonGreedyExplorer(e["eps_stable"], kind="linear", eps_init=e["eps_init"], warmup_steps=e["warmup_steps"],
                                     decay_steps=e["decay_steps"], is_break_tie=case["is_break_tie"])
    ex6 = O.explorer6(e["eps_stable"], e["eps_init"], e["warmup_steps"], e["decay_steps"], "linear", case["is_break_tie"])
    full = O.egreedy_prob(ex6, 1, case["values"])
    if "action" in case:
        assert mine.prob(case["values"], case["action"]) == pytest.approx(case["expected"], rel=1.5e-8)
        assert full[case["action"] - 1] == pytest.approx(case["expected"], rel=1.5e-8)
    else:
        assert mine.prob(case["values"]) == pytest.approx(case["expected"], rel=1.5e-8)
        assert list(full) == pytest.approx(case["expected"], rel=1.5e-8)


def test_greedy_explorer_golden(pkg):
    g = pkg.GreedyExplorer()
    for case in GOLD["greedy"]:
        if "plan" in case:
            assert g.plan_values(case["values"]) == case["plan"]
        elif "action" in case:
            assert g.prob(case["values"], case["action"]) == case["prob"]
        else:
            assert g.prob(case["values"]) == case["prob"]


def test_oracle_egreedy_plan_visits_all_actions_and_follows_prob():
    """epsilon_greedy_explorer.jl test: 300 plans at eps 0.9 visit all 4 actions (both tie modes); the empirical
    frequencies follow prob()."""
    values = np.array([0.1, 0.5, 0.5, 0.3], np.float32)
    n = 40000
    qv = np.repeat(values[:, None], n, axis=1)
    for brk in (True, False):
        ex6 = O.explorer6(0.1, 0.9, 10 ** 9, 100, "linear", brk)          # long warm-up: eps stays 0.9
        rng = O.splitmix_states_fast(n, 77)
        a = O.egreedy_plan(ex6, 1, qv, rng)
        assert set(np.unique(a[:300])) == {1, 2, 3, 4}
        freq = np.bincount(a, minlength=5)[1:] / n
        np.testing.assert_allclose(freq, O.egreedy_prob(ex6, 1, values), atol=0.01)
    # eps = 0: greedy, but one uniform is still drawn per column (the reference always calls rand(s.rng))
    rng = O.splitmix_states_fast(8, 5)
    before = rng.copy()
    a = O.egreedy_plan(O.explorer6(0.0, 0.0), 1, qv[:, :8], rng)
    assert np.all(a == 2) and not np.array_equal(rng, before)


def test_batch_explorer_advances_the_step_per_column(pkg):
    """batch_explorer.jl:15-21: column i of one batched plan! sees get_eps(step + i)."""
    n = 5000
    ex6 = O.explorer6(0.0, 1.0, 0, n, "linear")                          # eps falls from 1 to 0 across ONE batch
    qv = np.repeat(np.array([[0.0], [1.0]], np.float32), n, axis=1)
    a = O.egreedy_plan(ex6, 1, qv, O.splitmix_states_fast(n, 3))
    greedy = a == 2
    assert greedy[: n // 10].mean() < 0.62 and greedy[-n // 10:].mean() > 0.95
    ex = pkg.EpsilonGreedyExplorer(0.0, kind="linear", eps_init=1.0, warmup_steps=0, decay_steps=n)
    ex.advance(n)
    assert ex.step == n + 1 and ex.get_eps() == 0.0
    st = pkg.EpsilonGreedyExplorer(0.1, kind="exp", eps_init=0.9, warmup_steps=3, decay_steps=7, step=11, is_break_tie=True).as_struct()
    assert (st.eps_stable, st.eps_init, st.warmup_steps, st.decay_steps, st.step, st.kind, st.is_break_tie) == (0.1, 0.9, 3, 7, 11, 1, 1)


def test_insert_sample_ratio_controller(pkg):
    c = pkg.InsertSampleRatioController(ratio=0.5, threshold=4)
    sampled = []
    for _ in range(12):
        c.on_insert()
        k = 0
        while c.on_sample():
            k += 1
        sampled.append(k)
    assert sampled[:3] == [0, 0, 0] and sum(sampled) == c.n_sampled
    assert c.n_sampled == int((c.n_inserted - c.threshold) * c.ratio) + 1   # one batch per two insertions after the threshold


def test_returns_on_empty_inputs_follow_the_reference_shape_rules(pkg):
    """basic.jl:227-235, 253-263, 408-417: with no time steps the loops never run — empty outputs of the promoted eltype, the reduced
    form returns `init` (zero when absent).  No device call is made (ctx is None here)."""
    g32 = np.float32(0.5)
    out = pkg.discount_rewards(None, np.zeros(0, np.float32), g32)
    assert out.shape == (0,) and out.dtype == np.float32
    assert pkg.discount_rewards(None, np.zeros(0, np.int64), 0.5).dtype == np.float64          # promote_type(Int, Float64)
    assert pkg.discount_rewards(None, np.zeros((3, 0), np.float32), g32, dims=2).shape == (3, 0)
    assert pkg.discount_rewards_reduced(None, np.zeros(0, np.float32), g32) == 0.0
    assert pkg.discount_rewards_reduced(None, np.zeros(0, np.float32), g32, init=4.0) == 4.0
    red = pkg.discount_rewards_reduced(None, np.zeros((3, 0), np.float32), g32, dims=2, init=np.array([-2.0, 0.0, 2.0], np.float32))
    assert red.tolist() == [-2.0, 0.0, 2.0]
    adv = pkg.generalized_advantage_estimation(None, np.zeros(0, np.float32), np.zeros(1, np.float32), g32, np.float32(0.3))
    assert adv.shape == (0,) and adv.dtype == np.float32
    with pytest.raises(TypeError):
        pkg.generalized_advantage_estimation(None, np.zeros(0, np.float32), np.zeros(1, np.float32), g32, 0.3)   # gamma / lambda types differ
    with pytest.raises(TypeError):
        pkg.discount_rewards(None, np.zeros((2, 2), np.float32), g32)                                            # 2-d rewards need dims


def test_julia_integer_seeding_helper(pkg):
    """sharding.julia_xoshiro_states == the oracle's restatement; first Float64 of Xoshiro(1234) is the value Julia's manual prints."""
    st = pkg.sharding.julia_xoshiro_states([1234, 123, 3, 2 ** 40 + 5])
    assert st.shape == (4, 4) and st.dtype == np.uint64
    for row, seed in zip(st, (1234, 123, 3, 2 ** 40 + 5)):
        assert np.array_equal(row, O.julia_xoshiro(seed))
    s = st[0].copy()
    assert (int(O.lib().orc_rng_next(O._p(s))) >> 11) * 2.0 ** -53 == 0.32597672886359486
    with pytest.raises(ValueError):
        pkg.sharding.julia_xoshiro_states([-1])


def test_debug_timer_mirrors_the_reference_labels(pkg):
    """test/core/base.jl:41-58: after enable_debug_timings the run loop fills the global timer with the labels of run.jl:46-72; off by
    default (and then nothing is recorded)."""
    core = pkg.core
    core.timer.clear()
    pkg.run(pkg.RandomPolicy(), StubVecEnv([3, 4]), pkg.StopAfterNSteps(10))
    assert core.timer == {}
    core.enable_debug_timings()
    try:
        pkg.run(pkg.RandomPolicy(), StubVecEnv([3, 4], auto_reset=False), pkg.StopAfterNSteps(123))
    finally:
        core.enable_debug_timings(False)
    assert isinstance(core.timer, core.TimerOutput)
    assert set(core.timer) == {"reset!", "push!(policy) PreActStage", "optimise! PreActStage", "push!(hook) PreActStage", "plan!", "act!",
                               "push!(policy) PostActStage", "optimise! PostActStage", "push!(hook) PostActStage"}
    assert all(n == 123 and sec >= 0 for n, sec in core.timer.values()) and "act!" in str(core.timer)


def test_reset_conditions_and_experiment(pkg):
    """reset_conditions.jl: ResetAfterNSteps(n) fires on its (n + 1)-th check (after n steps) and the whole batch is force-reset;
    ResetIfEnvTerminated never fires for a batched env.  Experiment bundles the four run arguments (run.jl:8-20)."""
    r = pkg.ResetAfterNSteps(3)
    assert [r.check(None, None) for _ in range(9)] == [False, False, False, True, False, False, False, True, False]
    assert pkg.ResetIfEnvTerminated().check(None, StubVecEnv([1])) is False
    env = StubVecEnv([50, 50])
    pkg.run(pkg.RandomPolicy(), env, pkg.StopAfterNSteps(10), None, pkg.ResetAfterNSteps(4))
    resets = [i for i, e in enumerate(env.log) if e == ("reset", True)]
    steps_before = [sum(1 for e in env.log[:i] if e[0] == "act_random") for i in resets]
    assert steps_before == [0, 4, 8]                               # run.jl:46 reset, then after every 4 steps
    env2 = StubVecEnv([2, 3])
    ex = pkg.Experiment(pkg.RandomPolicy(), env2, pkg.StopAfterNSteps(5), pkg.BatchStepsPerEpisode(2))
    assert pkg.run(ex) is ex and ex.hook[()] == [[2, 2], [3]]


class StubFusedAgent:
    """The surface run() uses of a device-resident OnPolicyAgent: run_episodes(n, budget) bookkeeping only.  As the library does
    without an episode budget, a call returns at the end of the last rollout its n steps complete, if there is one."""
    fusable = True

    def __init__(self, T):
        self.T, self._t, self.calls, self.pushed = T, 0, [], []

    def push(self, stage, env, action=None):
        self.pushed.append(stage)
        self.env = env

    def run_episodes(self, max_steps, budget):
        assert budget is None and max_steps >= 1
        first = self.T - self._t                 # steps to the end of the rollout being filled
        steps = max_steps if max_steps < first else max_steps - (max_steps - first) % self.T
        self.calls.append(("run_episodes", max_steps, steps))
        for _ in range(steps):
            self.env._step()
        self._t = (self._t + steps) % self.T
        return steps, 0

    def plan(self, env):
        from_stage = pkg_core.FusedAction("policy")
        self.calls.append(("plan",))
        return from_stage

    def act_fused(self, env):
        self.calls.append(("act_fused",))
        env._step()

    def optimise(self, stage):
        pass


def test_fused_fast_path_hands_whole_stretches_to_run_episodes(pkg):
    """run() with a fusable agent + a hook that does nothing per step + StopAfterNSteps: calls of the remaining steps (no
    episode budget) until exactly n env steps ran — a call that ends at a rollout boundary is followed by one for the rest — and the
    stage loop otherwise."""
    global pkg_core
    pkg_core = pkg.core
    agent = StubFusedAgent(T=8)
    env = StubVecEnv([5, 7])
    pkg.run(agent, env, pkg.StopAfterNSteps(21), pkg.DeviceEpisodeStats())   # per_step = False: nothing happens at the act stages
    assert agent.calls == [("run_episodes", 21, 16), ("run_episodes", 5, 5)]
    assert agent._t == 5 and env.log[0] == ("reset", True) and env.log[-1] == ("check",)
    assert agent.pushed == ["PreExperimentStage", "PreEpisodeStage", "PostExperimentStage"]   # run.jl:47: the forced reset starts an episode
    # a second run continues filling the same rollout: 3 more steps complete it
    pkg.run(agent, env, pkg.StopAfterNSteps(4), pkg.EmptyHook())
    assert agent.calls[-2:] == [("run_episodes", 4, 3), ("run_episodes", 1, 1)]
    # a per-step hook (or a reset condition) falls back to the stage protocol: plan! -> act_fused per step
    agent2 = StubFusedAgent(T=8)
    pkg.run(agent2, StubVecEnv([5, 7]), pkg.StopAfterNSteps(3), pkg.BatchStepsPerEpisode(2))
    assert agent2.calls == [("plan",), ("act_fused",)] * 3
    agent3 = StubFusedAgent(T=8)
    pkg.run(agent3, StubVecEnv([5, 7]), pkg.StopAfterNSteps(3), pkg.EmptyHook(), pkg.ResetAfterNSteps(2))
    assert agent3.calls == [("plan",), ("act_fused",)] * 3


def test_replay_agent_stage_logic_with_stubs(pkg):
    """learners.Agent (agent_base.jl:18-66 for a device ring): an episode-start frame for every lane at each PreEpisodeStage (run() pushes
    one after every forced reset), one frame + one controller insertion per PostActStage, the learner trains while the controller allows,
    re-entering run() on a filled ring is fine (the device ring keeps EpisodesBuffer's bookkeeping), soft-reset envs get their pending
    episode starts at PreActStage."""
    class Traj:
        def __init__(self):
            self.frames, self.first_states, self.pending_starts = 0, 0, 0
            self.controller = pkg.InsertSampleRatioController(ratio=0.5, threshold=3)

        def push_env(self, env, first_state_only=False):
            if first_state_only == 2:
                self.pending_starts += 1
            elif first_state_only:
                self.first_states += 1
            else:
                self.frames += 1

    class Learner:
        updates = 0

        def update(self):
            Learner.updates += 1

    class Policy:
        learner = Learner()
        optimise = pkg.QBasedPolicy.optimise              # the real method: `while trajectory.controller.on_sample(): learner.update()`

        def plan(self, env):
            return pkg.core.FusedAction("policy")

        def act_fused(self, env):
            env._step()

    traj = Traj()
    agent = pkg.Agent(Policy(), traj)
    env = StubVecEnv([4, 6])
    pkg.run(agent, env, pkg.StopAfterNSteps(9))
    assert traj.first_states == 1 and traj.frames == 9 and traj.controller.n_inserted == 9
    assert Learner.updates == traj.controller.n_sampled == int((9 - 3) * 0.5) + 1
    soft = 0 if getattr(env, "auto_reset", True) else 9
    assert traj.pending_starts == soft                      # one (cheap, masked) episode-start push per step for soft-reset envs only
    pkg.run(agent, env, pkg.StopAfterNSteps(2))             # re-entry: the forced reset starts a new episode for every lane
    assert traj.first_states == 2 and traj.frames == 11
    pkg.run(agent, env, pkg.StopAfterNSteps(4), None, pkg.ResetAfterNSteps(2))
    assert traj.first_states == 2 + 1 + 1                   # this run's start + the forced reset after its 2nd step
