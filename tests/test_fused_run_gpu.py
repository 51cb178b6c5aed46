"""GPU tests of run(agent, env, StopAfterNSteps(n), hook) on the fused PPO and DQN paths (b200rl_onpolicy_run_episodes /
b200rl_replay_run_episodes without an episode budget).

Each case runs two twins built from the same seeds: one through run(), one through the calls a StopAfterNSteps run is made of,
issued by hand: iterate(k) for whole rollouts from an empty one, collect(m) + update() otherwise (PPO), run_replay(m) per log
window (DQN), a log flush after each.  Both must leave the same state bit for bit (env fields and streams, rollout columns and
fill, parameters, Adam moments and step, last_stats; for DQN the ring, target, explorer streams and step and the controller
counters), the same episode log, and the same kernel launches apart from log flushes, of which run() may issue fewer."""
import numpy as np
import pytest

import test_episode_log_gpu as EL
import test_stop_episodes_gpu as SE

pytestmark = pytest.mark.gpu


class CountedFlushes:
    """launches the flushes of a DeviceEpisodeLog issue, counted apart from the run's own"""

    def __init__(self, ctx, hook):
        self.launches = 0
        flush = hook.flush

        def counted():
            l0 = ctx.launch_count()
            flush()
            self.launches += ctx.launch_count() - l0
        hook.flush = counted


def _stages(pkg, agent, env, hook, body):
    """run()'s experiment stages around `body`, as run() issues them for a fused run"""
    core = pkg.core
    hook.push(core.PreExperimentStage, agent, env)
    agent.push(core.PreExperimentStage, env)
    env.reset_(is_force=True)
    agent.push(core.PreEpisodeStage, env)
    body()
    agent.push(core.PostExperimentStage, env)
    hook.push(core.PostExperimentStage, agent, env)
    env.check()


def _onpolicy_by_hand(pkg, agent, n, hook):
    """the calls of a StopAfterNSteps(n) run: whole rollouts as iterate(k) (one at a time when the stats are fetched; at most
    window // T per log window), a partial rollout as collect(m) and update() when it fills"""
    logs, window = pkg.core._episode_log_window(hook)
    stop, T = pkg.StopAfterNSteps(n), agent.T
    while True:
        if agent._t == 0 and stop.remaining() >= T and (window is None or T <= window):
            k = 1 if agent.fetch_stats else stop.remaining() // T
            k = k if window is None else min(k, window // T)
            agent.iterate(k, want_stats=agent.fetch_stats)
            m = k * T
        else:
            m = min(T - agent._t, stop.remaining(), window or n)
            agent.collect(m)
            if agent._t == T:
                agent.update(want_stats=agent.fetch_stats)
        for h in logs:
            h.flush()
        if stop.advance(m):
            return


def _run(pkg, ctx, make, runs, by_hand, capacity, state):
    """the twins of one case: (state, episode log lists, launches without flushes, all launches) each"""
    out = []
    for fused in (True, False):
        s = make()
        hook = pkg.DeviceEpisodeLog(s["env"].n, capacity=capacity) if capacity else pkg.EmptyHook()
        flushes = CountedFlushes(ctx, hook) if capacity else None
        l0 = ctx.launch_count()
        for n in runs:
            if fused:
                pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(n), hook)
            else:
                _stages(pkg, s["agent"], s["env"], hook, lambda: by_hand(s, n, hook))
        launches = ctx.launch_count() - l0
        lists = (hook.rewards, hook.steps) if capacity else None
        out.append((state(s), lists, launches - (flushes.launches if flushes else 0), launches))
        s["close"]()
    (a, la, na, ta), (b, lb, nb, tb) = out
    EL._same(a, b)
    assert la == lb
    assert na == nb
    assert ta == tb if not capacity else ta <= tb


ON_CASES = {   # (StopAfterNSteps of consecutive runs, DeviceEpisodeLog capacity or None, fetch_stats); T = 8
    "whole-rollouts": ([32, 11], None, False),
    "partial-rollout": ([29, 11], None, False),
    "log-window": ([29, 11], 12, False),
    "log-window-whole": ([32, 13], 12, False),
    "stats": ([29, 11], None, True),
    "stats-log-window": ([32, 13], 12, True),
}


@pytest.mark.parametrize("case", sorted(ON_CASES))
def test_onpolicy_steps_match_the_calls_by_hand(pkg, ctx, case):
    runs, capacity, fetch_stats = ON_CASES[case]
    cfg = SE.ON_CONFIGS["ppo-cartpole"]

    def make():
        env, net, agent = SE._onpolicy(pkg, ctx, cfg)
        agent.fetch_stats = fetch_stats

        def close():
            agent.close(); net.close(); env.close()
        return dict(env=env, net=net, agent=agent, close=close)

    def state(s):
        st = SE._on_state(pkg, s["env"], s["net"], s["agent"])
        st["t"] = np.array([s["agent"]._t, s["agent"].n_updates], np.int64)
        last = s["agent"].last_stats
        st["last_stats"] = np.zeros(0, np.float32) if last is None else np.array(last, copy=True)
        return st

    _run(pkg, ctx, make, runs, lambda s, n, hook: _onpolicy_by_hand(pkg, s["agent"], n, hook), capacity, state)


def _dqn_by_hand(pkg, s, n, hook):
    logs, window = pkg.core._episode_log_window(hook)
    for j in range(0, n, window or n):
        s["agent"].run_replay(s["env"], min(n - j, window or n))
        for h in logs:
            h.flush()


@pytest.mark.parametrize("runs,capacity", [([40, 9], None), ([40, 9], 12)])
def test_dqn_steps_match_the_calls_by_hand(pkg, ctx, runs, capacity):
    def make():
        s = SE._dqn(pkg, ctx, "exp")
        s["close"] = lambda: EL._dqn_close(s)
        return s

    def state(s):
        st = SE._dqn_state(pkg, s)
        st["explorer_step"] = np.array([s["policy"].explorer.step], np.int64)
        return st

    _run(pkg, ctx, make, runs, lambda s, n, hook: _dqn_by_hand(pkg, s, n, hook), capacity, state)
