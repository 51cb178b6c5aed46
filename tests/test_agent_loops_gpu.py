"""The host side of the agent loops: the optimiser step of an H = 128 actor-critic update against the oracle, CUDA-graph replayed
iterations (b200rl_onpolicy_iterate) and replayed "1 step + m updates" units (b200rl_replay_run) against eager launches —
results bit for bit, and the host counters (launches, optimiser steps, env steps) exactly as an eager run leaves them."""
import numpy as np
import pytest

import oracle_lib as O
from test_nn_gpu import make_net
from test_replay_fused_gpu import _assert_same, _close, _setup, _state

pytestmark = pytest.mark.gpu


def test_h128_ppo_update_matches_the_oracle(pkg, ctx):
    """An actor-critic pair with H = 128 has 34 691 parameters: more CTAs (136) than an H100 has SMs for the single-launch
    reduce + clip + Adam, so the update runs the staged optimiser kernels.  Same oracle loop as test_nn_gpu's PPO test."""
    n, T, E, M = 256, 8, 2, 2
    env = pkg.B200VecEnv(ctx, "CartPole", n, O.splitmix_states_fast(n, 1), auto_reset=True)
    net, desc, params = make_net(pkg, ctx, 4, 128, 2, 0, 0, 21)
    agent = pkg.OnPolicyAgent(ctx, net, env, pkg.onpolicy_config(update_freq=T, n_epochs=E, n_microbatches=M), O.splitmix_states_fast(n, 2))
    env.reset_(is_force=True)
    agent.collect(T)
    R = pkg.learners
    S, A, LP = agent.rollout(R.ROLL_STATE), agent.rollout(R.ROLL_ACTION), agent.rollout(R.ROLL_LOGP)
    stats = agent.update(want_stats=True)
    ADV, RET = agent.rollout(R.ROLL_ADV), agent.rollout(R.ROLL_RET)
    nt = n * T
    mean, inv_std = O.adv_norm(np.asfortranarray(ADV).ravel(order="F"))
    sf = np.asfortranarray(S[:, :, :T]).reshape(4, nt, order="F")
    af, lf = A.ravel(order="F"), LP.ravel(order="F")
    advf, retf = ADV.ravel(order="F"), RET.ravel(order="F")
    hyper = O.hyper_array()
    p = params.copy(); m = np.zeros_like(p); v = np.zeros_like(p); bt = np.array([0.9, 0.999], np.float32)
    B = nt // M
    row = 0
    for e in range(E):
        for mb in range(M):
            key = (0 * 1000003 + e * 7919 + 12345) & 0xFFFFFFFF
            idx = np.array([O.perm_index(mb * B + j, nt, key) for j in range(B)], np.int32)
            g, l = O.ac_loss_grad(0, desc, hyper, p, sf, af, lf, advf, retf, idx, mean, inv_std)
            gc, gn = O.clip_by_global_norm(g.astype(np.float32), 0.5)
            O.adam_step(p, gc, m, v, bt)
            tol = 1e-5 * (1 + row)
            assert stats[row, 0] == pytest.approx(l["actor_loss"], rel=tol, abs=2e-6), (row, "actor")
            assert stats[row, 1] == pytest.approx(l["critic_loss"], rel=tol), (row, "critic")
            assert stats[row, 2] == pytest.approx(l["entropy"], rel=tol), (row, "entropy")
            assert stats[row, 4] == pytest.approx(gn, rel=10 * tol), (row, "gnorm")
            row += 1
    diff = np.abs(net.get() - p)
    assert np.mean(diff <= 2e-5) > 0.998 and diff.max() < 2e-4
    assert agent.fill() == (0, T)
    agent.close(); net.close(); env.close()


def _make(pkg, ctx, hidden, n=512, T=8, seed=11):
    env = pkg.B200VecEnv(ctx, "CartPole", n, O.splitmix_states_fast(n, seed), auto_reset=True)
    params = O.glorot_params(O.ac_desc(4, hidden, 2, 0), 77)
    params = params + 0.05 * np.random.default_rng(3).standard_normal(params.size).astype(np.float32)
    net = pkg.Network(ctx, 4, hidden, 2, params, act=0, kind=pkg.KIND_CATEGORICAL)
    cfg = pkg.onpolicy_config(update_freq=T, n_epochs=2, n_microbatches=2)
    agent = pkg.OnPolicyAgent(ctx, net, env, cfg, O.splitmix_states_fast(n, seed + 1), host_actions=False)
    env.reset_(is_force=True)
    return env, net, agent


def _onpolicy_state(pkg, env, net, agent, stats):
    R = pkg.learners
    return dict(params=net.get(), m=net.get(R.NET_M), v=net.get(R.NET_V), bt=net.get(R.NET_BETA_T), state=env.internal_state(),
                erng=env.rng_state(), prng=agent.rollout(R.ROLL_RNG), stats=np.asarray(stats), ep=env.episode_stats(), steps=net.step_count())


def _assert_same_onpolicy(a, b):
    for k in ("params", "m", "v", "bt", "state", "erng", "prng", "stats"):
        assert np.asarray(a[k]).tobytes(order="A") == np.asarray(b[k]).tobytes(order="A"), k
    assert a["ep"] == b["ep"] and a["steps"] == b["steps"]


def test_h128_iterate_is_bit_identical_to_eager_iterations(pkg, ctx):
    T, iters = 8, 5
    outs = []
    for graph in (True, False):
        env, net, agent = _make(pkg, ctx, 128, T=T)
        l0 = ctx.launch_count()
        if graph:
            stats = agent.iterate(iters, want_stats=True)
            assert agent.graph_active()
        else:
            for _ in range(iters):
                agent.collect(T)
                stats = agent.update(want_stats=True)
        outs.append(dict(_onpolicy_state(pkg, env, net, agent, stats), launches=ctx.launch_count() - l0))
        agent.close(); net.close(); env.close()
    a, b = outs
    _assert_same_onpolicy(a, b)
    assert a["launches"] == b["launches"]
    assert a["ep"]["env_steps"] == iters * T * 512 and a["steps"] == iters * 4


def test_iterate_recaptures_when_the_max_timeout_changes(pkg, ctx):
    """MaxTimeoutEnv's limit is a launch argument of the fused rollout: a graph captured before set_max_timeout must not be
    replayed after it."""
    T = 8
    outs = []
    for graph in (True, False):
        env, net, agent = _make(pkg, ctx, 64, T=T, seed=5)
        stats = None
        for phase in range(2):
            if phase == 1:
                env.set_max_timeout(7)
            if graph:
                stats = agent.iterate(3, want_stats=True)
            else:
                for _ in range(3):
                    agent.collect(T)
                    stats = agent.update(want_stats=True)
        if graph:
            assert agent.graph_active()
        outs.append(_onpolicy_state(pkg, env, net, agent, stats))
        agent.close(); net.close(); env.close()
    _assert_same_onpolicy(*outs)
    assert outs[0]["ep"]["episodes"] > 0


def test_replay_units_keep_the_host_counters(pkg, ctx):
    """ratio 1, threshold 1: every call of run(agent, env, StopAfterNSteps(1)) is one "1 step + 1 update" unit — eager on the
    first call, captured on the second, replayed after that.  Every call adds the same launches, optimiser steps and env steps."""
    lanes = 127
    fast, stage = _setup(pkg, ctx, 100, ratio=1.0, threshold=1), _setup(pkg, ctx, 100, ratio=1.0, threshold=1)
    stage["agent"].fusable = False
    deltas = []
    for _ in range(10):
        l0, s0, e0 = ctx.launch_count(), fast["net"].step_count(), fast["env"].episode_stats()["env_steps"]
        pkg.run(fast["agent"], fast["env"], pkg.StopAfterNSteps(1), pkg.EmptyHook())
        deltas.append((ctx.launch_count() - l0, fast["net"].step_count() - s0, fast["env"].episode_stats()["env_steps"] - e0))
        pkg.run(stage["agent"], stage["env"], pkg.StopAfterNSteps(1), pkg.EmptyHook())
    assert fast["agent"].graph_active()
    assert deltas == [deltas[0]] * 10, deltas
    assert deltas[0][1:] == (1, lanes)
    assert fast["agent"]._replay is not None and stage["agent"]._replay is None
    _assert_same(_state(pkg, fast), _state(pkg, stage))
    _close(fast); _close(stage)
