"""GPU parity of the learner kernels (K6 policy inference, K7 loss + backward, K8 clip + Adam,
rollout plumbing, PPO / A2C updates) against the CPU oracle through the C ABI.
Tolerance: fp32 losses / gradients / parameters within 1e-5 relative (BASELINE north_star);
env integers / terminal flags / RNG streams bit-exact."""
import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu

REL = 1e-5
# A Gaussian log-density -0.5 (log v + d^2 / v + log 2pi) is a sum of O(1) terms that can cancel to ~0: "1e-5 relative" is asserted on
# the value (rtol) or, near a zero crossing, on the constant term every log-density contains (0.5 log 2pi = 0.919): atol = 1e-5 * 0.919
LOGP_ATOL = 1e-5 * 0.9189385


def rel_err(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)


def make_net(pkg, ctx, n_in, hidden, n_out, act, kind, seed):
    desc = O.ac_desc(n_in, hidden, n_out, act, kind == pkg.KIND_GAUSSIAN)
    rng = np.random.default_rng(seed)
    q = kind == pkg.KIND_Q
    params = O.glorot_params(desc, seed, q_net=q)
    params = params + 0.05 * rng.standard_normal(params.size).astype(np.float32)  # non-zero biases
    return pkg.Network(ctx, n_in, hidden, n_out, params, act=act, kind=kind), desc, params


@pytest.mark.parametrize("n_in,hidden,n_out,act", [(4, 64, 2, 0), (4, 64, 2, 1), (2, 64, 3, 0), (4, 128, 2, 0)])
def test_policy_act_categorical(pkg, ctx, n_in, hidden, n_out, act):
    net, desc, params = make_net(pkg, ctx, n_in, hidden, n_out, act, pkg.KIND_CATEGORICAL, 11)
    n = 5000
    rng = np.random.default_rng(0)
    obs = rng.standard_normal((n_in, n)).astype(np.float32)
    seeds = O.splitmix_states_fast(n, 4242)
    d_rng = ctx.malloc(n * 32); ctx.h2d(d_rng, seeds)
    out = net.act(obs, d_rng)
    ref = O.act_discrete(desc, params, obs, seeds)
    assert rel_err(out["heads"], ref["logits"]) < REL
    assert rel_err(out["value"], ref["value"]) < REL
    safe = ref["margin"] > 1e-4  # Gumbel arg-max decided by more than fp32 noise
    assert safe.mean() > 0.99
    assert np.array_equal(out["action"][safe], ref["action"][safe])
    np.testing.assert_allclose(out["logp"][safe], ref["logp"][safe], rtol=1e-5, atol=2e-6)
    rng_after = np.empty((n, 4), np.uint64); ctx.d2h(rng_after, d_rng)
    assert np.array_equal(rng_after, ref["rng"])          # n_out Float64 draws per env, bit-exact stream
    crit = net.values(obs)
    assert rel_err(crit, ref["value"]) < REL
    ctx.free(d_rng)


def test_policy_act_gaussian(pkg, ctx):
    net, desc, params = make_net(pkg, ctx, 3, 64, 1, 1, pkg.KIND_GAUSSIAN, 5)
    n = 4000
    rng = np.random.default_rng(1)
    obs = rng.standard_normal((3, n)).astype(np.float32)
    seeds = O.splitmix_states_fast(n, 77)
    d_rng = ctx.malloc(n * 32); ctx.h2d(d_rng, seeds)
    out = net.act(obs, d_rng)
    ref = O.act_gaussian(desc, O.hyper_array(), params, obs, seeds)
    sp = np.logaddexp(0, out["heads"][1].astype(np.float64))
    assert rel_err(out["heads"][0], ref["mu"]) < REL and rel_err(sp, ref["sigma"]) < REL
    # sampling only: z = mu + sigma * randn, randn = Box-Muller on two Float32 uniforms — the device logf / cosf differ from the host
    # libm by a few ulps, which is the whole tolerance here (the stream itself is bit-exact, see rng_after below)
    np.testing.assert_allclose(out["action"], ref["action"], rtol=2e-5, atol=2e-5)
    # log-probability of the GIVEN action (what the reference itself tests: test/utils/networks.jl:59-71, logp ≈ diagnormlogpdf(mu, sigma, a)):
    # the oracle's diagnormlogpdf at the device's own sampled action, 1e-5
    lp_given = np.array([O.lib().orc_normlogpdf1(float(m), float(sg), float(a)) for m, sg, a in zip(ref["mu"], ref["sigma"], out["action"])], np.float32)
    np.testing.assert_allclose(out["logp"], lp_given, rtol=1e-5, atol=LOGP_ATOL)
    rng_after = np.empty((n, 4), np.uint64); ctx.d2h(rng_after, d_rng)
    assert np.array_equal(rng_after, ref["rng"])
    ctx.free(d_rng)


CASES = [  # algo, kind, n_in, hidden, n_out, act, total, B
    ("ppo", 0, 4, 64, 2, 0, 3000, 2048), ("ppo", 0, 4, 64, 2, 1, 1500, 1000), ("a2c", 0, 2, 64, 3, 0, 900, None),
    ("a2c", 1, 3, 64, 1, 1, 2000, None), ("ppo", 1, 3, 64, 1, 0, 2000, 777), ("ppo", 0, 4, 128, 2, 0, 1200, 1000),
]


@pytest.mark.parametrize("algo,kind,n_in,hidden,n_out,act,total,B", CASES)
def test_loss_grad_and_adam_step(pkg, ctx, algo, kind, n_in, hidden, n_out, act, total, B):
    net, desc, params = make_net(pkg, ctx, n_in, hidden, n_out, act, kind, 3)
    rng = np.random.default_rng(7)
    states = rng.standard_normal((n_in, total)).astype(np.float32)
    gaussian = kind == 1
    actions = rng.uniform(-2, 2, total).astype(np.float32) if gaussian else rng.integers(1, n_out + 1, total).astype(np.int32)
    logp_old = (-0.7 + 0.2 * rng.standard_normal(total)).astype(np.float32)
    adv = rng.standard_normal(total).astype(np.float32); ret = rng.standard_normal(total).astype(np.float32)
    idx = None if B is None else rng.permutation(total)[:B].astype(np.int32)
    cfg = pkg.onpolicy_config(clip_range=0.2, w_entropy=0.01, algo=algo, max_grad_norm=0.5)
    mean, inv_std = O.adv_norm(adv)
    oalgo = {("ppo", 0): 0, ("a2c", 1): 1, ("ppo", 1): 2, ("a2c", 0): 3}[(algo, kind)]
    hyper = O.hyper_array(clip_range=0.2, w_entropy=0.01)
    g_ref, l_ref = O.ac_loss_grad(oalgo, desc, hyper, params, states, actions, logp_old, adv, ret, idx, mean, inv_std)
    got = net.ac_step(cfg, states, actions, logp_old, adv, ret, idx, mean, inv_std, apply_update=False)
    g = net.get(pkg.learners.NET_GRAD)
    assert rel_err(g, g_ref) < REL
    for k in ("actor_loss", "critic_loss", "entropy", "loss"):
        assert got[k] == pytest.approx(l_ref[k], rel=REL, abs=1e-6), k
    assert np.array_equal(net.get(), params)                      # apply_update = False leaves parameters alone
    # two optimiser steps: clip_by_global_norm! + Adam vs the oracle applied to the oracle gradient
    p = params.copy(); m = np.zeros_like(p); v = np.zeros_like(p); bt = np.array([0.9, 0.999], np.float32)
    for step in range(2):
        g_ref, _ = O.ac_loss_grad(oalgo, desc, hyper, p, states, actions, logp_old, adv, ret, idx, mean, inv_std)
        gc, gn = O.clip_by_global_norm(g_ref.astype(np.float32), 0.5)
        O.adam_step(p, gc, m, v, bt)
        got = net.ac_step(cfg, states, actions, logp_old, adv, ret, idx, mean, inv_std, apply_update=True)
        assert got["grad_norm"] == pytest.approx(gn, rel=REL)
        np.testing.assert_allclose(net.get(), p, rtol=0, atol=3e-6)
    np.testing.assert_allclose(net.get(pkg.learners.NET_M), m, rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(net.get(pkg.learners.NET_BETA_T), bt, rtol=1e-6)


def test_opt_state_export_import_roundtrip(pkg, ctx):
    net, desc, params = make_net(pkg, ctx, 4, 64, 2, 0, 0, 9)
    rng = np.random.default_rng(2)
    for which in (pkg.learners.NET_M, pkg.learners.NET_V, pkg.learners.NET_PARAMS):
        x = rng.standard_normal(net.nparams).astype(np.float32)
        net.set(which, x)
        assert np.array_equal(net.get(which), x)


def replay_rollout_on_oracle(kind, seeds, n, T, actions, continuous=False):
    """Teacher-forced oracle rollout: same env seeds, the GPU's actions, fused auto-reset."""
    ref = O.OracleVecEnv(kind, n, seeds)
    ref.reset(force=True)
    obs = [ref.get(O.F_OBS).T.copy()]
    rew, term = [], []
    for t in range(T):
        a = np.clip(actions[:, t], -2, 2) if continuous else actions[:, t]
        ref.step(a, auto_reset=True)
        rew.append(ref.get(O.F_REWARD).copy()); term.append(ref.get(O.F_TERMINAL).copy())
        obs.append(ref.get(O.F_OBS).T.copy())
    return np.stack(obs, axis=2), np.stack(rew, axis=1), np.stack(term, axis=1), ref


@pytest.mark.parametrize("use_host_perm", [True, False])
def test_ppo_cartpole_rollout_and_update(pkg, ctx, use_host_perm):
    """BASELINE config 2 at a size the oracle finishes quickly: N = 1024 CartPole envs, T = 32,
    4 epochs x 4 microbatches, actor/critic 4-64-64."""
    n, T, E, M = 1024, 32, 4, 4
    env_seeds = O.splitmix_states_fast(n, 1); pol_seeds = O.splitmix_states_fast(n, 2)
    env = pkg.B200VecEnv(ctx, "CartPole", n, env_seeds, auto_reset=True)
    net, desc, params = make_net(pkg, ctx, 4, 64, 2, 0, 0, 21)
    cfg = pkg.onpolicy_config(update_freq=T, n_epochs=E, n_microbatches=M)
    agent = pkg.OnPolicyAgent(ctx, net, env, cfg, pol_seeds)
    env.reset_(is_force=True)
    agent.collect(T)
    R = pkg.learners
    S, A, LP = agent.rollout(R.ROLL_STATE), agent.rollout(R.ROLL_ACTION), agent.rollout(R.ROLL_LOGP)
    RW, TM, V = agent.rollout(R.ROLL_REWARD), agent.rollout(R.ROLL_TERMINAL), agent.rollout(R.ROLL_VALUE)
    # (1) env side bit-exact given the actions
    obs_ref, rew_ref, term_ref, ref_env = replay_rollout_on_oracle(O.KIND_CARTPOLE, env_seeds, n, T, A)
    assert np.array_equal(S[:, :, :T].view(np.uint32), np.asfortranarray(obs_ref[:, :, :T]).view(np.uint32))
    assert np.array_equal(RW, rew_ref) and np.array_equal(TM, term_ref)
    assert np.array_equal(env.rng_state(), ref_env.get(O.F_RNG))
    assert TM.sum() > 0                                             # the rollout did cross episode ends
    # (2) policy side: same streams, actions agree wherever the Gumbel margin is not fp32 noise
    rng_state = pol_seeds.copy()
    n_bad = 0
    for t in range(T):
        o = O.act_discrete(desc, params, S[:, :, t], rng_state)
        safe = o["margin"] > 1e-4
        n_bad += int((~safe).sum())
        assert np.array_equal(A[safe, t], o["action"][safe])
        np.testing.assert_allclose(LP[safe, t], o["logp"][safe], rtol=1e-5, atol=2e-6)
        np.testing.assert_allclose(V[:, t], o["value"], rtol=1e-5, atol=2e-6)
        rng_state = o["rng"]
    assert n_bad < 0.01 * n * T
    assert np.array_equal(agent.rollout(R.ROLL_RNG).T, rng_state)
    # (3) update
    nt = n * T
    perm = None
    if use_host_perm:
        perm = np.stack([np.random.default_rng(100 + e).permutation(nt) for e in range(E)]).astype(np.int32)
    stats = agent.update(perm, want_stats=True)
    V = agent.rollout(R.ROLL_VALUE)
    np.testing.assert_allclose(V[:, T], O.critic_values(desc, params, obs_ref[:, :, T]), rtol=1e-5, atol=2e-6)
    ADV, RET = agent.rollout(R.ROLL_ADV), agent.rollout(R.ROLL_RET)
    adv_ref = O.gae(RW, V, np.float32(0.99), np.float32(0.95), terminal=TM, dims=2, dtype=np.float32)
    assert np.array_equal(ADV, adv_ref)                             # GAE bit-exact on identical inputs
    np.testing.assert_allclose(RET, adv_ref + V[:, :T], rtol=0, atol=1e-6)
    mean, inv_std = O.adv_norm(np.asfortranarray(ADV).ravel(order="F"))
    np.testing.assert_allclose(agent.rollout(R.ROLL_NORM), [mean, inv_std], rtol=1e-6)
    # oracle optimiser loop on the flattened (N*T) rollout (flat index = env + N*t)
    sf = np.asfortranarray(S[:, :, :T]).reshape(4, nt, order="F")
    af, lf = A.ravel(order="F"), LP.ravel(order="F")
    advf, retf = ADV.ravel(order="F"), RET.ravel(order="F")
    hyper = O.hyper_array()
    p = params.copy(); m = np.zeros_like(p); v = np.zeros_like(p); bt = np.array([0.9, 0.999], np.float32)
    B = nt // M
    row = 0
    for e in range(E):
        for mb in range(M):
            if use_host_perm:
                idx = perm[e, mb * B:(mb + 1) * B]
            else:
                key = (0 * 1000003 + e * 7919 + 12345) & 0xFFFFFFFF
                idx = np.array([O.perm_index(mb * B + j, nt, key) for j in range(B)], np.int32)
            g, l = O.ac_loss_grad(0, desc, hyper, p, sf, af, lf, advf, retf, idx, mean, inv_std)
            gc, gn = O.clip_by_global_norm(g.astype(np.float32), 0.5)
            O.adam_step(p, gc, m, v, bt)
            tol = 1e-5 * (1 + row)  # parameters drift apart by fp32 rounding as steps accumulate
            assert stats[row, 0] == pytest.approx(l["actor_loss"], rel=tol, abs=2e-6), (row, "actor")
            assert stats[row, 1] == pytest.approx(l["critic_loss"], rel=tol), (row, "critic")
            assert stats[row, 2] == pytest.approx(l["entropy"], rel=tol), (row, "entropy")
            assert stats[row, 4] == pytest.approx(gn, rel=10 * tol), (row, "gnorm")
            row += 1
    diff = np.abs(net.get() - p)                                  # 16 Adam steps apart: fp32 rounding of tiny gradient components
    assert np.mean(diff <= 2e-5) > 0.998 and diff.max() < 2e-4    # moves a few weights by a fraction of one lr step
    assert agent.fill() == (0, T)
    if not use_host_perm:  # the device permutation really is a permutation
        assert sorted(O.perm_index(q, 4096, 99) for q in range(4096)) == list(range(4096))


def test_a2c_pendulum_gaussian_rollout_and_update(pkg, ctx):
    """BASELINE config 3 shape: Pendulum (continuous torque), A2C with GAE(lambda = 0.95), Gaussian head."""
    n, T = 512, 16
    env_seeds = O.splitmix_states_fast(n, 31); pol_seeds = O.splitmix_states_fast(n, 32)
    env = pkg.B200VecEnv(ctx, "Pendulum", n, env_seeds, auto_reset=True)
    net, desc, params = make_net(pkg, ctx, 3, 64, 1, 1, pkg.KIND_GAUSSIAN, 8)
    cfg = pkg.onpolicy_config(update_freq=T, n_epochs=1, n_microbatches=1, algo="a2c", w_entropy=0.01)
    agent = pkg.OnPolicyAgent(ctx, net, env, cfg, pol_seeds)
    env.reset_(is_force=True)
    agent.collect(T)
    R = pkg.learners
    S, A, LP = agent.rollout(R.ROLL_STATE), agent.rollout(R.ROLL_ACTION), agent.rollout(R.ROLL_LOGP)
    RW, TM = agent.rollout(R.ROLL_REWARD), agent.rollout(R.ROLL_TERMINAL)
    obs_ref, rew_ref, term_ref, _ = replay_rollout_on_oracle(O.KIND_PENDULUM, env_seeds, n, T, A, continuous=True)
    assert np.array_equal(S[:, :, :T].view(np.uint32), np.asfortranarray(obs_ref[:, :, :T]).view(np.uint32))
    assert np.array_equal(RW, rew_ref) and np.array_equal(TM, term_ref)
    o = O.act_gaussian(desc, O.hyper_array(), params, S[:, :, 0], pol_seeds)
    np.testing.assert_allclose(A[:, 0], o["action"], rtol=2e-5, atol=2e-5)      # sampling only (Box-Muller ulps)
    lp_given = np.array([O.lib().orc_normlogpdf1(float(m), float(sg), float(a)) for m, sg, a in zip(o["mu"], o["sigma"], A[:, 0])], np.float32)
    np.testing.assert_allclose(LP[:, 0], lp_given, rtol=1e-5, atol=LOGP_ATOL)   # given-action log-prob at 1e-5
    stats = agent.update(None, want_stats=True)
    V, ADV, RET = agent.rollout(R.ROLL_VALUE), agent.rollout(R.ROLL_ADV), agent.rollout(R.ROLL_RET)
    assert np.array_equal(ADV, O.gae(RW, V, np.float32(0.99), np.float32(0.95), terminal=TM, dims=2, dtype=np.float32))
    assert np.array_equal(RET, O.discount_rewards(RW, np.float32(0.99), terminal=TM, init=V[:, T].copy(), dims=2, dtype=np.float32))
    nt = n * T
    mean, inv_std = O.adv_norm(ADV.ravel(order="F"))
    g, l = O.ac_loss_grad(1, desc, O.hyper_array(w_entropy=0.01), params, np.asfortranarray(S[:, :, :T]).reshape(3, nt, order="F"),
                          A.ravel(order="F"), LP.ravel(order="F"), ADV.ravel(order="F"), RET.ravel(order="F"), None, mean, inv_std)
    # actor_loss = -mean(logp_a * A_hat) is a sum of terms of both signs (A_hat has zero mean): 1e-5 is asserted relative to the size
    # of the summands, mean |logp_a * A_hat| — the conditioning-aware form of the north star's "1e-5 relative" for a cancelling sum
    a_hat = (ADV.ravel(order="F") - mean) * inv_std
    l1_mass = float(np.mean(np.abs(LP.ravel(order="F").astype(np.float64) * a_hat)))
    assert abs(stats[0, 0] - l["actor_loss"]) <= 1e-5 * max(l1_mass, abs(l["actor_loss"]))
    assert stats[0, 1] == pytest.approx(l["critic_loss"], rel=1e-5)
    assert stats[0, 2] == pytest.approx(l["entropy"], rel=1e-5)
    gc, gn = O.clip_by_global_norm(g.astype(np.float32), 0.5)
    assert stats[0, 4] == pytest.approx(gn, rel=1e-5)
    assert rel_err(net.get(pkg.learners.NET_GRAD), gc) < 1e-5      # the clipped gradient itself, L2-relative
    p = params.copy(); m = np.zeros_like(p); v = np.zeros_like(p); bt = np.array([0.9, 0.999], np.float32)
    O.adam_step(p, gc, m, v, bt)
    np.testing.assert_allclose(net.get(), p, rtol=0, atol=3e-6)


def test_run_loop_with_host_actions_matches_fused_path(pkg, ctx):
    """run(agent, env, StopAfterNSteps, hook) with host action buffers every step (the reference's
    stage protocol) must produce the same parameters as the fused device path."""
    n, T = 256, 8
    outs = []
    for host in (True, False):
        env = pkg.B200VecEnv(ctx, "CartPole", n, O.splitmix_states_fast(n, 5), auto_reset=True)
        net, desc, params = make_net(pkg, ctx, 4, 64, 2, 0, 0, 2)
        cfg = pkg.onpolicy_config(update_freq=T, n_epochs=2, n_microbatches=2)
        agent = pkg.OnPolicyAgent(ctx, net, env, cfg, O.splitmix_states_fast(n, 6), host_actions=host)
        hook = pkg.DeviceEpisodeStats()
        pkg.run(agent, env, pkg.StopAfterNSteps(3 * T), hook)
        assert agent.n_updates == 3
        outs.append((net.get(), env.internal_state(), hook.stats))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
    assert outs[0][2] == outs[1][2] and outs[0][2]["env_steps"] == 3 * T * n


def test_tensor_core_and_cuda_core_paths_agree(pkg, ctx):
    """K6/K7 exist as wgmma (3-term fp16 split, H = 64) and FP32-FFMA kernels; both must meet the oracle
    and each other well inside the 1e-5 bar."""
    net, desc, params = make_net(pkg, ctx, 4, 64, 2, 0, 0, 17)
    rng = np.random.default_rng(3)
    total, B = 5000, 4096
    states = rng.standard_normal((4, total)).astype(np.float32)
    actions = rng.integers(1, 3, total).astype(np.int32)
    logp_old = (-0.7 + 0.2 * rng.standard_normal(total)).astype(np.float32)
    adv = rng.standard_normal(total).astype(np.float32); ret = rng.standard_normal(total).astype(np.float32)
    idx = rng.permutation(total)[:B].astype(np.int32)
    cfg = pkg.onpolicy_config(clip_range=0.2, w_entropy=0.01)
    g_ref, l_ref = O.ac_loss_grad(0, desc, O.hyper_array(clip_range=0.2, w_entropy=0.01), params, states, actions, logp_old, adv, ret, idx, 0.1, 0.9)
    out = {}
    try:
        for tc in (0, 1):
            pkg._lib.check(ctx.lib.b200rl_set_tensor_cores(tc))
            got = net.ac_step(cfg, states, actions, logp_old, adv, ret, idx, 0.1, 0.9, apply_update=False)
            out[tc] = (net.get(pkg.learners.NET_GRAD), got, net.values(states[:, :1000]))
            assert rel_err(out[tc][0], g_ref) < REL, tc
            assert got["loss"] == pytest.approx(l_ref["loss"], rel=REL, abs=1e-6), tc
    finally:
        pkg._lib.check(ctx.lib.b200rl_set_tensor_cores(1))
    assert rel_err(out[1][0], out[0][0]) < 5e-6
    assert rel_err(out[1][2], out[0][2]) < 5e-6


# ---------------------------------------------------------------------------------------------------------------------------
# BASELINE sizes: configs[1] (65 536 CartPole envs, PPO) and configs[2] (32 768 Pendulum envs, A2C + GAE(0.95), Gaussian head).
# The env side is replayed on the oracle at full size (bit-exact), the policy on sampled columns, and the first optimiser step of
# the update on the WHOLE first minibatch (524 288 / 1 048 576 samples through the OpenMP oracle) at 1e-5.
def _first_step_reference(oalgo, desc, hyper, params, S, A, LP, ADV, RET, idx, ns, T, max_grad_norm=0.5):
    nt = A.size
    sf = np.asfortranarray(S[:, :, :T]).reshape(ns, nt, order="F")
    advf = ADV.ravel(order="F")
    mean, inv_std = O.adv_norm(advf)
    g, l = O.ac_loss_grad(oalgo, desc, hyper, params, sf, A.ravel(order="F"), LP.ravel(order="F"), advf, RET.ravel(order="F"), idx, mean, inv_std)
    gc, gn = O.clip_by_global_norm(g.astype(np.float32), max_grad_norm)
    return l, gn, (mean, inv_std), advf


def test_ppo_cartpole_at_baseline_size_65536(pkg, ctx):
    n, T, E, M = 65536, 32, 4, 4
    env_seeds = O.splitmix_states_fast(n, 0x9E37); pol_seeds = O.splitmix_states_fast(n, 0x1234)
    env = pkg.B200VecEnv(ctx, "CartPole", n, env_seeds, auto_reset=True)
    net, desc, params = make_net(pkg, ctx, 4, 64, 2, 0, 0, 123)
    agent = pkg.OnPolicyAgent(ctx, net, env, pkg.onpolicy_config(update_freq=T, n_epochs=E, n_microbatches=M), pol_seeds, host_actions=False)
    env.reset_(is_force=True)
    agent.collect(T)
    R = pkg.learners
    S, A, LP = agent.rollout(R.ROLL_STATE), agent.rollout(R.ROLL_ACTION), agent.rollout(R.ROLL_LOGP)
    RW, TM = agent.rollout(R.ROLL_REWARD), agent.rollout(R.ROLL_TERMINAL)
    obs_ref, rew_ref, term_ref, ref_env = replay_rollout_on_oracle(O.KIND_CARTPOLE, env_seeds, n, T, A)
    assert np.array_equal(S[:, :, :T].view(np.uint32), np.asfortranarray(obs_ref[:, :, :T]).view(np.uint32))      # 2 M env-steps bit-exact
    assert np.array_equal(RW, rew_ref) and np.array_equal(TM, term_ref) and np.array_equal(env.rng_state(), ref_env.get(O.F_RNG))
    assert np.array_equal(env.flags(), ref_env.get(O.F_FLAGS)) and np.array_equal(env.t(), ref_env.get(O.F_T))
    o = O.act_discrete(desc, params, S[:, :, 0], pol_seeds)                         # column 0: the policy streams start here
    safe = o["margin"] > 1e-4
    assert safe.mean() > 0.99 and np.array_equal(A[safe, 0], o["action"][safe])
    np.testing.assert_allclose(LP[safe, 0], o["logp"][safe], rtol=1e-5, atol=2e-6)
    nt = n * T
    perm = np.stack([np.random.default_rng(500 + e).permutation(nt) for e in range(E)]).astype(np.int32)
    stats = agent.update(perm, want_stats=True)
    V, ADV, RET = agent.rollout(R.ROLL_VALUE), agent.rollout(R.ROLL_ADV), agent.rollout(R.ROLL_RET)
    np.testing.assert_allclose(V[:, T], O.critic_values(desc, params, obs_ref[:, :, T]), rtol=1e-5, atol=2e-6)
    assert np.array_equal(ADV, O.gae(RW, V, np.float32(0.99), np.float32(0.95), terminal=TM, dims=2, dtype=np.float32))   # GAE bit-exact at full size
    l, gn, (mean, inv_std), _ = _first_step_reference(0, desc, O.hyper_array(), params, S, A, LP, ADV, RET, perm[0, :nt // M], 4, T)
    np.testing.assert_allclose(agent.rollout(R.ROLL_NORM), [mean, inv_std], rtol=1e-6)
    assert stats[0, 0] == pytest.approx(l["actor_loss"], rel=1e-5, abs=2e-6)
    assert stats[0, 1] == pytest.approx(l["critic_loss"], rel=1e-5)
    assert stats[0, 2] == pytest.approx(l["entropy"], rel=1e-5)
    assert stats[0, 4] == pytest.approx(gn, rel=1e-5)
    assert np.isfinite(stats).all() and np.isfinite(net.get()).all()
    agent.close(); net.close(); env.close()


def test_a2c_pendulum_at_baseline_size_32768(pkg, ctx):
    n, T = 32768, 32
    env_seeds = O.splitmix_states_fast(n, 31); pol_seeds = O.splitmix_states_fast(n, 32)
    env = pkg.B200VecEnv(ctx, "Pendulum", n, env_seeds, auto_reset=True)
    net, desc, params = make_net(pkg, ctx, 3, 64, 1, 1, pkg.KIND_GAUSSIAN, 8)
    cfg = pkg.onpolicy_config(update_freq=T, n_epochs=1, n_microbatches=1, algo="a2c", w_entropy=0.01)
    agent = pkg.OnPolicyAgent(ctx, net, env, cfg, pol_seeds, host_actions=False)
    env.reset_(is_force=True)
    agent.collect(T)
    R = pkg.learners
    S, A, LP = agent.rollout(R.ROLL_STATE), agent.rollout(R.ROLL_ACTION), agent.rollout(R.ROLL_LOGP)
    RW, TM = agent.rollout(R.ROLL_REWARD), agent.rollout(R.ROLL_TERMINAL)
    obs_ref, rew_ref, term_ref, ref_env = replay_rollout_on_oracle(O.KIND_PENDULUM, env_seeds, n, T, A, continuous=True)
    assert np.array_equal(S[:, :, :T].view(np.uint32), np.asfortranarray(obs_ref[:, :, :T]).view(np.uint32))      # 1 M env-steps bit-exact
    assert np.array_equal(RW, rew_ref) and np.array_equal(TM, term_ref) and np.array_equal(env.rng_state(), ref_env.get(O.F_RNG))
    o = O.act_gaussian(desc, O.hyper_array(), params, S[:, :, 0], pol_seeds)
    lp_given = np.array([O.lib().orc_normlogpdf1(float(m), float(sg), float(a)) for m, sg, a in zip(o["mu"], o["sigma"], A[:, 0])], np.float32)
    np.testing.assert_allclose(LP[:, 0], lp_given, rtol=1e-5, atol=LOGP_ATOL)
    stats = agent.update(None, want_stats=True)
    V, ADV, RET = agent.rollout(R.ROLL_VALUE), agent.rollout(R.ROLL_ADV), agent.rollout(R.ROLL_RET)
    assert np.array_equal(ADV, O.gae(RW, V, np.float32(0.99), np.float32(0.95), terminal=TM, dims=2, dtype=np.float32))
    assert np.array_equal(RET, O.discount_rewards(RW, np.float32(0.99), terminal=TM, init=V[:, T].copy(), dims=2, dtype=np.float32))
    l, gn, (mean, inv_std), advf = _first_step_reference(1, desc, O.hyper_array(w_entropy=0.01), params, S, A, LP, ADV, RET, None, 3, T)
    a_hat = (advf - mean) * inv_std
    l1_mass = float(np.mean(np.abs(LP.ravel(order="F").astype(np.float64) * a_hat)))
    assert abs(stats[0, 0] - l["actor_loss"]) <= 1e-5 * max(l1_mass, abs(l["actor_loss"]))
    assert stats[0, 1] == pytest.approx(l["critic_loss"], rel=1e-5)
    assert stats[0, 2] == pytest.approx(l["entropy"], rel=1e-5)
    assert stats[0, 4] == pytest.approx(gn, rel=1e-5)
    agent.close(); net.close(); env.close()
