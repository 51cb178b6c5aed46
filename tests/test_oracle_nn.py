"""Second opinion on the UNPINNED learner restatement (RLZoo PPO/A2C/DQN, Optimisers Adam are
absent from /root/reference): the oracle's hand-written gradients must agree with PyTorch
autograd on the same loss written with torch ops, and its Adam with torch.optim.Adam(eps=1e-8).
Also pins the in-tree formulas: clip_by_global_norm! (basic.jl:19-29), normlogpdf against the
closed form used by the reference tests (RLCore/test/utils/distributions.jl:19-22: mu=10,
sigma=5, x=4), TargetNetwork sync (target_network.jl:70-88)."""
import numpy as np
import pytest
import torch

import oracle_lib as O
import q_ref as Q
from q_ref import unpack_mlp

torch.set_num_threads(2)


def make_batch(ns, total, rng, gaussian):
    states = rng.standard_normal((ns, total)).astype(np.float32)
    actions = rng.uniform(-2, 2, total).astype(np.float32) if gaussian else rng.integers(1, 3, total).astype(np.int32)
    logp_old = (-0.7 + 0.2 * rng.standard_normal(total)).astype(np.float32)
    adv = rng.standard_normal(total).astype(np.float32)
    ret = rng.standard_normal(total).astype(np.float32)
    return states, actions, logp_old, adv, ret


@pytest.mark.parametrize("algo,act", [(0, O.ACT_RELU), (0, O.ACT_TANH), (3, O.ACT_RELU), (1, O.ACT_TANH), (2, O.ACT_RELU)])
def test_actor_critic_grad_matches_autograd(algo, act):
    gaussian = algo in (1, 2)
    ns, H, total, B = (3 if gaussian else 4), 64, 700, 512
    n_out = 1 if gaussian else 2
    desc = O.ac_desc(ns, H, n_out, act, gaussian)
    rng = np.random.default_rng(algo * 10 + act)
    params = O.glorot_params(desc, seed=1) + 0.05 * rng.standard_normal(O.ac_nparams(desc)).astype(np.float32)
    states, actions, logp_old, adv, ret = make_batch(ns, total, rng, gaussian)
    idx = rng.permutation(total)[:B].astype(np.int32)
    hyper = O.hyper_array(clip_range=0.2, w_entropy=0.01)
    mean, inv_std = O.adv_norm(adv)
    grad, losses = O.ac_loss_grad(algo, desc, hyper, params, states, actions, logp_old, adv, ret, idx, mean, inv_std)

    p = torch.tensor(params, dtype=torch.float64, requires_grad=True)
    heads = [1, 1] if gaussian else [2]
    actor, na = unpack_mlp(p, ns, H, heads, act)
    critic, _ = unpack_mlp(p[na:], ns, H, [1], act)
    x = torch.tensor(states.T[idx], dtype=torch.float64)
    A = (torch.tensor(adv[idx], dtype=torch.float64) - mean) * inv_std
    z = actor(x)
    if gaussian:
        mu, sigma = z[:, 0], torch.nn.functional.softplus(z[:, 1])
        a = torch.tensor(actions[idx], dtype=torch.float64)
        s = sigma + 1e-8
        logp = -0.5 * (torch.log(s * s) + (a - mu) ** 2 / (s * s) + float(np.float32(np.log(np.float32(2 * np.pi)))))
        ent = (torch.log(sigma) + 0.5 * (np.log(2 * np.pi) + 1)).mean()
    else:
        lp = torch.log_softmax(z, dim=1)
        logp = lp[torch.arange(B), torch.tensor(actions[idx] - 1, dtype=torch.long)]
        ent = -(lp.exp() * lp).sum(1).mean()
    if algo in (0, 2):
        ratio = torch.exp(logp - torch.tensor(logp_old[idx], dtype=torch.float64))
        actor_loss = -torch.min(ratio * A, torch.clamp(ratio, 0.8, 1.2) * A).mean()
    else:
        actor_loss = -(logp * A).mean()
    v = critic(x)[:, 0]
    critic_loss = ((torch.tensor(ret[idx], dtype=torch.float64) - v) ** 2).mean()
    loss = 1.0 * actor_loss + 0.5 * critic_loss - 0.01 * ent
    loss.backward()
    g_t = p.grad.numpy()
    assert losses["actor_loss"] == pytest.approx(actor_loss.item(), rel=2e-5, abs=1e-6)
    assert losses["critic_loss"] == pytest.approx(critic_loss.item(), rel=2e-5)
    assert losses["entropy"] == pytest.approx(ent.item(), rel=2e-5)
    assert losses["loss"] == pytest.approx(loss.item(), rel=2e-5, abs=1e-6)
    assert np.linalg.norm(grad - g_t) <= 2e-5 * np.linalg.norm(g_t)


R_, T_ = O.ACT_RELU, O.ACT_TANH
# (ns, H, na, act, huber, double_dqn, weighted, tie): every observation width 1..4, head width 1..4, both hidden widths and both
# activations the TD loss + backward kernel accepts
DQN_GRAD_CASES = [
    pytest.param(4, 128, 2, R_, True, False, True, False, id="True-False-True"),
    pytest.param(4, 128, 2, R_, False, False, False, False, id="False-False-False"),
    pytest.param(4, 128, 2, R_, True, True, False, False, id="True-True-False"),
    pytest.param(1, 64, 4, R_, True, False, True, False, id="ns1-H64-na4-relu"),
    pytest.param(2, 128, 3, T_, True, True, False, False, id="ns2-H128-na3-tanh-double"),
    pytest.param(3, 64, 1, T_, False, False, False, False, id="ns3-H64-na1-tanh"),
    pytest.param(4, 128, 4, R_, False, False, True, False, id="ns4-H128-na4-relu"),
    pytest.param(4, 64, 2, T_, True, False, False, False, id="ns4-H64-na2-tanh"),
    pytest.param(1, 128, 3, T_, False, True, True, False, id="ns1-H128-na3-tanh-double"),
    pytest.param(3, 128, 4, R_, True, True, False, False, id="ns3-H128-na4-relu-double"),
    pytest.param(2, 64, 1, R_, True, False, False, False, id="ns2-H64-na1-relu"),
    # the online net's Q(s') of actions 2 and 3 tie exactly; the target net's differ: "first maximum wins" decides R
    pytest.param(2, 64, 3, R_, True, True, False, True, id="ns2-H64-na3-relu-double-tie"),
]


@pytest.mark.parametrize("ns,H,na,act,huber,double_dqn,weighted,tie", DQN_GRAD_CASES)
def test_dqn_grad_matches_autograd(ns, H, na, act, huber, double_dqn, weighted, tie):
    B = 400
    desc = O.ac_desc(ns, H, na, act)
    rng = np.random.default_rng(4)
    p = O.glorot_params(desc, 2, q_net=True); pt = O.glorot_params(desc, 3, q_net=True)
    if tie:
        p = Q.tie_actions(p, ns, H, na, 2, 3)
    s = rng.standard_normal((ns, B)).astype(np.float32); s2 = rng.standard_normal((ns, B)).astype(np.float32)
    a = rng.integers(1, na + 1, B).astype(np.int32); r = (3 * rng.standard_normal(B)).astype(np.float32)
    t = (rng.random(B) < 0.2).astype(np.uint8); w = rng.random(B).astype(np.float32) if weighted else None
    grad, loss, td = O.dqn_loss_grad(desc, p, pt, s, a, r, t, s2, w, 0.99, huber, double_dqn)
    g64, L64, e64 = Q.dqn_loss_grad(p, pt, ns, H, na, act, s, a, r, t, s2, w, 0.99, huber, double_dqn)
    assert loss == pytest.approx(L64, rel=2e-5)
    np.testing.assert_allclose(td, e64, rtol=1e-4, atol=1e-5)
    assert np.linalg.norm(grad - g64) <= 2e-5 * np.linalg.norm(g64)
    if tie:
        qo, qt = Q.q_values(p, ns, H, na, act, s2), Q.q_values(pt, ns, H, na, act, s2)
        assert np.array_equal(qo[:, 1], qo[:, 2]) and np.array_equal(*O.q_values(desc, p, s2)[1:])    # float64 and the oracle's float32
        # on these samples action 3's target value would move the TD error by far more than the tolerance: the rule is observable
        moved = (qo.argmax(1) == 1) & (t == 0) & (np.abs(qt[:, 2] - qt[:, 1]) > 1e-2)
        assert moved.mean() > 0.1


def test_adam_matches_torch_optim():
    rng = np.random.default_rng(0)
    n = 1000
    p0 = rng.standard_normal(n).astype(np.float32)
    p = p0.copy(); m = np.zeros(n, np.float32); v = np.zeros(n, np.float32); bt = np.array([0.9, 0.999], np.float32)
    P = torch.tensor(p0.copy(), requires_grad=True)
    opt = torch.optim.Adam([P], lr=1e-3, betas=(0.9, 0.999), eps=1e-8)
    for _ in range(20):
        g = rng.standard_normal(n).astype(np.float32)
        O.adam_step(p, g, m, v, bt)
        P.grad = torch.tensor(g); opt.step()
    np.testing.assert_allclose(p, P.detach().numpy(), rtol=0, atol=2e-6)


def test_clip_by_global_norm():
    g = np.array([3.0, 4.0, 0.0, 12.0], np.float32)  # norm 13
    c, gn = O.clip_by_global_norm(g, 0.5)
    assert gn == pytest.approx(13.0) and np.linalg.norm(c) == pytest.approx(0.5, rel=1e-6)
    c, gn = O.clip_by_global_norm(g, 20.0)  # clip_norm > gn: untouched
    assert np.array_equal(c, g) and gn == pytest.approx(13.0)


def test_normlogpdf_reference_vectors_and_target_sync():
    """RLCore/test/utils/distributions.jl:19-62: normlogpdf(10, 5, 4) ~ logpdf(Normal(10, 5), 4) and
    diagnormlogpdf([10, 1], [5, 6], [4, 3]) ~ logpdf(MvNormal([10, 1], Diagonal([25, 36])), [4, 3]) — Distributions.jl's
    values are the closed forms scipy evaluates."""
    from scipy import stats
    L = O.lib()
    f = O.C.c_float
    ref1 = stats.norm(10.0, 5.0).logpdf(4.0)
    assert L.orc_normlogpdf(f(10), f(5), f(4)) == pytest.approx(ref1, rel=2e-7)
    assert L.orc_normlogpdf1(f(10), f(5), f(4)) == pytest.approx(ref1, rel=2e-7)
    mu, sg, x = (np.array(v, np.float32) for v in ([10, 1], [5, 6], [4, 3]))
    ref2 = stats.multivariate_normal(mean=[10, 1], cov=np.diag([25.0, 36.0])).logpdf([4, 3])
    assert L.orc_diagnormlogpdf(O._p(mu), O._p(sg), O._p(x), 2) == pytest.approx(ref2, rel=3e-7)
    # test/utils/networks.jl:59-71 identity: a d = 1 diagnormlogpdf is the univariate form the Gaussian head evaluates, bit for bit
    rng = np.random.default_rng(0)
    for m, s_, xx in rng.standard_normal((200, 3)).astype(np.float32):
        s_ = np.float32(abs(s_) + 0.05)
        a = L.orc_diagnormlogpdf(O._p(np.array([m], np.float32)), O._p(np.array([s_], np.float32)), O._p(np.array([xx], np.float32)), 1)
        assert a == L.orc_normlogpdf1(f(m), f(s_), f(xx))
        assert a == pytest.approx(stats.norm(float(m), float(s_)).logpdf(float(xx)), rel=2e-5, abs=2e-6)
    t = np.arange(5, dtype=np.float32); m = np.ones(5, np.float32)
    L.orc_target_sync(O._p(t), O._p(m), 5, O.C.c_float(0.0))
    assert np.array_equal(t, m)                                  # rho = 0: hard copy
    t = np.zeros(5, np.float32)
    L.orc_target_sync(O._p(t), O._p(m), 5, O.C.c_float(0.75))
    np.testing.assert_allclose(t, 0.25)


def test_gumbel_max_sampling_distribution_and_logp():
    desc = O.ac_desc(4, 64, 2)
    p = O.glorot_params(desc, 5)
    n = 20000
    obs = np.tile(np.array([[0.3], [-0.2], [0.1], [0.5]], np.float32), (1, n))
    out = O.act_discrete(desc, p, obs, O.splitmix_states_fast(n, 99))
    probs = np.exp(out["logits"][:, 0] - np.logaddexp.reduce(out["logits"][:, 0]))
    freq = np.mean(out["action"] == 2)
    assert abs(freq - probs[1]) < 4 * np.sqrt(probs[1] * (1 - probs[1]) / n)
    lp = out["logits"] - np.logaddexp.reduce(out["logits"], axis=0)
    np.testing.assert_allclose(out["logp"], lp[out["action"] - 1, np.arange(n)], rtol=1e-5, atol=1e-6)


def test_perm_index_is_a_bijection():
    for n in (1, 2, 3, 7, 64, 1000, 4096, 5000, 8192):   # even and odd bit counts, with and without cycle walking
        for key in (0, 12345):
            assert sorted(O.perm_index(q, n, key) for q in range(n)) == list(range(n))
    a = [O.perm_index(q, 4096, 1) for q in range(4096)]
    b = [O.perm_index(q, 4096, 2) for q in range(4096)]
    assert a != b and a != list(range(4096))


def test_trajectory_length_and_iteration_semantics():
    """RLCore/test/policies/agent.jl:27-34: length 0 after the first state, 1 after the first
    transition; q_based_policy.jl:40-58: a sample is (state, next_state, action, reward, terminal)."""
    tr = O.OracleTraj(ns=2, lanes=1, cap=4)
    tr.push_state(np.array([[1.0], [1.0]], np.float32))
    assert len(tr) == 0
    for k in range(1, 7):  # wrap around a capacity-4 ring
        tr.push([k], [float(k)], [k % 3 == 0], np.full((2, 1), k + 1, np.float32))
        assert len(tr) == min(k, 4)
    got = set()
    slots = O.splitmix_states_fast(64, 5)
    b = tr.sample(slots, 64)
    for k in range(64):
        a = int(b["action"][k])
        assert 3 <= a <= 6                                     # oldest two were dropped
        assert b["state"][0, k] == a and b["next_state"][0, k] == a + 1 and b["reward"][k] == a and b["terminal"][k] == (a % 3 == 0)
        got.add(a)
    assert got == {3, 4, 5, 6}


def test_prioritized_sampling_follows_priorities():
    tr = O.OracleTraj(ns=1, lanes=4, cap=8, prioritized=True, default_priority=1.0)
    tr.push_state(np.zeros((1, 4), np.float32))
    for k in range(8):
        tr.push(np.arange(4) + 1, np.full(4, k, np.float32), np.zeros(4, np.uint8), np.full((1, 4), k + 1, np.float32))
    assert tr.total_priority() == pytest.approx(32.0)
    b = tr.sample(O.splitmix_states_fast(8, 1), 8, prioritized=True)
    tr.update_priority(b["key"][:1], np.array([1000.0], np.float32))
    b2 = tr.sample(O.splitmix_states_fast(4000, 2), 4000, prioritized=True, beta=0.5)
    frac = np.mean(b2["key"] == b["key"][0])
    assert frac > 0.9 and b2["weight"].max() == pytest.approx(1.0) and b2["weight"].min() > 0
