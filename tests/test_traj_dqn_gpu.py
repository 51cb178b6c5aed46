"""GPU parity of K3/K4 (trajectory ring push, uniform / prioritised sampling + gather, sum-tree
priority updates, from a tree held on chip to config 5's 2^21 leaves) and the DQN update (config 5's shape and the edges of the
TD loss + backward kernel's tiling) against the CPU oracle and float64 autograd."""
import numpy as np
import pytest

import oracle_lib as O
import q_ref as Q

pytestmark = pytest.mark.gpu


def fill_both(pkg, ctx, ns, lanes, cap, frames, prioritized, B, seed=0, default_priority=1.0, na=2):
    slots = O.splitmix_states_fast(B, 900 + seed)
    tr = pkg.Trajectory(ctx, ns, cap, lanes=lanes, batch_size=B, sampler_rng=slots, prioritized=prioritized, default_priority=default_priority)
    ref = O.OracleTraj(ns, lanes, cap, prioritized, default_priority)
    rng = np.random.default_rng(seed)
    obs = rng.standard_normal((ns, lanes)).astype(np.float32)
    tr.push_state(obs); ref.push_state(obs)
    assert len(tr) == len(ref) == 0
    for k in range(frames):
        a = rng.integers(1, na + 1, lanes).astype(np.int32); r = rng.standard_normal(lanes).astype(np.float32)
        t = (rng.random(lanes) < 0.1).astype(np.uint8); obs = rng.standard_normal((ns, lanes)).astype(np.float32)
        tr.push(a, r, t, obs); ref.push(a, r, t, obs)
        assert len(tr) == len(ref) == min(k + 1, cap)
    return tr, ref, slots


def assert_batches_equal(b, rb):
    for k in ("state", "action", "reward", "terminal", "next_state", "key"):
        assert np.array_equal(b[k], rb[k]), k


@pytest.mark.parametrize("lanes,cap,frames", [(1, 16, 40), (8, 32, 20), (64, 10, 35)])
def test_uniform_sampling_bit_exact(pkg, ctx, lanes, cap, frames):
    B = 256
    tr, ref, slots = fill_both(pkg, ctx, 4, lanes, cap, frames, False, B)
    s = slots.copy()
    for _ in range(3):
        b = tr.sample()
        rb = ref.sample(s, B)         # oracle advances `s` in place
        assert_batches_equal(b, rb)
    assert np.array_equal(tr.sampler_rng(), s)


def _priorities(rng, key):
    """log-uniform in 1e-6 .. 1e3, about 5 % exactly 0; the draws of one key in a batch carry one value"""
    prio = np.exp(rng.uniform(np.log(1e-6), np.log(1e3), key.size)).astype(np.float32)
    prio[rng.random(key.size) < 0.05] = 0.0
    _, first, inv = np.unique(key, return_index=True, return_inverse=True)
    return prio[first[inv]]


def _check_sum_tree(tr, keys=None):
    """the exported tree bit for bit: every internal node is float32(left + right) of its children, the leaf of every entry that is
    not sampleable (and every padding leaf) is 0; `keys` (drawn) have a positive leaf and the sampleable flag"""
    st = tr.export_state()
    tree, flag = st["tree"], st["flag"]
    L = tree.size // 2
    assert np.array_equal(tree[1:L], tree[2::2] + tree[3::2])
    leaves = tree[L:]
    sampleable = np.zeros(L, bool)
    sampleable[:flag.size] = (flag & 2) != 0
    assert not leaves[~sampleable].any()
    if keys is not None:
        assert (leaves[keys] > 0).all() and sampleable[keys].all()
    return leaves


C5 = (4096, 256, 4096)   # lanes, capacity, batch of bench.py --config c5


# The sum tree has L = 2^ceil(log2(lanes (cap + 1))) leaves; both tree kernels keep its top 4096 nodes on chip and walk the levels
# below them in global memory.
@pytest.mark.parametrize("lanes,cap,frames,B", [
    pytest.param(1, 64, 100, 512, id="1-64-100"),
    pytest.param(16, 32, 50, 512, id="16-32-50"),
    pytest.param(31, 65, 80, 512, id="31-65-80-512"),              # 2046 slots, L = 2^11: every level on chip
    pytest.param(128, 63, 80, 512, id="128-63-80-512"),            # 8192 slots = L: one level in global memory, no padding leaves
    pytest.param(1000, 100, 110, 2048, id="1000-100-110-2048"),    # 101 000 slots, L = 2^17: padding leaves
    pytest.param(4096, 255, 260, 4096, id="4096-255-260-4096"),    # 2^20 slots = L
    pytest.param(*C5[:2], 260, C5[2], id="4096-256-260-4096"),     # 1 052 672 slots, L = 2^21, + one DQN update
])
def test_prioritized_sampling_and_updates_bit_exact(pkg, ctx, lanes, cap, frames, B):
    tr, ref, slots = fill_both(pkg, ctx, 4, lanes, cap, frames, True, B, seed=3, default_priority=2.0)
    assert tr.total_priority() == ref.total_priority() == 2.0 * cap * lanes
    s = slots.copy()
    rng = np.random.default_rng(0)
    obs = np.zeros((4, lanes), np.float32)
    for it in range(4):
        b = tr.sample(beta=0.5)
        rb = ref.sample(s, B, prioritized=True, beta=0.5)
        assert_batches_equal(b, rb)
        assert np.array_equal(b["priority"], rb["priority"])
        np.testing.assert_allclose(b["weight"], rb["weight"], rtol=2e-6)
        _check_sum_tree(tr, b["key"])
        prio = _priorities(rng, b["key"])
        tr.update_priority(prio); ref.update_priority(b["key"], prio)
        assert tr.total_priority() == ref.total_priority()
        _check_sum_tree(tr)
        # pushing after priority updates keeps both trees in step (wrap-around drops old leaves, new entries get the default)
        for _ in range(5):
            tr.push(np.ones(lanes, np.int32), np.zeros(lanes, np.float32), np.zeros(lanes, np.uint8), obs)
            ref.push(np.ones(lanes, np.int32), np.zeros(lanes, np.float32), np.zeros(lanes, np.uint8), obs)
            assert tr.total_priority() == ref.total_priority()
    if (lanes, cap, B) == C5:
        _dqn_priority_write_back(pkg, ctx, tr, ref, s, B)
    tr.close()


def _dqn_priority_write_back(pkg, ctx, tr, ref, s, B):
    """one DQNLearner.update with the Q-network of config c5 (4-128-128-2): the leaves it writes back are (|td| + 1e-6)^0.6 of the
    device's TD errors (device powf: within 2 ulp of NumPy's); with the oracle's leaves set to them the next draw is bit-exact"""
    desc = O.ac_desc(4, 128, 2)
    net = pkg.Network(ctx, 4, 128, 2, O.glorot_params(desc, 2, q_net=True), kind=pkg.KIND_Q)
    learner = pkg.DQNLearner(ctx, net, tr, pkg.dqn_config(per_beta=0.4, per_alpha=0.6, per_eps=1e-6))
    learner.update()
    key = tr.batch()["key"]
    assert np.array_equal(key, ref.sample(s, B, prioritized=True, beta=0.4)["key"])
    want = ((np.abs(learner.last_td()) + np.float32(1e-6)) ** np.float32(0.6)).astype(np.float32)
    got = _check_sum_tree(tr, key)[key]
    ulps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32))
    _, inv = np.unique(key, return_inverse=True)
    best = np.full(inv.max() + 1, np.iinfo(np.int64).max)
    np.minimum.at(best, inv, ulps)                              # a key drawn twice holds the value of one of its draws
    assert best.max() <= 2, best.max()
    ref.update_priority(key, got)
    assert tr.total_priority() == ref.total_priority()
    b, rb = tr.sample(beta=0.4), ref.sample(s, B, prioritized=True, beta=0.4)
    assert_batches_equal(b, rb)
    assert np.array_equal(b["priority"], rb["priority"])
    np.testing.assert_allclose(b["weight"], rb["weight"], rtol=2e-6)
    net.close()


def _drive(pkg, ctx, env, tr, ref, steps, hook):
    """random-policy steps with trajectory pushes the way learners.Agent does them; the oracle ring gets the same calls"""
    for _ in range(steps):
        if not env.auto_reset:
            env.reset_(is_force=False)                                        # soft reset of the finished sub-envs ...
            tr.push_env(env, first_state_only=2); ref.push_episode_start(env.state(), pending_only=True)   # ... whose episodes start here
        env.act_random_()
        tr.push_env(env)
        ref.push(env.last_action(), env.reward(), env.flags(), env.state())
        hook.push("PostActStage", None, env)


@pytest.mark.parametrize("auto_reset", [True, False])
def test_episodes_buffer_length_identity_per_lane(pkg, ctx, auto_reset):
    """RLCore/test/core/base.jl:20 per lane: length(container) == steps + episodes - 1 — every episode's first state is a frame of its
    own and the entry straddling two episodes is stored but never sampleable; the sampleable entries are exactly the steps.
    (With the in-kernel auto-reset an episode that ends on the very last step has already started its successor: that frame counts.)"""
    n, steps, B = 96, 70, 2048
    env = pkg.B200VecEnv(ctx, "CartPole", n, O.splitmix_states_fast(n, 5), auto_reset=auto_reset)
    slots = O.splitmix_states_fast(B, 6)
    tr = pkg.Trajectory(ctx, 4, 200, lanes=n, batch_size=B, sampler_rng=slots)
    ref = O.OracleTraj(4, n, 200)
    hook = pkg.BatchStepsPerEpisode(n)
    env.reset_(is_force=True)
    tr.push_env(env, first_state_only=True); ref.push_state(env.state())     # PreEpisodeStage after the forced reset
    assert np.array_equal(tr.lane_lengths(), np.zeros(n, np.int64))           # test/policies/agent.jl:30 (0 after the first state)
    _drive(pkg, ctx, env, tr, ref, steps, hook)
    finished = np.array([len(s) for s in hook[()]])
    assert finished.sum() > n                                                 # CartPole under the random policy: ~3 episodes per lane
    last_step_terminal = env.is_terminated()
    started = 1 + finished - (0 if auto_reset else last_step_terminal.astype(int))   # soft reset: the successor of a just-finished episode has not begun
    lengths = tr.lane_lengths()
    assert np.array_equal(lengths, steps + started - 1)
    assert np.array_equal(lengths, ref.lane_lengths())
    assert tr.n_sampleable() == ref.n_sampleable() == steps * n               # every step is sampleable, no straddling entry is
    s = slots.copy()
    b = tr.sample(); rb = ref.sample(s, B)
    assert_batches_equal(b, rb) and np.array_equal(tr.sampler_rng(), s)
    # a sampled terminal transition really ends an episode; a non-terminal one is followed by its true successor state
    term = b["terminal"].astype(bool)
    assert term.any() and (~term).any()
    # forced reset in the middle (ResetAfterNSteps / re-entering run): an episode-start frame for every lane, nothing else changes
    env.reset_(is_force=True)
    tr.push_env(env, first_state_only=True); ref.push_state(env.state())
    assert np.array_equal(tr.lane_lengths(), lengths + 1) and tr.n_sampleable() == steps * n
    _drive(pkg, ctx, env, tr, ref, 5, hook)
    assert tr.n_sampleable() == ref.n_sampleable() == (steps + 5) * n
    assert_batches_equal(tr.sample(), ref.sample(s, B))
    tr.close(); env.close()


def test_single_lane_matches_agent_jl_lengths_and_wraps(pkg, ctx):
    """test/policies/agent.jl:27-34 (length 0 after the first state, 1 after the first transition) with lanes = 1, then far past the
    capacity: the ring keeps the newest cap entries, overwritten entries leave the sampleable set (and the sum tree)."""
    cap, B = 16, 64
    slots = O.splitmix_states_fast(B, 1)
    tr = pkg.Trajectory(ctx, 4, cap, lanes=1, batch_size=B, sampler_rng=slots, prioritized=True, default_priority=1.5)
    ref = O.OracleTraj(4, 1, cap, True, 1.5)
    rng = np.random.default_rng(0)
    obs = rng.standard_normal((4, 1)).astype(np.float32)
    tr.push_state(obs); ref.push_state(obs)
    assert len(tr) == 0
    for k in range(60):
        term = np.uint8(1 if k % 7 == 6 else 0)
        nxt = rng.standard_normal((4, 1)).astype(np.float32)
        a, r, t = np.array([1 + k % 2], np.int32), np.array([k], np.float32), np.array([term], np.uint8)
        tr.push(a, r, t, nxt); ref.push(a, r, t, nxt)
        if k == 0:
            assert len(tr) == 1
        if term:                                                    # PreEpisodeStage of the next episode (the reference's reset + push)
            s0 = rng.standard_normal((4, 1)).astype(np.float32)
            tr.push_episode_start(s0, pending_only=True); ref.push_episode_start(s0, pending_only=True)
        assert len(tr) == len(ref) <= cap and tr.n_sampleable() == ref.n_sampleable()
        assert tr.total_priority() == ref.total_priority() == 1.5 * tr.n_sampleable()
    s = slots.copy()
    b = tr.sample(beta=0.4); rb = ref.sample(s, B, prioritized=True, beta=0.4)
    assert_batches_equal(b, rb) and np.array_equal(b["priority"], rb["priority"])
    assert set(b["reward"].astype(int)) <= set(range(60 - cap - 3, 60))     # only recent transitions survive
    tr.close()


def test_push_env_matches_host_push(pkg, ctx):
    n = 128
    env = pkg.B200VecEnv(ctx, "CartPole", n, O.splitmix_states_fast(n, 12), auto_reset=True)
    slots = O.splitmix_states_fast(64, 1)
    tr = pkg.Trajectory(ctx, 4, 50, lanes=n, batch_size=64, sampler_rng=slots)
    ref = O.OracleTraj(4, n, 50)
    env.reset_(is_force=True)
    tr.push_env(env, first_state_only=True); ref.push_state(env.state())
    for _ in range(30):
        env.act_random_()
        tr.push_env(env)
        ref.push(env.last_action(), env.reward(), env.flags(), env.state())     # flags: bit1 = the env has already auto-reset
    assert np.array_equal(tr.lane_lengths(), ref.lane_lengths()) and tr.n_sampleable() == ref.n_sampleable() == 30 * n
    s = slots.copy()
    assert_batches_equal(tr.sample(), ref.sample(s, 64))


def _update_case(id_, **kw):
    c = dict(ns=4, H=128, na=2, act=O.ACT_RELU, B=1024, huber=True, double_dqn=False, prioritized=False, n_step=1, tie=False, teacher=True, seed=2)
    c.update(kw)
    return pytest.param(c, id=id_)


# The first three are config 5's Q-net 4 -> H -> H -> 2 at B = 1024 (a multiple of both tiles: 128 samples at H = 64, 64 at H = 128)
# against the oracle's own 4-update chain.  The rest run 3 updates, each from the device's parameters, Adam state and target
# (teacher forcing), at the edges of the kernel's tiling: B = "wave+k" is one tile for every CTA of the grid, then k samples more.
UPDATE_CASES = [
    _update_case("128-True-False-True", prioritized=True, teacher=False),
    _update_case("64-False-False-False", H=64, huber=False, teacher=False),
    _update_case("128-True-True-True", double_dqn=True, prioritized=True, teacher=False),
    _update_case("ns1-H64-na4-relu-B1000-per", ns=1, H=64, na=4, B=1000, prioritized=True),                  # last tile: 104 of 128
    _update_case("ns2-H128-na3-tanh-B1000-double", ns=2, na=3, act=O.ACT_TANH, B=1000, double_dqn=True),     # last tile: 40 of 64
    _update_case("ns3-H64-na1-tanh-B1", ns=3, H=64, na=1, act=O.ACT_TANH, B=1, huber=False),                 # one sample, one CTA
    _update_case("ns4-H128-na4-relu-per-wave+37", na=4, B="wave+37", huber=False, prioritized=True),
    _update_case("ns4-H64-na2-tanh-n3-wave+129", H=64, act=O.ACT_TANH, B="wave+129", n_step=3),
    # the online net's Q(s') of actions 2 and 3 tie exactly (same head row and bias), the target net's differ: first maximum wins
    _update_case("ns2-H64-na3-relu-double-tie", ns=2, H=64, na=3, B=1000, double_dqn=True, tie=True, seed=4),   # the tie wins ~45 %
]


def _assert_grad_blocks(gdev, g64, scale, ns, H, na):
    """the device's clipped gradient against float64 autograd times the device's clip factor, per parameter block: relative L2 error
    1e-5 of the block, or of the whole gradient for a block whose norm is below 1e-3 of it.  Measured on an H100 80GB HBM3 (700 W): at most
    6.2e-7 for B >= 1000, 3.1e-6 for the single sample (its TD error is 0.045, so the float32 rounding of R - Q is 3e-6 of it)."""
    ref = g64 * scale
    whole = np.linalg.norm(ref)
    err = {}
    for name, sl in Q.blocks(ns, H, na):
        nb = np.linalg.norm(ref[sl])
        err[name] = np.linalg.norm(gdev[sl] - ref[sl]) / (nb if nb >= 1e-3 * whole else whole)
    assert max(err.values()) <= 1e-5, err


def _assert_preconditions(c, pd, b, e64):
    """the batch reaches both Huber branches and has terminals; double DQN: no rounding near-tie of the online Q(s') decides R"""
    ns, H, na, act = c["ns"], c["H"], c["na"], c["act"]
    B = e64.size
    if B >= 1000:
        assert (np.abs(e64) < 1).mean() >= 0.1 and (np.abs(e64) >= 1).mean() >= 0.1
        assert 0.05 <= b["terminal"].mean() <= 0.3
    if c["double_dqn"]:
        qo = Q.q_values(pd, ns, H, na, act, b["next_state"])
        if c["tie"]:
            assert np.array_equal(qo[:, 1], qo[:, 2]) and (qo.argmax(1) == 1).mean() >= 0.1
            qo = qo[:, :2]
        top = np.sort(qo, axis=1)
        assert (top[:, -1] - top[:, -2] > 1e-4 * (1 + np.abs(top[:, -1]))).all()


@pytest.mark.parametrize("case", UPDATE_CASES)
def test_dqn_update_parity(pkg, ctx, case):
    """Sample + TD update + priority write-back of a Q-net ns -> H -> H -> na against the oracle's clip + Adam step, and the
    device's loss, TD errors and gradient blocks against float64 autograd at the device's own parameters."""
    c = case
    ns, H, na, act, B, lanes = c["ns"], c["H"], c["na"], c["act"], c["B"], 32
    huber, double_dqn, prioritized, n_step = c["huber"], c["double_dqn"], c["prioritized"], c["n_step"]
    if isinstance(B, str):
        import torch
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        ctas, tm = (2 * sms, 128) if H == 64 else (sms, 64)      # nn_dqn_max_partials, Cfg<H>::TM
        B = ctas * tm + int(B.split("+")[1])
        assert B > ctas * tm                                    # some CTAs run a second tile
    tr, ref, slots = fill_both(pkg, ctx, ns, lanes, 64, 80, prioritized, B, seed=5, na=na)
    if n_step > 1:
        tr.set_nstep(n_step, 0.99)
    desc = O.ac_desc(ns, H, na, act)
    p0 = O.glorot_params(desc, c["seed"], q_net=True) + 0.05 * np.random.default_rng(1).standard_normal(O.q_nparams(desc)).astype(np.float32)
    pt = p0 * np.float32(0.9)
    if c["tie"]:
        p0 = Q.tie_actions(p0, ns, H, na, 2, 3)
    net = pkg.Network(ctx, ns, H, na, p0, act=act, kind=pkg.KIND_Q)
    net.set(pkg.learners.NET_TARGET, pt)
    cfg = pkg.dqn_config(huber=huber, double_dqn=double_dqn, target_update_freq=3, max_grad_norm=10.0, per_beta=0.4)
    learner = pkg.DQNLearner(ctx, net, tr, cfg)
    p = p0.copy()
    m = np.zeros_like(p); v = np.zeros_like(p); bt = np.array([0.9, 0.999], np.float32)
    q_ref = O.q_values(desc, p, np.asfortranarray(np.random.default_rng(3).standard_normal((ns, 100)).astype(np.float32)))
    np.testing.assert_allclose(net.values(np.random.default_rng(3).standard_normal((ns, 100)).astype(np.float32)), q_ref, rtol=1e-5, atol=2e-6)
    R = pkg.learners
    for it in range(3 if c["teacher"] else 4):
        if c["tie"]:                                         # Adam's step unties the rows: tie them again
            net.set(R.NET_PARAMS, Q.tie_actions(net.get(), ns, H, na, 2, 3))
        pd, ptd = net.get(), net.get(R.NET_TARGET)
        if c["teacher"]:
            p, pt, m, v, bt = pd.copy(), ptd, net.get(R.NET_M), net.get(R.NET_V), net.get(R.NET_BETA_T)
        stats = learner.update(want_stats=True)
        b = tr.batch()                                       # the batch the update used (teacher forcing for the oracle)
        w = b["weight"] if prioritized else None
        g, loss, td = Q.oracle_dqn_loss_grad(desc, p, pt, b, w, huber, double_dqn)
        gc, gn = O.clip_by_global_norm(g.astype(np.float32), 10.0)
        O.adam_step(p, gc, m, v, bt)
        tol = 2e-5 * (1 + it)
        assert stats["loss"] == pytest.approx(loss, rel=tol)
        assert stats["grad_norm"] == pytest.approx(gn, rel=10 * tol)
        dtd = learner.last_td()
        np.testing.assert_allclose(dtd, td, rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(net.get(), p, rtol=0, atol=5e-6)
        g64, loss64, e64 = Q.dqn_loss_grad(pd, ptd, ns, H, na, act, b["state"], b["action"], b["reward"], b["terminal"], b["next_state"], w,
                                           0.99, huber, double_dqn, b["discount"] if n_step > 1 else None)
        if c["teacher"]:
            _assert_preconditions(c, pd, b, e64)
        assert stats["loss"] == pytest.approx(loss64, rel=1e-5)
        np.testing.assert_allclose(dtd, e64, rtol=1e-5, atol=2e-6)
        gnd = np.float32(stats["grad_norm"])
        scale = np.float32(10.0) / max(np.float32(10.0), gnd) if gnd >= 10.0 else 1.0    # optim::clip_scale
        _assert_grad_blocks(net.get(R.NET_GRAD), g64, scale, ns, H, na)
        if prioritized:
            newp = (np.abs(td) + np.float32(1e-6)) ** np.float32(0.6)
            ref.update_priority(b["key"], newp.astype(np.float32))
            assert tr.total_priority() == pytest.approx(ref.total_priority(), rel=1e-5)
        if (it + 1) % 3 == 0:
            pt = p.copy()                                    # hard target sync (rho = 0)
            np.testing.assert_allclose(net.get(pkg.learners.NET_TARGET), net.get(), rtol=0, atol=0)
        else:
            assert not np.array_equal(net.get(pkg.learners.NET_TARGET), net.get())


def test_q_act_epsilon_greedy(pkg, ctx):
    import ctypes as C
    ns, na, n = 4, 2, 20000
    desc = O.ac_desc(ns, 128, na)
    p = O.glorot_params(desc, 4, q_net=True)
    net = pkg.Network(ctx, ns, 128, na, p, kind=pkg.KIND_Q)
    obs = np.asfortranarray(np.random.default_rng(0).standard_normal((ns, n)).astype(np.float32))
    d_obs = ctx.malloc(obs.nbytes); ctx.h2d(d_obs, obs)
    d_rng = ctx.malloc(n * 32); ctx.h2d(d_rng, O.splitmix_states_fast(n, 8))
    d_act = ctx.malloc(n * 4)
    greedy = O.q_values(desc, p, obs).argmax(0) + 1
    for eps, lo, hi in ((0.0, 1.0, 1.0), (0.5, 0.70, 0.80)):
        pkg._lib.check(ctx.lib.b200rl_net_q_act(net.h, C.c_void_p(d_obs), n, C.c_void_p(d_rng), C.c_float(eps), C.c_void_p(d_act)))
        a = np.empty(n, np.int32); ctx.d2h(a, d_act)
        agree = np.mean(a == greedy)
        assert lo - 0.01 <= agree <= hi + 0.01 and a.min() >= 1 and a.max() <= na
    for d in (d_obs, d_rng, d_act):
        ctx.free(d)
