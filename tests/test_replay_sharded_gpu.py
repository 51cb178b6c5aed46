"""GPU tests of the sharded DQN replay loop (DESIGN.md §3): two ranks in ONE process (two ctx on cuda:0, driven by two threads,
peer exchange, not exclusive) against one rank over the union of their envs, the stage protocol and the oracle.

(1) A window with the threshold past its end (no update) equals one rank over the 2N-lane union bit for bit: env fields, rank
    r's lanes of the ring and sum-tree leaves, explorer streams and the global explorer step.
(2) On each rank the device loop (run_replay) equals the stage protocol driven in the same two threads, bit for bit; the
    replicas end bit-identical.  (Ranks sharing a device launch the update units eagerly; the graph replay is what an unsharded
    run and one rank per GPU use.)
(3) One sharded update equals the oracle's gradient over the union of both ranks' batches, then clip and Adam.
(4) A mid-run per-rank checkpoint restored into other seeds continues bit for bit on both ranks.
(5) evaluate_explore on the shards equals one rank over the union.
(6) Mismatched N, n_steps, controller or explorer step: both ranks refuse, return, and touch nothing.
The real two-process / two-GPU wiring (CUDA IPC handles) is exercised by bench_replay_sharded.py.

Ranks that share a device in one process must not allocate device memory or set a kernel attribute for the first time while the
peer rank's kernel waits inside an exchange (both serialise with running kernels): every test creates its handles, grows the ctx
scratch and launches each kernel once (an unsharded run of the same configuration) before the two threads start."""
import ctypes as C
import gc
import threading

import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu


def _in_threads(fns):
    errs = []

    def wrap(f):
        try:
            f()
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=wrap, args=(f,)) for f in fns]
    [t.start() for t in th]
    [t.join(timeout=120) for t in th]
    assert not any(t.is_alive() for t in th), "a rank is stuck in the exchange"
    if errs:
        raise errs[0]


def _two_ranks(pkg):
    L = pkg._lib
    ctxs = [pkg.Context(0), pkg.Context(0)]
    regions = (C.c_void_p * 2)()
    for r, ctx in enumerate(ctxs):
        L.check(ctx.lib.b200rl_comm_init(ctx.h, 2, r, None))        # no NCCL: peer exchange only
        p = C.c_void_p()
        L.check(ctx.lib.b200rl_comm_p2p_export(ctx.h, None, C.byref(p)))
        regions[r] = p
    for ctx in ctxs:
        L.check(ctx.lib.b200rl_comm_p2p_attach(ctx.h, regions))
    return ctxs


@pytest.fixture(scope="module")
def pairs(pkg):
    """two independent pairs of ranks (each its own exchange) and one unsharded ctx"""
    p = [_two_ranks(pkg), _two_ranks(pkg)]
    one = pkg.Context(0)
    yield p, one
    for ctxs in p:
        for c in ctxs:
            c.close()
    one.close()


_NA = {"CartPole": 2, "MountainCar": 3}


def _explorer(pkg, name, total, steps):
    if name in ("linear", "exp", "break_tie"):   # linear: the decay ends inside the window
        return pkg.EpsilonGreedyExplorer(0.05, kind="exp" if name == "exp" else "linear", eps_init=1.0, warmup_steps=total,
                                         decay_steps=total * max(steps // 2, 1), is_break_tie=name == "break_tie")
    if name == "speedy":
        return pkg.EpsilonSpeedyExplorer(2.0 / (total * steps))
    return {"weighted": pkg.WeightedSoftmaxExplorer, "gumbel": pkg.GumbelSoftmaxExplorer, "greedy": pkg.GreedyExplorer}[name]()


def _agent(pkg, ctx, n_total, case, seed=100, explorer=None, steps=10):
    sh = pkg.sharding
    env_kind, hidden, act = case.get("env", "CartPole"), case.get("hidden", 64), case.get("act", 0)
    ns, na = 4 if env_kind == "CartPole" else 2, _NA[env_kind]
    q0 = O.glorot_params(O.ac_desc(ns, hidden, na, act), 7, q_net=True)
    kind = pkg.KIND_DUELING if case.get("dueling") else pkg.KIND_Q
    if kind == pkg.KIND_DUELING:
        q0 = np.random.default_rng(7).uniform(-0.3, 0.3, pkg.Network.count_params(ctx, ns, hidden, na, act=act, kind=kind)).astype(np.float32)
    cfg = pkg.dqn_config(huber=case.get("huber", True), double_dqn=case.get("double_dqn", False),
                         target_update_freq=case.get("target_freq", 3), max_grad_norm=case.get("max_grad_norm", 0.0))
    ex = explorer if explorer is not None else _explorer(pkg, case.get("explorer", "linear"), n_total, steps)
    return sh.dqn_rank_agent(ctx, env_kind, n_total, seed, q0, hidden, na, cfg, ex, case.get("cap", 8), case.get("B", 64), act=act,
                             kind=kind, prioritized=case.get("prioritized", True), n_step=case.get("n_step", 1),
                             ratio=case.get("ratio", 1.0), threshold=case.get("threshold", 1000))


def _close(s):
    s["agent"].close()
    for k in ("policy", "traj", "net", "env"):
        s[k].close()


def _state(pkg, s):
    ck = pkg.checkpoint.checkpoint_replay(s["env"], s["net"], s["agent"])
    return {k: np.array(v, copy=True) for k, v in ck.items()}


def _assert_same(a, b, skip=()):
    assert sorted(a) == sorted(b)
    for k in a:
        if k not in skip:
            assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


def _prepare(ranks, fusable=True):
    """the serial set-up before two ranks run in threads: the replay handles, the ctx scratch past every launch's need (and no
    garbage left whose finaliser could free device memory inside a thread)"""
    gc.collect()
    for s in ranks:
        s["agent"].fusable = fusable
        s["net"].values(np.zeros((s["net"].n_in, 8192), np.float32))
        if fusable:
            assert s["agent"].replay_supported(s["env"])


def _warm(pkg, one, n_total, case):
    """every kernel of the configuration launched once, unsharded, fused and staged (function attributes set)"""
    for fusable in (True, False):
        w = _agent(pkg, one, n_total, dict(case, threshold=1), seed=5, steps=4)
        w["agent"].fusable = fusable
        pkg.run(w["agent"], w["env"], pkg.StopAfterNSteps(4), pkg.EmptyHook())
        pkg.learners.evaluate(w["policy"], w["env"], 2)
        _close(w)


def _run_pair(pkg, ranks, steps, fusable=True):
    _prepare(ranks, fusable)
    _in_threads([lambda s=s: pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(steps), pkg.EmptyHook()) for s in ranks])


def _lane_view(ck, r, n, world, ns):
    """rank r's share of a checkpoint over world * n lanes (env columns, ring lanes, sum-tree leaves)"""
    lo, hi, L = r * n, (r + 1) * n, world * n
    out = {}
    for k, v in ck.items():
        v = np.asarray(v)
        if k in ("env/state", "env/obs"):
            out[k] = v[:, lo:hi]
        elif k in ("env/reward", "env/flags", "env/t", "env/action", "env/episode_return", "env/rng", "policy/explorer_rng",
                   "traj/head", "traj/count", "traj/pending"):
            out[k] = v[lo:hi]
        elif k == "traj/state":
            out[k] = v.reshape(-1, L, ns)[:, lo:hi]
        elif k in ("traj/action", "traj/reward", "traj/flag"):
            out[k] = v.reshape(-1, L)[:, lo:hi]
        elif k == "traj/tree":
            leaves = v[v.size // 2:]
            F = ck["traj/action"].size // L
            out[k] = leaves[:F * L].reshape(F, L)[:, lo:hi]
    return out


COLLECT = [
    dict(env="CartPole", hidden=64, explorer="linear", n=127),
    dict(env="CartPole", hidden=64, explorer="exp", n=1),
    dict(env="MountainCar", hidden=64, explorer="break_tie", n=127, act=1),
    dict(env="CartPole", hidden=64, explorer="speedy", n=4096),
    dict(env="MountainCar", hidden=64, explorer="weighted", n=127, prioritized=False),
    dict(env="CartPole", hidden=64, explorer="gumbel", n=127),
    dict(env="CartPole", hidden=64, explorer="greedy", n=127),
    dict(env="CartPole", hidden=128, explorer="linear", n=127, act=1),          # staged collect
    dict(env="MountainCar", hidden=128, explorer="gumbel", n=1),
    dict(env="CartPole", hidden=64, explorer="linear", n=127, tc_off=True),    # tensor cores off: staged collect
]


@pytest.mark.parametrize("case", COLLECT, ids=[f"{c['env']}-H{c['hidden']}-{c['explorer']}-N{c['n']}{'-notc' if c.get('tc_off') else ''}"
                                               for c in COLLECT])
def test_collect_window_equals_one_rank_over_the_union(pkg, pairs, case):
    (ctxs, _), one = pairs
    n, steps = case["n"], 9
    lib = ctxs[0].lib
    if case.get("tc_off"):
        lib.b200rl_set_tensor_cores(0)
    try:
        ranks = [_agent(pkg, c, 2 * n, case, steps=steps) for c in ctxs]
        union = _agent(pkg, one, 2 * n, case, steps=steps)
        pkg.run(union["agent"], union["env"], pkg.StopAfterNSteps(steps), pkg.EmptyHook())    # (first: launches every kernel)
        _run_pair(pkg, ranks, steps)
    finally:
        lib.b200rl_set_tensor_cores(1)
    assert union["agent"]._replay is not None and all(s["agent"]._replay is not None for s in ranks)
    ns = 4 if case["env"] == "CartPole" else 2
    cu = _state(pkg, union)
    for r, s in enumerate(ranks):
        cr = _state(pkg, s)
        want = _lane_view(cu, r, n, 2, ns)
        _assert_same(_lane_view(cr, 0, n, 1, ns), want)
        assert np.array_equal(cr["policy/explorer_step"], cu["policy/explorer_step"])           # the global explorer step
        assert s["net"].step_count() == 0
    if hasattr(union["policy"].explorer, "step"):
        assert union["policy"].explorer.step == 1 + steps * 2 * n
    assert sum(s["traj"].n_sampleable() for s in ranks) == union["traj"].n_sampleable()
    st = [_state(pkg, s)["env/episode_stats"] for s in ranks]
    assert np.array_equal((st[0] + st[1])[[0, 2]], cu["env/episode_stats"][[0, 2]])
    for s in ranks + [union]:
        _close(s)


LOOP = [
    dict(ratio=1.0, threshold=2, prioritized=True, target_freq=3),
    dict(ratio=0.25, threshold=2, prioritized=False, explorer="exp", target_freq=2),
    dict(ratio=1.0, threshold=3, n_step=3, dueling=True, explorer="gumbel", target_freq=4),
    dict(ratio=1.0, threshold=2, hidden=128, act=1, double_dqn=True, huber=False, max_grad_norm=1.0, target_freq=3),
]


@pytest.mark.parametrize("case", LOOP, ids=[f"r{c['ratio']}-{'per' if c.get('prioritized', True) else 'uni'}-n{c.get('n_step', 1)}"
                                            f"{'-duel' if c.get('dueling') else ''}-H{c.get('hidden', 64)}" for c in LOOP])
def test_device_loop_equals_stage_protocol_on_every_rank(pkg, pairs, case):
    (fast_ctx, stage_ctx), one = pairs
    n, steps = 127, 14
    _warm(pkg, one, 2 * n, case)
    fast = [_agent(pkg, c, 2 * n, case, steps=steps) for c in fast_ctx]
    stage = [_agent(pkg, c, 2 * n, case, steps=steps) for c in stage_ctx]
    _run_pair(pkg, fast, steps)
    _run_pair(pkg, stage, steps, fusable=False)
    _run_pair(pkg, fast, 5)                                                  # re-entry: graphs warm
    _run_pair(pkg, stage, 5, fusable=False)
    assert all(s["agent"]._replay is not None for s in fast) and all(s["agent"]._replay is None for s in stage)
    ck = [[_state(pkg, s) for s in p] for p in (fast, stage)]
    for r in range(2):
        _assert_same(ck[0][r], ck[1][r])
    for k in ("net/params", "net/adam_m", "net/adam_v", "net/beta_t", "net/target", "net/step", "policy/explorer_step"):
        assert np.array_equal(ck[0][0][k], ck[0][1][k]), k                   # replicas bit-identical
    # (ranks sharing a device launch the units eagerly — a graph upload may wait for the peer's exchange; one rank per device
    # replays them as graphs, bench_replay_sharded.py)
    assert fast[0]["net"].step_count() > 3 and not any(s["agent"].graph_active() for s in fast)
    assert not np.array_equal(ck[0][0]["traj/state"], ck[0][1]["traj/state"])
    for s in fast + stage:
        _close(s)


@pytest.mark.parametrize("huber,double_dqn,prioritized", [(True, False, True), (False, False, False), (True, True, True)])
def test_one_sharded_update_matches_the_oracle(pkg, pairs, huber, double_dqn, prioritized):
    (ctxs, _), one = pairs
    n, threshold, hidden = 127, 6, 64
    case = dict(ratio=1.0, threshold=threshold, huber=huber, double_dqn=double_dqn, prioritized=prioritized, max_grad_norm=10.0, B=256)
    _warm(pkg, one, 2 * n, case)
    ranks = [_agent(pkg, c, 2 * n, case, steps=threshold) for c in ctxs]
    p0 = ranks[0]["net"].get().copy()
    stats = [None, None]

    def go(r):
        stats[r] = ranks[r]["agent"].run_replay(ranks[r]["env"], threshold, want_stats=True)   # exactly one update, at the last step
    ranks[0]["env"].reset_(is_force=True); ranks[1]["env"].reset_(is_force=True)
    for s in ranks:
        s["traj"].push_env(s["env"], first_state_only=True)
    _prepare(ranks)
    _in_threads([lambda r=r: go(r) for r in range(2)])
    assert ranks[0]["net"].step_count() == ranks[1]["net"].step_count() == 1
    desc = O.ac_desc(4, hidden, 2)
    g_sum, loss_sum = None, 0.0
    for s in ranks:
        b = s["traj"].batch()
        w = b["weight"] if prioritized else None
        g, loss, _ = O.dqn_loss_grad(desc, p0, p0, b["state"], b["action"], b["reward"], b["terminal"], b["next_state"], w, 0.99, huber, double_dqn)
        g_sum = g if g_sum is None else g_sum + g
        loss_sum += loss
    g = (g_sum / 2).astype(np.float32)                                        # the mean over the global batch of 2 B
    gc, gn = O.clip_by_global_norm(g, 10.0)
    p, m, v, bt = p0.copy(), np.zeros_like(p0), np.zeros_like(p0), np.array([0.9, 0.999], np.float32)
    O.adam_step(p, gc, m, v, bt)
    for r, s in enumerate(ranks):
        np.testing.assert_allclose(s["net"].get(), p, rtol=0, atol=5e-6)
        assert stats[r]["loss"] == pytest.approx(loss_sum / 2, rel=2e-5)      # global (all-reduced)
        assert stats[r]["grad_norm"] == pytest.approx(gn, rel=2e-4)
        np.testing.assert_allclose(stats[r]["mean_abs_td"], np.abs(s["learner"].last_td()).astype(np.float64).mean(), rtol=1e-6)  # own
    assert np.array_equal(ranks[0]["net"].get(), ranks[1]["net"].get())
    for s in ranks:
        _close(s)


def test_checkpoint_mid_run_continues_on_both_ranks(pkg, pairs):
    (a_ctx, b_ctx), one = pairs
    n, case = 127, dict(ratio=1.0, threshold=2, target_freq=3)
    _warm(pkg, one, 2 * n, case)
    a = [_agent(pkg, c, 2 * n, case, seed=300, steps=20) for c in a_ctx]
    _run_pair(pkg, a, 9)
    ck = [pkg.checkpoint.checkpoint_replay(s["env"], s["net"], s["agent"]) for s in a]
    _run_pair(pkg, a, 11)
    final = [_state(pkg, s) for s in a]
    b = [_agent(pkg, c, 2 * n, case, seed=999, steps=20) for c in b_ctx]       # other seeds
    _run_pair(pkg, b, 4)
    for r in range(2):
        pkg.checkpoint.restore_replay(ck[r], b[r]["env"], b[r]["net"], b[r]["agent"])
    _run_pair(pkg, b, 11)
    for r in range(2):
        _assert_same(final[r], _state(pkg, b[r]))
    for s in a + b:
        _close(s)


@pytest.mark.parametrize("name,hidden", [("linear", 64), ("gumbel", 64), ("speedy", 128), ("greedy", 64)])
def test_evaluate_explore_on_shards_equals_the_union(pkg, pairs, name, hidden):
    (ctxs, _), one = pairs
    n, steps, K = 127, 40, 2
    case = dict(hidden=hidden, explorer=name)
    ranks = [_agent(pkg, c, 2 * n, case, steps=steps) for c in ctxs]
    union = _agent(pkg, one, 2 * n, case, steps=steps)
    res = [pkg.learners.evaluate(s["policy"], s["env"], steps, max_episodes=K) for s in ranks]   # no exchange: rank by rank
    ru = pkg.learners.evaluate(union["policy"], union["env"], steps, max_episodes=K)
    for k in ("returns", "lengths"):
        assert np.array_equal(np.concatenate([res[0][k], res[1][k]], axis=1), ru[k], equal_nan=(k == "returns")), k
    assert np.array_equal(np.concatenate([res[0]["counts"], res[1]["counts"]]), ru["counts"])
    assert np.array_equal(np.concatenate([s["policy"].explorer_rng() for s in ranks]), union["policy"].explorer_rng())
    if hasattr(union["policy"].explorer, "step"):
        assert ranks[0]["policy"].explorer.step == ranks[1]["policy"].explorer.step == union["policy"].explorer.step == 1 + steps * 2 * n
    for s in ranks + [union]:
        _close(s)


def test_disagreeing_ranks_refuse_and_touch_nothing(pkg, pairs):
    (ctxs, _), one = pairs
    L = pkg._lib
    n, case = 64, dict(ratio=1.0, threshold=2)
    _warm(pkg, one, 2 * n, case)
    ranks = [_agent(pkg, c, 2 * n, case, steps=8) for c in ctxs]
    _run_pair(pkg, ranks, 3)                                                  # live handles, warm
    hs = [s["agent"]._handle(s["env"]) for s in ranks]

    def attempt(args):
        before = [_state(pkg, s) for s in ranks]
        codes = [None, None]

        def go(r):
            ex, ctl, k = args[r]
            codes[r] = ctxs[r].lib.b200rl_replay_run(hs[r], C.c_void_p(ranks[r]["policy"]._d_rng), C.byref(ex), C.byref(ctl), k, None)
        _in_threads([lambda r=r: go(r) for r in range(2)])
        assert codes == [L.ERR_INVALID, L.ERR_INVALID], codes
        for r in range(2):
            _assert_same(before[r], _state(pkg, ranks[r]))

    def base(r):
        c = ranks[r]["traj"].controller
        return [ranks[r]["policy"].explorer.as_struct(), L.InsertSampleRatio(c.ratio, c.threshold, c.n_inserted, c.n_sampled), 4]
    a = [base(0), base(1)]; a[1][2] = 5                                          # n_steps
    attempt(a)
    a = [base(0), base(1)]; a[1][1].threshold += 1                               # controller
    attempt(a)
    a = [base(0), base(1)]; a[0][1].n_sampled += 1
    attempt(a)
    a = [base(0), base(1)]; a[1][0].step += 1                                    # explorer step
    attempt(a)
    a = [base(0), base(1)]; a[0][0].decay_steps = 0; a[0][0].warmup_steps = 0    # a rank that refuses for its own reason
    a[0][0].eps_init = 2.0
    attempt(a)
    # a different N per rank
    odd = [_agent(pkg, ctxs[0], 2 * n, case, steps=8)]
    ex1 = ranks[1]["policy"].explorer
    e = pkg.B200VecEnv(ctxs[1], "CartPole", n + 1, O.splitmix_states_fast(n + 1, 3), auto_reset=True)
    t = pkg.Trajectory(ctxs[1], 4, 8, lanes=n + 1, batch_size=64, sampler_rng=O.splitmix_states_fast(64, 4))
    t.controller = pkg.InsertSampleRatioController(ratio=1.0, threshold=2)
    lr = pkg.DQNLearner(ctxs[1], ranks[1]["net"], t, ranks[1]["learner"].cfg)
    pol = pkg.QBasedPolicy(ctxs[1], lr, ex1, O.splitmix_states_fast(n + 1, 5), n + 1)
    ag = pkg.Agent(pol, t)
    odd.append(dict(env=e, net=ranks[1]["net"], traj=t, learner=lr, policy=pol, agent=ag))
    _prepare(odd)
    hs_odd = [odd[0]["agent"]._handle(odd[0]["env"]), ag._handle(e)]
    before = [_state(pkg, s) for s in odd]
    codes = [None, None]

    def go(r):
        s = odd[r]
        c = s["traj"].controller
        ctl = L.InsertSampleRatio(c.ratio, c.threshold, c.n_inserted, c.n_sampled)
        ex = s["policy"].explorer.as_struct()
        codes[r] = ctxs[r].lib.b200rl_replay_run(hs_odd[r], C.c_void_p(s["policy"]._d_rng), C.byref(ex), C.byref(ctl), 3, None)
    _in_threads([lambda r=r: go(r) for r in range(2)])
    assert codes == [L.ERR_INVALID, L.ERR_INVALID], codes
    for r in range(2):
        _assert_same(before[r], _state(pkg, odd[r]))
    odd[0]["agent"].close(); odd[0]["policy"].close(); odd[0]["traj"].close(); odd[0]["net"].close(); odd[0]["env"].close()
    ag.close(); pol.close(); t.close(); e.close()
    for s in ranks:
        _close(s)
