"""The forward pass of every network kind, on every path that runs it, against float64 (ac_ref.py), per sample and per output
row within 1e-5 (|ref| + scale) — the scale being the same sums with every term in absolute value.

Paths: "tc" (H = 64, the tensor-core forward of tc_fwd.cuh, a 3-term fp16 split on wgmma), "ffma64" (H = 64 with
b200rl_set_tensor_cores(0)), "ffma128" (H = 128, FP32 FFMA).  Entry points: b200rl_net_act (actor heads, sampled actions,
log-probs, critic values), b200rl_net_values (nn_mlp_forward: Q, dueling Q, critic values), and the fused kernels of fwd_tc.cu —
the rollout (every recorded value and log-prob), the greedy evaluation (modes 0 and 2) and the DQN collect window (the actions
pushed into the replay ring).  N runs over the edges of a 128-sample tile, of the forward's grid and of the fused kernels'
resident-slot groups, all computed from the device's SM count."""
import contextlib
import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import ac_ref as R
import oracle_lib as O

pytestmark = pytest.mark.gpu

PATHS = {"tc": (64, 1), "ffma64": (64, 0), "ffma128": (128, 1)}
HEADS = [("cat", R.KIND_CATEGORICAL, n) for n in (1, 2, 3, 4)] + [("gauss", R.KIND_GAUSSIAN, 1)] + \
        [("q", R.KIND_Q, n) for n in (1, 2, 3, 4)] + [("duel", R.KIND_DUELING, n) for n in (1, 2, 3)]
HEAD_IDS = [f"{name}{n}" for name, _, n in HEADS]
K_SLOTS, TM = 2, 128          # fwd_tc.cu: resident tiles per CTA of the fused kernels, samples per tile


@pytest.fixture(scope="module")
def sms(ctx):
    """SMs of device 0 (the driver API: no runtime library to initialise for one attribute)"""
    cu = C.CDLL("libcuda.so.1")
    dev, n = C.c_int(), C.c_int()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), 0) == 0
    assert cu.cuDeviceGetAttribute(C.byref(n), 16, dev) == 0          # CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT
    return n.value


@contextlib.contextmanager
def tensor_cores(pkg, ctx, on):
    pkg._lib.check(ctx.lib.b200rl_set_tensor_cores(int(on)))
    try:
        yield
    finally:
        pkg._lib.check(ctx.lib.b200rl_set_tensor_cores(1))


def run_direct(pkg, ctx, path, kind, n_in, n_out, act, mag, N, seed, what):
    """b200rl_net_act (actor-critic kinds) and b200rl_net_values on one case, every output against float64"""
    H, tc = PATHS[path]
    p, x = R.make_case(kind, n_in, n_out, act, H, mag, N, seed)
    ref = R.forward(p, n_in, H, kind, n_out, act, x)
    with tensor_cores(pkg, ctx, tc):
        net = pkg.Network(ctx, n_in, H, n_out, p, act=act, kind=kind)
        try:
            if kind in (R.KIND_Q, R.KIND_DUELING):
                R.check(net.values(x), *ref["q"], f"{what}: Q")
                return
            seeds = O.splitmix_states_fast(N, seed + 7)
            d_rng = ctx.malloc(N * 32); ctx.h2d(d_rng, seeds)
            try:
                out = net.act(x, d_rng)
                rng_after = np.empty((N, 4), np.uint64); ctx.d2h(rng_after, d_rng)
            finally:
                ctx.free(d_rng)
            R.check(out["heads"], *ref["heads"], f"{what}: heads")
            R.check(out["value"], *ref["value"], f"{what}: act value")
            R.check(net.values(x), *ref["value"], f"{what}: values()")
            z, S = ref["heads"]
            cols = np.arange(N)
            if kind == R.KIND_GAUSSIAN:
                o = O.act_gaussian(O.ac_desc(n_in, H, 1, act, True), O.hyper_array(), p, x, seeds)
                lp, Slp = R.gaussian_logp(z[0], z[1], S[0], S[1], out["action"])
                R.check(out["logp"], lp, Slp, f"{what}: log-density of the sampled action")
            else:
                o = O.act_discrete(O.ac_desc(n_in, H, n_out, act), p, x, seeds)
                lp, Slp = ref["logp"]
                a = out["action"] - 1
                assert np.all((a >= 0) & (a < n_out)), what
                R.check(out["logp"], lp[a, cols], Slp[a, cols], f"{what}: log-prob of the sampled action")
                # the Gumbel arg-max where the oracle's margin clears the float32 noise of the log-probs (4x their tolerance)
                safe = o["margin"] > 4 * R.BAR * (np.abs(lp) + Slp).max(0) if n_out > 1 else np.ones(N, bool)
                assert safe.mean() > 0.9, (what, safe.mean())
                bad = np.flatnonzero(safe & (out["action"] != o["action"]))
                assert bad.size == 0, f"{what}: sampled action differs at safe margin, samples {bad[:8]}"
            assert np.array_equal(rng_after, o["rng"]), f"{what}: policy streams"
        finally:
            net.close()


# ---- every head x observation width x activation x path, N = 300 (two whole tiles and a partial one) -------------------------
@pytest.mark.parametrize("act", [0, 1], ids=["relu", "tanh"])
@pytest.mark.parametrize("n_in", [1, 2, 3, 4], ids=lambda n: f"in{n}")
@pytest.mark.parametrize("name,kind,n_out", HEADS, ids=HEAD_IDS)
@pytest.mark.parametrize("path", list(PATHS))
def test_forward_shapes(pkg, ctx, path, name, kind, n_out, n_in, act):
    run_direct(pkg, ctx, path, kind, n_in, n_out, act, "unit", 300, 40 + n_in + 10 * n_out,
               f"{path} {name}{n_out} in{n_in} {'relu' if act == 0 else 'tanh'} N=300")


# ---- tile and grid edges --------------------------------------------------------------------------------------------------
# g * TM +- 1 for the forward's own grid g and tile TM (nn.cu): act() (nn_policy_act) runs sm_count CTAs per network at H = 64,
# sm_count / 2 at H = 128; values() (nn_mlp_forward) 2 sm_count at H = 64, sm_count at H = 128; TM = 128 at H = 64, 64 at H = 128
EDGES = ["1", "63", "64", "65", "127", "128", "129"] + [f"{g}-grid{d}" for g in ("act", "values") for d in ("-1", "", "+1")]
EDGE_SHAPES = [("cat4-in4-relu", R.KIND_CATEGORICAL, 4, 4, 0), ("gauss-in3-tanh", R.KIND_GAUSSIAN, 1, 3, 1),
               ("q4-in2-tanh", R.KIND_Q, 4, 2, 1), ("duel3-in3-relu", R.KIND_DUELING, 3, 3, 0)]


def edge_n(edge, sms, H):
    if "grid" not in edge:
        return int(edge)
    g, rest = edge.split("-grid")
    ctas = (sms if g == "act" else 2 * sms) if H == 64 else (sms // 2 if g == "act" else sms)
    return ctas * (128 if H == 64 else 64) + int(rest or 0)


@pytest.mark.parametrize("edge", EDGES)
@pytest.mark.parametrize("shape,kind,n_out,n_in,act", EDGE_SHAPES, ids=[s[0] for s in EDGE_SHAPES])
@pytest.mark.parametrize("path", list(PATHS))
def test_forward_tile_and_grid_edges(pkg, ctx, sms, path, shape, kind, n_out, n_in, act, edge):
    N = edge_n(edge, sms, PATHS[path][0])
    run_direct(pkg, ctx, path, kind, n_in, n_out, act, "unit", N, 7, f"{path} {shape} N={N} ({edge})")


# ---- operand magnitudes ---------------------------------------------------------------------------------------------------
MAG_CASES = [(m, a) for m, act in R.MAGNITUDES.items() for a in ((0, 1) if act is None else (act,))]
MAG_HEADS = [("cat4", R.KIND_CATEGORICAL, 4), ("gauss", R.KIND_GAUSSIAN, 1), ("q4", R.KIND_Q, 4), ("duel3", R.KIND_DUELING, 3)]


@pytest.mark.parametrize("mag,act", MAG_CASES, ids=[f"{m}-{'relu' if a == 0 else 'tanh'}" for m, a in MAG_CASES])
@pytest.mark.parametrize("name,kind,n_out", MAG_HEADS, ids=[h[0] for h in MAG_HEADS])
@pytest.mark.parametrize("path", list(PATHS))
def test_forward_magnitudes(pkg, ctx, path, name, kind, n_out, mag, act):
    n_in = R.ENV_NIN.get(mag, 4)
    run_direct(pkg, ctx, path, kind, n_in, n_out, act, mag, 1000, 21, f"{path} {name} in{n_in} {mag} N=1000")


@pytest.mark.parametrize("name,kind,n_out", MAG_HEADS, ids=[h[0] for h in MAG_HEADS])
def test_forward_past_the_fp16_envelope_is_nan(pkg, ctx, name, kind, n_out):
    """relu H1 ~ 1100 in one feature: 64 H1 > 65504 rounds to inf in the fp16 operand, and the tensor-core forward must not return
    finite outputs for those samples.  (The FFMA paths have no such limit.)"""
    p, x = R.make_case(kind, 4, n_out, 0, 64, "unit", 500, 3)
    offsets = [0] if kind in (R.KIND_Q, R.KIND_DUELING) else [0, R.nparams(4, 64, R.head_rows(kind, n_out))]   # (actor and critic)
    for off in offsets:
        p[off + 64 * 4] = 1100.0                                 # b1[0]: H1[0] = relu(W1[0] x + 1100), |W1 x| < 10
    with tensor_cores(pkg, ctx, 1):
        _check_non_finite(pkg, ctx, name, kind, p, x, n_out)


def _check_non_finite(pkg, ctx, name, kind, p, x, n_out):
    net = pkg.Network(ctx, 4, 64, n_out, p, act=0, kind=kind)
    try:
        if kind in (R.KIND_Q, R.KIND_DUELING):
            q = net.values(x)
            assert not np.isfinite(q).any(), f"{name}: {np.isfinite(q).sum()} finite Q-values past the envelope"
            return
        d_rng = ctx.malloc(500 * 32); ctx.h2d(d_rng, O.splitmix_states_fast(500, 1))
        try:
            out = net.act(x, d_rng)
        finally:
            ctx.free(d_rng)
        for k in ("heads", "logp", "value"):
            assert not np.isfinite(out[k]).any(), f"{name}: {np.isfinite(out[k]).sum()} finite {k} past the envelope"
        assert not np.isfinite(net.values(x)).any(), f"{name}: finite values() past the envelope"
    finally:
        net.close()


# ---- fused rollout --------------------------------------------------------------------------------------------------------
def _check_rollout_columns(desc_kind, n_in, n_out, act, p, S, A, LP, V, cols, what, chunk=8192):
    """values and log-probs recorded in columns `cols` against float64 on the recorded states and actions, in chunks of envs
    (bounded host memory; the chunks run on a thread pool, NumPy releases the GIL in its array operations)"""
    def one(t, e0):
        e = slice(e0, min(e0 + chunk, S.shape[1]))
        ref = R.forward(p, n_in, 64, desc_kind, n_out, act, np.ascontiguousarray(S[:, e, t]))
        R.check(V[e, t], *ref["value"], f"{what}: value column {t}, envs {e.start}..{e.stop - 1}")
        if t >= A.shape[1]:
            return
        z, Sz = ref["heads"]
        if desc_kind == R.KIND_GAUSSIAN:
            lp, Slp = R.gaussian_logp(z[0], z[1], Sz[0], Sz[1], A[e, t])
        else:
            a = A[e, t] - 1
            c = np.arange(a.size)
            lp, Slp = ref["logp"][0][a, c], ref["logp"][1][a, c]
        R.check(LP[e, t], lp, Slp, f"{what}: log-prob column {t}, envs {e.start}..{e.stop - 1}")
    with ThreadPoolExecutor(8) as pool:
        for f in [pool.submit(one, t, e0) for t in cols for e0 in range(0, S.shape[1], chunk)]:
            f.result()


ROLLOUTS = {  # env, N (or edge), T, algo, epochs, microbatches, head kind, n_out, act
    "cartpole-ppo-65536-T32": ("CartPole", 65536, 32, "ppo", 4, 4, R.KIND_CATEGORICAL, 2, 0),
    "pendulum-a2c-inside": ("Pendulum", "inside", 3, "a2c", 1, 1, R.KIND_GAUSSIAN, 1, 1),
    "pendulum-a2c-outside": ("Pendulum", "outside", 3, "a2c", 1, 1, R.KIND_GAUSSIAN, 1, 1),
}


def slots_n(edge, sms):
    """N just inside / outside the K_SLOTS * 2 * sm_count tiles the fused kernels keep resident in one group"""
    return K_SLOTS * 2 * sms * TM + (1 if edge == "outside" else 0)


@pytest.mark.parametrize("case", list(ROLLOUTS))
def test_fused_rollout_against_float64(pkg, ctx, sms, case):
    """every value and log-prob of all T columns (and the bootstrap value) of the rollout on the recorded states and actions.
    65 536 CartPole envs at T = 32 is the benchmark's shape.  'outside' has more tiles than the rollout kernel keeps resident: the
    rollout steps through b200rl_net_act launches instead, which must meet the same bar."""
    kind, n, T, algo, E, M, hk, n_out, act = ROLLOUTS[case]
    n = slots_n(n, sms) if isinstance(n, str) else n
    n_in = 4 if kind == "CartPole" else 3
    envkw = dict(continuous=True) if kind == "Pendulum" else {}
    env = pkg.B200VecEnv(ctx, kind, n, O.splitmix_states_fast(n, 0x9E37), auto_reset=True, **envkw)
    p, _ = R.make_case(hk, n_in, n_out, act, 64, "unit", 16, 123)
    net = pkg.Network(ctx, n_in, 64, n_out, p, act=act, kind=hk)
    cfg = pkg.onpolicy_config(update_freq=T, n_epochs=E, n_microbatches=M, algo=algo)
    agent = pkg.OnPolicyAgent(ctx, net, env, cfg, O.splitmix_states_fast(n, 0x1234), host_actions=False)
    try:
        env.reset_(is_force=True)
        l0 = ctx.launch_count()
        agent.collect(T)
        launches = ctx.launch_count() - l0
        assert (launches < T) == (case != "pendulum-a2c-outside"), launches      # one fused launch, or per-step launches
        Rl = pkg.learners
        S, A, LP = agent.rollout(Rl.ROLL_STATE), agent.rollout(Rl.ROLL_ACTION), agent.rollout(Rl.ROLL_LOGP)
        agent.update()                                          # writes the bootstrap value V(s_T) with the collect's parameters
        V = agent.rollout(Rl.ROLL_VALUE)
        S = agent.rollout(Rl.ROLL_STATE)
        _check_rollout_columns(hk, n_in, n_out, act, p, S, A, LP, V, range(T + 1), f"{case} N={n}")
    finally:
        agent.close(); net.close(); env.close()


# ---- fused evaluation (greedy) and DQN collect ----------------------------------------------------------------------------
def _greedy_check(q, S, a1, what):
    """a1 (1-based actions) against the float64 first maximum of q = (value, scale) rows, where the margin is safe"""
    z, Sz = q
    _, safe = R.margin_of(z, R.BAR * (np.abs(z) + Sz))
    assert safe.mean() > 0.9, (what, safe.mean())
    bad = np.flatnonzero(safe & (a1 != z.argmax(0) + 1))
    assert bad.size == 0, f"{what}: {bad.size} greedy actions differ from the float64 arg-max at a safe margin, e.g. envs {bad[:8]}"


def _q_policy(pkg, ctx, net, n_in, n, seed):
    traj = pkg.Trajectory(ctx, n_in, 4, lanes=n, batch_size=32, sampler_rng=O.splitmix_states_fast(32, seed), prioritized=False)
    traj.controller = pkg.InsertSampleRatioController(ratio=1.0, threshold=10 ** 9)      # no update: the Q-network stays fixed
    learner = pkg.DQNLearner(ctx, net, traj, pkg.dqn_config())
    return traj, pkg.QBasedPolicy(ctx, learner, pkg.GreedyExplorer(), O.splitmix_states_fast(n, seed + 1), n)


EVALS = {  # env, n_in, head kind, n_out, act
    "mode0-cartpole-cat2": ("CartPole", 4, R.KIND_CATEGORICAL, 2, 0),
    "mode0-pendulum-gauss": ("Pendulum", 3, R.KIND_GAUSSIAN, 1, 1),
    "mode2-mountaincar-q3": ("MountainCar", 2, R.KIND_Q, 3, 1),
    "mode2-pendulum-duel3": ("Pendulum", 3, R.KIND_DUELING, 3, 0),
}


@pytest.mark.parametrize("edge", ["inside", "outside"])
@pytest.mark.parametrize("case", list(EVALS))
def test_fused_greedy_evaluation_against_float64(pkg, ctx, sms, case, edge):
    """one window step of b200rl_evaluate from the forced reset: the action each env received (its last action) against the float64
    greedy action on the reset state (a twin env, same seeds, reset the same way).  'outside': a second group of resident tiles."""
    kind, n_in, hk, n_out, act = EVALS[case]
    envkw = {}
    if kind == "Pendulum":     # continuous torque for the Gaussian head, 3 discrete torques for the dueling Q-network
        envkw = dict(params=pkg.pendulum_params(continuous=hk == R.KIND_GAUSSIAN, n_actions=3))
    n = slots_n(edge, sms)
    seeds = O.splitmix_states_fast(n, 9)
    env, twin = (pkg.B200VecEnv(ctx, kind, n, seeds, auto_reset=True, **envkw) for _ in range(2))
    p, _ = R.make_case(hk, n_in, n_out, act, 64, "unit", 16, 55)
    net = pkg.Network(ctx, n_in, 64, n_out, p, act=act, kind=hk)
    traj = policy = None
    what = f"{case} N={n} ({edge})"
    try:
        twin.reset_(is_force=True)
        x = twin.state()
        ref = R.forward(p, n_in, 64, hk, n_out, act, x)
        l0 = ctx.launch_count()
        if hk in (R.KIND_Q, R.KIND_DUELING):
            traj, policy = _q_policy(pkg, ctx, net, n_in, n, 3)
            pkg.evaluate(policy, env, 1)
        else:
            pkg.evaluate(net, env, 1)
        assert ctx.launch_count() - l0 <= 2, what                 # the forced reset and one fused window
        a = env.last_action()
        if hk == R.KIND_GAUSSIAN:
            mu, Smu = ref["heads"][0][0], ref["heads"][1][0]
            R.check(a, np.clip(mu, -2.0, 2.0), Smu, f"{what}: greedy torque clamp(mu)")
        else:
            _greedy_check(ref["q"] if "q" in ref else ref["heads"], x, a, what)
    finally:
        if policy is not None:
            policy.close(); traj.close()
        net.close(); env.close(); twin.close()


@pytest.mark.parametrize("edge", ["inside", "outside"])
@pytest.mark.parametrize("qkind", ["q2", "duel2"])
def test_fused_dqn_collect_against_float64(pkg, ctx, sms, qkind, edge):
    """run(Agent(QBasedPolicy(GreedyExplorer)), CartPole, StopAfterNSteps(3)) on the fused collect window, no update: every action
    in the replay ring (as checkpoint_replay exports it) is the float64 first arg-max of Q on the state stored with it"""
    n = slots_n(edge, sms)
    hk = R.KIND_Q if qkind == "q2" else R.KIND_DUELING
    env = pkg.B200VecEnv(ctx, "CartPole", n, O.splitmix_states_fast(n, 17), auto_reset=True)
    p, _ = R.make_case(hk, 4, 2, 0, 64, "unit", 16, 66)
    net = pkg.Network(ctx, 4, 64, 2, p, act=0, kind=hk)
    traj, policy = _q_policy(pkg, ctx, net, 4, n, 5)
    agent = pkg.Agent(policy, traj)
    what = f"{qkind} N={n} ({edge})"
    try:
        pkg.run(agent, env, pkg.StopAfterNSteps(3), pkg.EmptyHook())
        assert agent._replay is not None, what                   # the fused collect ran
        ck = pkg.checkpoint.checkpoint_replay(env, net, agent)
        F = ck["traj/flag"].size // n                             # frames per lane (cap + 1), slot-major: k = slot * lanes + lane
        st = ck["traj/state"].reshape(F * n, 4).T
        took = (ck["traj/flag"] & 2) != 0                         # frames an action was taken in
        assert took.sum() >= n, (what, took.sum())
        ref = R.forward(p, 4, 64, hk, 2, 0, st[:, took])
        _greedy_check(ref["q"], st[:, took], ck["traj/action"][took], what)
    finally:
        agent.close(); policy.close(); traj.close(); net.close(); env.close()
