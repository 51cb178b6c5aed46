"""The PPO / A2C loss + backward (K7) on every path that runs it, against float64 (ac_grad_ref.py): every entry of every parameter
block of both networks within 1e-5 (|g| + scale), and the four losses, read back through Network.ac_step and NET_GRAD.

Paths: "tc" (H = 64, nn_tc.cu: four wgmma GEMMs per tile on 3-term fp16 splits, actor and critic CTAs), "ffma64" (H = 64 with
b200rl_set_tensor_cores(0)) and "ffma128" (H = 128); categorical 3-4 actions run FFMA on every path.  B runs over the tile and
grid edges of each kernel, computed from the device's SM count and the actor : critic split rule (tc_split.h), with the partial
gradient rows dirtied by an earlier launch so that a row a role fails to write shows.  Magnitudes: the sweep of ac_grad_ref
(small critic residuals, a near-deterministic policy, unnormalised and zero advantages, every PPO clip regime, clamped sigma,
Pendulum-scale returns, the split-structured case), the PPO clip edge hit exactly, and the fp16 envelope of the critic's dP1
operand on both sides.  Then the optimiser step (clip_by_global_norm against the float64 gradient) on the separate and the fused
path, and the first minibatch of a PPO CartPole rollout at the benchmark's shape."""
import contextlib
import ctypes as C

import numpy as np
import pytest

import ac_grad_ref as G
import ac_ref as R
import oracle_lib as O

pytestmark = pytest.mark.gpu

PATHS = {"tc": (64, 1), "ffma64": (64, 0), "ffma128": (128, 1)}
HEADS = [("cat1", R.KIND_CATEGORICAL, 1), ("cat2", R.KIND_CATEGORICAL, 2), ("cat3", R.KIND_CATEGORICAL, 3),
         ("cat4", R.KIND_CATEGORICAL, 4), ("gauss", R.KIND_GAUSSIAN, 1)]
FP16_MAX, FP16_INF_FROM = 65504.0, 65520.0      # largest fp16; round-to-nearest gives inf from 65520 on


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


def cfg_of(pkg, hp, max_grad_norm=0.5):
    return pkg.onpolicy_config(clip_range=hp["clip_range"], w_actor=hp["w_actor"], w_critic=hp["w_critic"], w_entropy=hp["w_entropy"],
                               min_sigma=hp["min_sigma"], max_sigma=hp["max_sigma"], normalize_advantage=hp["normalize_adv"],
                               algo=hp["algo"], max_grad_norm=max_grad_norm)


def run_step(pkg, ctx, path, kind, n_in, n_out, act, case, idx=None, dirty=True, apply_update=False, max_grad_norm=0.5):
    """NET_GRAD and the losses of one ac_step on `path`.  dirty: an FFMA launch first writes a nonzero gradient into every partial
    row (the batch repeated to >= 17 000 samples: every one of its CTAs has tiles), so a row the tensor-core kernel fails to write
    (or to zero-fill) shows in the sum"""
    H, tc = PATHS[path]
    p, x, a, lp, adv, ret, hp, mean, inv_std = case
    net = pkg.Network(ctx, n_in, H, n_out, p, act=act, kind=kind)
    try:
        cfg = cfg_of(pkg, hp, max_grad_norm)
        if dirty and path == "tc":
            k = -(-17000 // x.shape[1])
            with tensor_cores(pkg, ctx, 0):
                net.ac_step(cfg, np.tile(x, k), np.tile(a, k), np.tile(lp, k), np.tile(adv, k), np.tile(ret, k), None, mean, inv_std,
                            apply_update=False)
        with tensor_cores(pkg, ctx, tc):
            got = net.ac_step(cfg, x, a, lp, adv, ret, idx, mean, inv_std, apply_update=apply_update)
        return net.get(pkg.learners.NET_GRAD), got
    finally:
        net.close()


def check_case(pkg, ctx, path, kind, n_in, n_out, act, case, what, idx=None, dirty=True):
    H = PATHS[path][0]
    ref = G.ref_of(case, n_in, H, kind, n_out, act, idx)
    assert not ref["ties"].any(), what
    g, got = run_step(pkg, ctx, path, kind, n_in, n_out, act, case, idx, dirty)
    G.check_grad(g, ref, n_in, H, kind, n_out, what)
    G.check_losses(got, ref, what)
    return ref, g


# ---- every head x observation width x activation x path, B = 300 (two whole tiles and a partial one) -----------------------
@pytest.mark.parametrize("act", [0, 1], ids=["relu", "tanh"])
@pytest.mark.parametrize("n_in", [1, 2, 3, 4], ids=lambda n: f"in{n}")
@pytest.mark.parametrize("name,kind,n_out", HEADS, ids=[h[0] for h in HEADS])
@pytest.mark.parametrize("path", list(PATHS))
def test_backward_shapes(pkg, ctx, path, name, kind, n_out, n_in, act):
    algo = "a2c" if (n_in + n_out) % 3 == 0 else "ppo"
    case = G.make_batch(kind, n_in, n_out, act, PATHS[path][0], "unit", 300, 40 + n_in + 10 * n_out, algo)
    check_case(pkg, ctx, path, kind, n_in, n_out, act, case, f"{path} {name} in{n_in} {'relu' if act == 0 else 'tanh'} {algo} B=300")


# ---- tile and grid edges --------------------------------------------------------------------------------------------------
def tc_actor_ctas(grid, gaussian, ntiles):
    """tc_split.h b200rl_tc_actor_ctas, restated"""
    r = 0.85 if gaussian else 0.87
    best, best_cost = grid // 2, 1e300
    for na in range(grid // 2, min(grid // 2 + 8, grid - 1) + 1):
        ca, cc = float(-(-ntiles // na)), r * float(-(-ntiles // (grid - na)))
        cost = max(ca, cc)
        if cost < best_cost - 1e-9:
            best, best_cost = na, cost
    return best


def _first_two_tile_b(grid, gaussian, role):
    """the smallest B at which some CTA of the role runs a second tile, under the split that B itself gets: B = (nt - 1) * 128 + 1
    for the first tile count nt above the role's CTA count (n_role * 128 + 1 where the split does not move)"""
    for nt in range(1, 2 * grid):
        na = tc_actor_ctas(grid, gaussian, nt)
        if nt > (na if role == "actor" else grid - na):
            return (nt - 1) * 128 + 1
    raise AssertionError(role)


def edge_b(path, edge, sms, gaussian):
    if path == "tc":
        grid = 2 * (sms // 2)
        if edge == "critic-2tiles":
            return _first_two_tile_b(grid, gaussian, "critic")
        if edge == "actor-2tiles":
            return _first_two_tile_b(grid, gaussian, "actor")
        if edge == "3tiles":           # every CTA of both roles runs three tiles or more
            nt = 3 * (grid // 2 + 8)
            return nt * 128
        return int(edge)
    H = PATHS[path][0]
    tm = 128 if H == 64 else 64
    ctas = sms if H == 64 else sms // 2       # nn_grid_ctas: CTAs per role
    return {"tm-1": tm - 1, "tm": tm, "tm+1": tm + 1, "grid+1": ctas * tm + 1, "3tiles": 3 * ctas * tm}.get(edge) or int(edge)


TC_EDGES = ["1", "127", "128", "129", "critic-2tiles", "actor-2tiles", "3tiles"]
FFMA_EDGES = ["1", "tm-1", "tm", "tm+1", "grid+1", "3tiles"]
EDGE_CASES = [(p, e) for p in PATHS for e in (TC_EDGES if p == "tc" else FFMA_EDGES)]
EDGE_SHAPES = [("cat2-in4-relu", R.KIND_CATEGORICAL, 2, 4, 0), ("gauss-in3-tanh", R.KIND_GAUSSIAN, 1, 3, 1)]


@pytest.mark.parametrize("order", ["idx-none", "idx-permuted"])
@pytest.mark.parametrize("shape,kind,n_out,n_in,act", EDGE_SHAPES, ids=[s[0] for s in EDGE_SHAPES])
@pytest.mark.parametrize("path,edge", EDGE_CASES, ids=[f"{p}-{e}" for p, e in EDGE_CASES])
def test_backward_tile_and_grid_edges(pkg, ctx, sms, path, edge, shape, kind, n_out, n_in, act, order):
    B = edge_b(path, edge, sms, kind == R.KIND_GAUSSIAN)
    what = f"{path} {shape} B={B} ({edge}, {order})"
    if order == "idx-none":
        case = G.make_batch(kind, n_in, n_out, act, PATHS[path][0], "unit", B, 5, "ppo")
        check_case(pkg, ctx, path, kind, n_in, n_out, act, case, what)
    else:                               # a permuted subset of a larger rollout
        extra = 37
        case = G.make_batch(kind, n_in, n_out, act, PATHS[path][0], "unit", B + extra, 6, "ppo")
        idx = np.random.default_rng(B).permutation(B + extra)[:B].astype(np.int32)
        check_case(pkg, ctx, path, kind, n_in, n_out, act, case, what, idx=idx)


# ---- operand magnitudes ---------------------------------------------------------------------------------------------------
def mag_cases():
    out = []
    for name, kind, n_out in (("cat2", R.KIND_CATEGORICAL, 2), ("gauss", R.KIND_GAUSSIAN, 1)):
        for mag in G.MAGNITUDES:
            if (mag in G.GAUSS_ONLY and kind != R.KIND_GAUSSIAN) or (mag in G.CAT_ONLY and kind != R.KIND_CATEGORICAL):
                continue
            acts = (1,) if mag == "pendulum" else (0,) if mag == "split-structured" else (0, 1)
            for act in acts:
                algo = "ppo" if mag in G.PPO_ONLY or mag == "split-structured" else ("a2c" if act else "ppo")
                out.append(pytest.param(kind, n_out, act, mag, algo, id=f"{name}-{mag}-{'relu' if act == 0 else 'tanh'}-{algo}"))
    return out


@pytest.mark.parametrize("kind,n_out,act,mag,algo", mag_cases())
@pytest.mark.parametrize("path", list(PATHS))
def test_backward_magnitudes(pkg, ctx, path, kind, n_out, act, mag, algo):
    n_in = 3 if mag == "pendulum" else 4
    B = 640 if mag == "split-structured" else 1000
    case = G.make_batch(kind, n_in, n_out, act, PATHS[path][0], mag, B, 21, algo)
    check_case(pkg, ctx, path, kind, n_in, n_out, act, case, f"{path} {mag} {algo} B={B}")


@pytest.mark.parametrize("path", list(PATHS))
def test_ppo_ratio_exactly_on_the_clip_edge(pkg, ctx, path):
    """clip_range = 0 and a float32 ratio of exactly 1.0 (actor head weights 0: the logits are exactly b3 = {0, -30}, the log-sum-exp
    is log(1.0f) = 0, and the action taken has log-probability -30 = logp_old): the ratio sits on both edges, where the `inside`
    rule (ratio <= 1 + clip_range) keeps the gradient.  Float64 puts the ratio 1e-13 below 1, on the lower edge, where A > 0 keeps
    it as well: both agree, so this tie is exact rather than near."""
    H = PATHS[path][0]
    n_in, B = 4, 700
    p, x = R.make_case(R.KIND_CATEGORICAL, n_in, 2, 0, H, "unit", B + 100, 9)
    o = R._offsets(n_in, H, 2)["head"]
    p[o] = 0.0
    p[o.stop - 2:o.stop] = [0.0, -30.0]
    hp = G.hyper(algo="ppo", clip_range=0.0, w_entropy=0.01, normalize_adv=False)
    n = x.shape[1]
    a = np.full(n, 2, np.int32)
    lp = np.full(n, -30.0, np.float32)
    adv = np.random.default_rng(1).uniform(0.5, 2.0, n).astype(np.float32)
    ret = np.random.default_rng(2).standard_normal(n).astype(np.float32)
    ref = G.ref_of((p, x, a, lp, adv, ret, hp, 0.0, 1.0), n_in, H, R.KIND_CATEGORICAL, 2, 0)
    k = np.flatnonzero(~(ref["actor"]["ties"] | ref["critic"]["ties"]))[:B]     # relu near-ties out (the ratio's is this case's)
    case = (p, np.ascontiguousarray(x[:, k]), a[k], lp[k], adv[k], ret[k], hp, 0.0, 1.0)
    ref = G.ref_of(case, n_in, H, R.KIND_CATEGORICAL, 2, 0)
    assert k.size == B and not (ref["actor"]["ties"] | ref["critic"]["ties"]).any()
    g, got = run_step(pkg, ctx, path, R.KIND_CATEGORICAL, n_in, 2, 0, case)
    G.check_grad(g, ref, n_in, H, R.KIND_CATEGORICAL, 2, f"{path} ratio on the clip edge")
    G.check_losses(got, ref, f"{path} ratio on the clip edge")
    hb = [b for b in G.block_names(n_in, H, R.KIND_CATEGORICAL, 2) if b[0] == "actor.b3"][0]
    assert abs(ref["grad"][hb[1] + 1]) > 0.5 * np.mean(adv[k]), "the surrogate's gradient must reach the head bias"


# ---- the fp16 envelope of the tensor-core backward's dP1 operand --------------------------------------------------------------
def _envelope_case(n_in, B, resid):
    """relu, critic W2 and head >= 0 (dP1 = sum_j W2 dP2 adds up: the dP1 operand peaks well above the dP2 one), R = V + resid;
    B samples without near-ties (drawn with spares)"""
    Bn = B
    B = B + B // 8
    p, x = R.make_case(R.KIND_CATEGORICAL, n_in, 2, 0, 64, "unit", B, 13)
    na = R.nparams(n_in, 64, 2)
    s = R._offsets(n_in, 64, 1)
    p[na + s["W2"].start:na + s["W2"].stop] = np.abs(p[na + s["W2"].start:na + s["W2"].stop])
    p[na + s["head"].start:na + s["head"].stop] = np.abs(p[na + s["head"].start:na + s["head"].stop])
    hp = G.hyper(algo="ppo", clip_range=0.2, w_entropy=0.01)
    rng = np.random.default_rng(3)
    a = rng.integers(1, 3, B).astype(np.int32)
    _, v = G._values(p, n_in, 64, R.KIND_CATEGORICAL, 2, 0, x)
    z, _ = G._values(p, n_in, 64, R.KIND_CATEGORICAL, 2, 0, x)
    lpv, _ = R.log_softmax(z, 0 * z)
    lp = (lpv[a - 1, np.arange(B)] - 0.1 * rng.standard_normal(B)).astype(np.float32)
    adv = rng.standard_normal(B).astype(np.float32)
    ret = (v + resid).astype(np.float32)
    mean, inv_std = float(np.float32(adv.astype(np.float64).mean())), float(np.float32(1 / (adv.astype(np.float64).std() + 1e-8)))
    ties = G.loss_grad(p, n_in, 64, R.KIND_CATEGORICAL, 2, 0, x, a, lp, adv, ret, hp, mean, inv_std)["ties"]
    k = np.flatnonzero(~ties)[:Bn]
    assert k.size == Bn
    return (p, np.ascontiguousarray(x[:, k]), a[k], lp[k], adv[k], ret[k], hp, mean, inv_std)


def _operands(ref, B):
    """the critic's dP2 / dP1 operands as the kernel forms them: scale_p = 2^floor(log2 B) * 4 times the float64 gradients"""
    sp = 2.0 ** np.floor(np.log2(1.0 / ref["inv_B"])) * 4.0
    return np.abs(ref["critic"]["dP2"]) * sp, np.abs(ref["critic"]["dP1"]) * sp


@pytest.mark.parametrize("side", ["inside", "outside"])
def test_critic_dp1_operand_fp16_envelope(pkg, ctx, side):
    """critic residuals that put the largest dP1 operand just inside fp16 (0.97 x 65504: every entry meets the bar) and just past it
    (1.1 x 65520, where the hi part rounds to inf): then the dW1 / db1 rows of the overflowing features must be NaN, never finite and
    wrong, and every other entry still meets the bar.  The FFMA path has no such limit and meets the bar on both."""
    n_in, B = 4, 2000
    base = _envelope_case(n_in, B, 1.0)
    ref1 = G.ref_of(base, n_in, 64, R.KIND_CATEGORICAL, 2, 0)
    p2, p1 = _operands(ref1, B)
    target = 0.97 * FP16_MAX if side == "inside" else 1.1 * FP16_INF_FROM
    resid = target / p1.max()
    assert p2.max() * resid < 0.5 * FP16_MAX, "the dP2 operand must stay inside: only dP1 crosses"
    case = _envelope_case(n_in, B, resid)
    ref = G.ref_of(case, n_in, 64, R.KIND_CATEGORICAL, 2, 0)
    assert not ref["ties"].any()
    _, p1 = _operands(ref, B)
    feat_max = p1.max(1)
    g, got = run_step(pkg, ctx, "tc", R.KIND_CATEGORICAL, n_in, 2, 0, case)
    what = f"tc critic residual {resid:.4g} ({side}: max dP1 operand {feat_max.max():.6g})"
    blocks = {b[0]: (b[1], b[2]) for b in G.block_names(n_in, 64, R.KIND_CATEGORICAL, 2)}
    if side == "inside":
        G.check_grad(g, ref, n_in, 64, R.KIND_CATEGORICAL, 2, what)
    else:
        over = feat_max >= 1.001 * FP16_INF_FROM
        under = feat_max <= 0.999 * FP16_MAX
        assert over.any() and (over | under).mean() > 0.9, (what, over.sum(), under.sum())
        a1, b1 = blocks["critic.W1"]
        W1 = g[a1:b1].reshape(n_in, 64)                       # W1 flat: entry f + 64 i
        c1, d1 = blocks["critic.b1"]
        bad = np.flatnonzero(over & (np.isfinite(W1).any(0) | np.isfinite(g[c1:d1])))
        assert bad.size == 0, f"{what}: features {bad[:8]} overflow the fp16 dP1 operand but have finite dW1 / db1 entries"
        keep = np.ones(g.size, bool)
        for f in np.flatnonzero(~under):
            keep[a1 + f + 64 * np.arange(n_in)] = False
            keep[c1 + f] = False
        gm = np.where(keep, g, ref["grad"])                  # the overflowing (and borderline) features' rows: checked above
        G.check_grad(gm, ref, n_in, 64, R.KIND_CATEGORICAL, 2, what)
    g, got = run_step(pkg, ctx, "ffma64", R.KIND_CATEGORICAL, n_in, 2, 0, case)
    G.check_grad(g, ref, n_in, 64, R.KIND_CATEGORICAL, 2, f"ffma64 {what}")


# ---- the optimiser step: clip_by_global_norm! of the gradient --------------------------------------------------------------
def clipped_ref(ref, max_norm):
    """clip_by_global_norm! (float32 rule: scale only when max_norm <= norm) of the float64 gradient, and its scale: each entry's
    own plus the clip factor's error (the norm of the kernel's gradient, within the bar of the norm of |g| + scale)"""
    g, S = ref["grad"], ref["scale"]
    gn = float(np.sqrt((g * g).sum()))
    if not (np.float32(max_norm) <= np.float32(gn)):
        return dict(ref, clip=1.0)
    c = max_norm / max(max_norm, gn)
    rel = float(np.sqrt(((np.abs(g) + S) ** 2).sum())) / gn
    return dict(ref, grad=c * g, scale=c * (S + np.abs(g) * rel), clip=c)


@pytest.mark.parametrize("path", ["tc", "ffma64"])
def test_clipped_gradient_of_the_optimiser_step(pkg, ctx, sms, path):
    """ac_step(apply_update = True): NET_GRAD is the clipped gradient that Adam applied, at a B where every CTA runs several tiles"""
    B = 3 * sms * 128 + 77
    case = G.make_batch(R.KIND_CATEGORICAL, 4, 2, 0, 64, "unit", B, 31, "ppo")
    ref = clipped_ref(G.ref_of(case, 4, 64, R.KIND_CATEGORICAL, 2, 0), 0.01)
    assert ref["clip"] < 0.5, "the case must clip"
    g, got = run_step(pkg, ctx, path, R.KIND_CATEGORICAL, 4, 2, 0, case, apply_update=True, max_grad_norm=0.01)
    G.check_grad(g, ref, 4, 64, R.KIND_CATEGORICAL, 2, f"{path} clipped gradient B={B}")


def _rollout(pkg, ctx, kind, n, T, hk, n_out, act, seed, algo="ppo", E=1, M=1):
    n_in = 4 if kind == "CartPole" else 3
    envkw = dict(continuous=True) if kind == "Pendulum" else {}
    env = pkg.B200VecEnv(ctx, kind, n, O.splitmix_states_fast(n, seed), auto_reset=True, **envkw)
    p, _ = R.make_case(hk, n_in, n_out, act, 64, "unit", 16, seed)
    net = pkg.Network(ctx, n_in, 64, n_out, p, act=act, kind=hk)
    cfg = pkg.onpolicy_config(update_freq=T, n_epochs=E, n_microbatches=M, algo=algo)
    agent = pkg.OnPolicyAgent(ctx, net, env, cfg, O.splitmix_states_fast(n, seed + 1), host_actions=False)
    env.reset_(is_force=True)
    agent.collect(T)
    return env, net, agent, p, n_in


def _flat_rollout(pkg, agent, n_in, T):
    Rl = pkg.learners
    S = agent.rollout(Rl.ROLL_STATE)
    nt = agent.n * T
    return (np.asfortranarray(S[:, :, :T]).reshape(n_in, nt, order="F"), agent.rollout(Rl.ROLL_ACTION).ravel(order="F"),
            agent.rollout(Rl.ROLL_LOGP).ravel(order="F"), agent.rollout(Rl.ROLL_ADV).ravel(order="F"),
            agent.rollout(Rl.ROLL_RET).ravel(order="F"), [float(v) for v in agent.rollout(Rl.ROLL_NORM)])


@pytest.mark.parametrize("n,T", [(64, 2), (1024, 32)], ids=["one-tile", "several-tiles-per-cta"])
def test_fused_optimiser_step_gradient(pkg, ctx, n, T):
    """OnPolicyAgent.update with one epoch of one minibatch (the whole rollout): K7 with the clip + Adam tail fused into its launch.
    NET_GRAD (the clipped gradient the tail applied) against the float64 gradient of the recorded rollout, clipped.  tanh trunks:
    no relu near-tie can sit in a rollout that cannot leave samples out (and the ratios are all ~1, far from the clip edges)."""
    env, net, agent, p, n_in = _rollout(pkg, ctx, "CartPole", n, T, R.KIND_CATEGORICAL, 2, 1, 77)
    try:
        l0 = ctx.launch_count()
        agent.update()
        launches = ctx.launch_count() - l0
        x, a, lp, adv, ret, (mean, inv_std) = _flat_rollout(pkg, agent, n_in, T)
        ref = G.loss_grad(p, n_in, 64, R.KIND_CATEGORICAL, 2, 1, x, a, lp, adv, ret, G.hyper(), mean, inv_std)
        assert not ref["ties"].any()
        G.check_grad(net.get(pkg.learners.NET_GRAD), clipped_ref(ref, 0.5), n_in, 64, R.KIND_CATEGORICAL, 2,
                     f"fused step n={n} T={T} ({launches} launches)")
    finally:
        agent.close(); net.close(); env.close()


def test_first_minibatch_of_the_benchmark_rollout(pkg, ctx):
    """PPO CartPole, 65 536 envs x T = 32 (the benchmark's shape): the gradient of the first minibatch (524 288 samples of the
    first epoch's permutation) of the recorded rollout, per block against float64.  The update computes the advantages, returns and
    their normalisation on the device; the gradient is then taken by ac_step with the update's initial parameters on exactly
    those inputs, less the samples the float64 reference flags as near-ties."""
    n, T, E, M = 65536, 32, 4, 4
    env, net, agent, p, n_in = _rollout(pkg, ctx, "CartPole", n, T, R.KIND_CATEGORICAL, 2, 0, 0x9E37, E=E, M=M)
    net2 = None
    try:
        nt = n * T
        perm = np.stack([np.random.default_rng(500 + e).permutation(nt) for e in range(E)]).astype(np.int32)
        agent.update(perm)
        x, a, lp, adv, ret, (mean, inv_std) = _flat_rollout(pkg, agent, n_in, T)
        idx = perm[0, :nt // M]
        hp = G.hyper()
        first = G.loss_grad_chunked(p, n_in, 64, R.KIND_CATEGORICAL, 2, 0, x[:, idx], a[idx], lp[idx], adv[idx], ret[idx], hp, mean, inv_std)
        ties = first["ties"]
        assert ties.mean() < 0.02, ties.sum()       # relu pre-activations within the bar of 0 (~1% of samples, two networks)
        idx = idx[~ties]
        ref = G.loss_grad_chunked(p, n_in, 64, R.KIND_CATEGORICAL, 2, 0, x[:, idx], a[idx], lp[idx], adv[idx], ret[idx], hp, mean, inv_std)
        net2 = pkg.Network(ctx, n_in, 64, 2, p, act=0, kind=R.KIND_CATEGORICAL)
        got = net2.ac_step(cfg_of(pkg, hp), x, a, lp, adv, ret, idx, mean, inv_std, apply_update=False)
        what = f"first minibatch of the 65536 x 32 rollout, B={idx.size} ({int(ties.sum())} near-ties left out)"
        G.check_grad(net2.get(pkg.learners.NET_GRAD), ref, n_in, 64, R.KIND_CATEGORICAL, 2, what)
        G.check_losses(got, ref, what)
    finally:
        if net2 is not None:
            net2.close()
        agent.close(); net.close(); env.close()
