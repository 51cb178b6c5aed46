"""The tensor-core PPO / A2C loss + backward (K7) for an actor and a critic with different trunk activations: the
runtime-activation instantiation of the kernel.  The actor and critic trunks share no parameter, so each half of the
gradient of a mixed pair equals the one of a network whose two trunks both use that half's activation:
  * at 4 096 samples, against the CPU oracle run once with each activation (1e-5);
  * at 65 536 samples (512 tiles of 128: every CTA of either role runs several tiles, so the whole per-tile pipeline turns
    over: dP1 written from the GEMM2 accumulators, GEMM3 / GEMM4 behind the next tile's GEMM1, the double-buffered x^T
    operand and H1 signs), against the same-activation instantiations of the kernel, which the oracle suites pin.  (At this
    size the relu actor's gradient of this data set is 4e-4 away from the oracle on the CUDA-core kernel as well, so the
    oracle is not the yardstick there.)"""
import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu

REL = 1e-5
HIDDEN = 64


def rel_err(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)


def critic_nparams(n_in):
    return n_in * HIDDEN + HIDDEN + HIDDEN * HIDDEN + HIDDEN + HIDDEN + 1


@pytest.fixture(scope="module")
def tc_on(pkg, ctx):
    pkg._lib.check(ctx.lib.b200rl_set_tensor_cores(1))
    yield


def make_batch(kind, n_in, n_out, total, B, gaussian):
    rng = np.random.default_rng(29)
    desc = O.ac_desc(n_in, HIDDEN, n_out, 0, gaussian)
    params = O.glorot_params(desc, 31)
    params = params + 0.05 * rng.standard_normal(params.size).astype(np.float32)   # non-zero biases
    states = rng.standard_normal((n_in, total)).astype(np.float32)
    actions = rng.uniform(-2, 2, total).astype(np.float32) if gaussian else rng.integers(1, n_out + 1, total).astype(np.int32)
    logp_old = (-0.7 + 0.2 * rng.standard_normal(total)).astype(np.float32)
    adv = rng.standard_normal(total).astype(np.float32); ret = rng.standard_normal(total).astype(np.float32)
    idx = rng.permutation(total)[:B].astype(np.int32)
    mean, inv_std = O.adv_norm(adv)
    return params, (states, actions, logp_old, adv, ret, idx, mean, inv_std)


def device_step(pkg, ctx, algo, kind, n_in, n_out, act_a, act_c, params, batch):
    net = pkg.Network(ctx, n_in, HIDDEN, n_out, params, act=act_a, kind=kind)
    try:
        if act_c != act_a:
            pkg._lib.check(ctx.lib.b200rl_net_set_critic_act(net.h, act_c))
        cfg = pkg.onpolicy_config(clip_range=0.2, w_entropy=0.01, algo=algo, max_grad_norm=0.5)
        got = net.ac_step(cfg, *batch, apply_update=False)
        return net.get(pkg.learners.NET_GRAD), got
    finally:
        net.close()


# algo, kind, n_in, n_out, actor act, critic act (0 relu, 1 tanh)
CASES = [("ppo", 0, 4, 2, 0, 1), ("a2c", 1, 3, 1, 1, 0)]


@pytest.mark.parametrize("algo,kind,n_in,n_out,act_a,act_c", CASES)
def test_mixed_activation_loss_grad_matches_oracle(pkg, ctx, tc_on, algo, kind, n_in, n_out, act_a, act_c):
    gaussian = kind == pkg.KIND_GAUSSIAN
    params, batch = make_batch(kind, n_in, n_out, 5000, 4096, gaussian)
    g, got = device_step(pkg, ctx, algo, kind, n_in, n_out, act_a, act_c, params, batch)
    oalgo = {("ppo", 0): 0, ("a2c", 1): 1}[(algo, kind)]
    hyper = O.hyper_array(clip_range=0.2, w_entropy=0.01)
    g_a, l_a = O.ac_loss_grad(oalgo, O.ac_desc(n_in, HIDDEN, n_out, act_a, gaussian), hyper, params, *batch)
    g_c, l_c = O.ac_loss_grad(oalgo, O.ac_desc(n_in, HIDDEN, n_out, act_c, gaussian), hyper, params, *batch)
    na = params.size - critic_nparams(n_in)
    assert rel_err(g[:na], g_a[:na]) < REL, "actor half"
    assert rel_err(g[na:], g_c[na:]) < REL, "critic half"
    assert got["actor_loss"] == pytest.approx(l_a["actor_loss"], rel=REL, abs=1e-6)
    assert got["entropy"] == pytest.approx(l_a["entropy"], rel=REL, abs=1e-6)
    assert got["critic_loss"] == pytest.approx(l_c["critic_loss"], rel=REL, abs=1e-6)


@pytest.mark.parametrize("algo,kind,n_in,n_out,act_a,act_c", CASES)
def test_mixed_activation_many_tiles_per_cta_matches_same_activation_kernels(pkg, ctx, tc_on, algo, kind, n_in, n_out, act_a, act_c):
    gaussian = kind == pkg.KIND_GAUSSIAN
    params, batch = make_batch(kind, n_in, n_out, 80000, 65536, gaussian)
    g, got = device_step(pkg, ctx, algo, kind, n_in, n_out, act_a, act_c, params, batch)
    g_a, got_a = device_step(pkg, ctx, algo, kind, n_in, n_out, act_a, act_a, params, batch)
    g_c, got_c = device_step(pkg, ctx, algo, kind, n_in, n_out, act_c, act_c, params, batch)
    na = params.size - critic_nparams(n_in)
    # the same FP32 operations in the same order, up to the compiler's contraction choices in the two instantiations
    assert rel_err(g[:na], g_a[:na]) < 1e-6, "actor half"
    assert rel_err(g[na:], g_c[na:]) < 1e-6, "critic half"
    assert got["actor_loss"] == pytest.approx(got_a["actor_loss"], rel=1e-6, abs=1e-7)
    assert got["entropy"] == pytest.approx(got_a["entropy"], rel=1e-6, abs=1e-7)
    assert got["critic_loss"] == pytest.approx(got_c["critic_loss"], rel=1e-6, abs=1e-7)
