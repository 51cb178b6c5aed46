"""CPU checks of the float64 PPO / A2C loss + backward reference (ac_grad_ref.py) and of the bar the loss + backward kernels are
held to.

- The reference's gradient and losses equal torch float64 autograd of the same loss, within round-off, on every sweep case.
- The float32 oracle (ac_loss_grad) meets 1e-5 (|g| + scale) per gradient entry and per loss on every case of the sweep.
- A NumPy emulation of the tensor-core backward (nn_tc.cu: GEMM2 / GEMM3 / GEMM4 on 3-term fp16 splits with the kernel's
  operand scales, per 128-sample tile) meets the same bar on the whole sweep, including a critic whose returns it fits to 1e-3
  and a near-deterministic policy: there the dP2 operand's lo part is an fp16 subnormal, but the honest scale of dz carries the
  rounding of V (or of the log-probabilities) and stays far above it.
- The emulation with a cross term lost (everywhere, or in the last K step only), without db2's lo column, without GEMM4's last K
  step, or with plain fp16 operands fails the bar on the "split-structured" case (one state repeated, every lo part of one sign,
  so a lost term adds up over the samples instead of cancelling)."""
import numpy as np
import pytest
import torch

import ac_grad_ref as G
import ac_ref as R
import oracle_lib as O

B = 640
HEADS = [("cat1", R.KIND_CATEGORICAL, 1), ("cat2", R.KIND_CATEGORICAL, 2), ("cat4", R.KIND_CATEGORICAL, 4), ("gauss", R.KIND_GAUSSIAN, 1)]


def sweep():
    out = []
    for name, kind, n_out in HEADS:
        for mag in G.MAGNITUDES:
            if (mag in G.GAUSS_ONLY and kind != R.KIND_GAUSSIAN) or (mag in G.CAT_ONLY and (kind != R.KIND_CATEGORICAL or n_out < 2)):
                continue
            acts = (R.TANH,) if mag == "pendulum" else (R.RELU,) if mag == "split-structured" else (R.RELU, R.TANH)
            for act in acts:
                algo = "a2c" if (mag not in G.PPO_ONLY and (n_out + act) % 2) else "ppo"
                out.append(pytest.param(kind, n_out, act, mag, algo, id=f"{name}-{mag}-{'relu' if act == R.RELU else 'tanh'}-{algo}"))
    return out


def _n_in(mag, n_out):
    return 3 if mag == "pendulum" else 1 + (n_out + 1) % 4


def _case(kind, n_out, act, mag, algo, H=64, b=B):
    n_in = _n_in(mag, n_out)
    case = G.make_batch(kind, n_in, n_out, act, H, mag, b, 7 + n_out, algo)
    return n_in, case, G.ref_of(case, n_in, H, kind, n_out, act)


def _torch_loss_grad(p, n_in, H, kind, n_out, act, case):
    """the same loss in torch float64, differentiated by autograd"""
    _, x, a, lp_old, adv, ret, hp, mean, inv_std = case
    Bn = x.shape[1]
    inv_B = float(np.float32(1) / np.float32(Bn))
    pt = torch.tensor(np.asarray(p, np.float64), requires_grad=True)
    rows = R.head_rows(kind, n_out)
    na = R.nparams(n_in, H, rows)
    fa, _ = __import__("q_ref").unpack_mlp(pt[:na], n_in, H, [1, 1] if kind == R.KIND_GAUSSIAN else [rows], act)
    fc, _ = __import__("q_ref").unpack_mlp(pt[na:], n_in, H, [1], act)
    xt = torch.tensor(np.asarray(x, np.float64).T)
    z, v = fa(xt), fc(xt)[:, 0]
    A = torch.tensor(adv, dtype=torch.float64)
    if hp["normalize_adv"]:
        A = (A - float(np.float32(mean))) * float(np.float32(inv_std))
    if kind == R.KIND_GAUSSIAN:
        mu, raw = z[:, 0], z[:, 1]
        sigma = torch.clamp(torch.nn.functional.softplus(raw), float(np.float32(hp["min_sigma"])), float(np.float32(hp["max_sigma"])))
        s = sigma + float(np.float32(1e-8))
        at = torch.tensor(a, dtype=torch.float64)
        logp_a = -0.5 * (torch.log(s * s) + (at - mu) ** 2 / (s * s) + R.LOG2PI)
        ent = torch.log(sigma) + 0.5 * (R.LOG2PI + 1.0)
    else:
        lp = torch.log_softmax(z, 1)
        logp_a = lp[torch.arange(Bn), torch.tensor(a.astype(np.int64) - 1)]
        ent = -(lp.exp() * lp).sum(1)
    if hp["algo"] == "a2c":
        l0 = -(logp_a * A)
    else:
        c = float(np.float32(hp["clip_range"]))
        r = torch.exp(logp_a - torch.tensor(lp_old, dtype=torch.float64))
        l0 = -torch.minimum(r * A, torch.clamp(r, float(np.float32(1 - np.float32(c))), float(np.float32(1 + np.float32(c)))) * A)
    sq = (torch.tensor(ret, dtype=torch.float64) - v) ** 2
    w = lambda k: float(np.float32(hp[k]))
    total = (w("w_actor") * l0.sum() + w("w_critic") * sq.sum() - w("w_entropy") * ent.sum()) * inv_B
    total.backward()
    losses = dict(actor_loss=l0.mean().item(), critic_loss=sq.mean().item(), entropy=ent.mean().item())
    return pt.grad.numpy(), losses


@pytest.mark.parametrize("kind,n_out,act,mag,algo", sweep())
def test_reference_matches_torch_autograd(kind, n_out, act, mag, algo):
    n_in, case, ref = _case(kind, n_out, act, mag, algo, b=256)
    g, losses = _torch_loss_grad(case[0], n_in, 64, kind, n_out, act, case)
    np.testing.assert_allclose(ref["grad"], g, rtol=0, atol=1e-11 * (np.abs(ref["scale"]).max() + 1e-300))
    assert np.all(np.abs(ref["grad"] - g) <= 1e-9 * (np.abs(g) + ref["scale"]))
    for k, v in losses.items():
        assert abs(ref["losses"][k][0] - v) <= 1e-11 * ref["losses"][k][1], k


def _oracle(kind, n_out, act, n_in, H, case):
    p, x, a, lp, adv, ret, hp, mean, inv_std = case
    oalgo = {("ppo", False): 0, ("a2c", True): 1, ("ppo", True): 2, ("a2c", False): 3}[(hp["algo"], kind == R.KIND_GAUSSIAN)]
    hy = O.hyper_array(clip_range=hp["clip_range"], w_actor=hp["w_actor"], w_critic=hp["w_critic"], w_entropy=hp["w_entropy"],
                       min_sigma=hp["min_sigma"], max_sigma=hp["max_sigma"], normalize_adv=int(hp["normalize_adv"]))
    return O.ac_loss_grad(oalgo, O.ac_desc(n_in, H, n_out, act, kind == R.KIND_GAUSSIAN), hy, p, x, a, lp, adv, ret, None, mean, inv_std)


@pytest.mark.parametrize("kind,n_out,act,mag,algo", sweep())
@pytest.mark.parametrize("H", [64, 128])
def test_oracle_meets_the_bar(oracle, H, kind, n_out, act, mag, algo):
    n_in, case, ref = _case(kind, n_out, act, mag, algo, H=H)
    g, losses = _oracle(kind, n_out, act, n_in, H, case)
    G.check_grad(g.astype(np.float32), ref, n_in, H, kind, n_out, f"oracle H={H} {mag}")
    G.check_losses({k: np.float32(v) for k, v in losses.items()}, ref, f"oracle H={H} {mag}")


@pytest.mark.parametrize("kind,n_out,act,mag,algo", [c for c in sweep() if c.values[0] != R.KIND_CATEGORICAL or c.values[1] <= 2])
def test_split_emulation_meets_the_bar(kind, n_out, act, mag, algo):
    """the tensor-core kernel's heads: categorical 1-2 and Gaussian"""
    n_in, case, ref = _case(kind, n_out, act, mag, algo)
    r = G.split_ratio(ref, case[1], act, n_in, 64, kind, n_out)
    assert r <= 0.5, r


def test_small_residuals_meet_the_honest_bar_not_the_naive_one():
    """the small-residual question: at |R - V| ~ 1e-3 the dP2 operand's lo part is subnormal, and against a bar that takes dz as
    exact (scale sum |terms| with |dz| in place of S_dz) the emulated split fails; against the honest bar it passes by a wide margin"""
    n_in, case, ref = _case(R.KIND_CATEGORICAL, 2, R.RELU, "critic-1e-3", "ppo", b=4096)
    assert G.split_ratio(ref, case[1], R.RELU, n_in, 64, R.KIND_CATEGORICAL, 2) < 0.05
    naive = dict(ref)
    t = ref["critic"]
    dz = t["dz"]
    g, _ = G._backward(t, case[1].astype(np.float64), G.V(dz.v, np.abs(dz.v)), R.RELU)
    naive_scale = np.concatenate([G.pack(g, R.KIND_Q)[1]])
    a = R.nparams(n_in, 64, 2)
    naive["scale"] = np.concatenate([ref["scale"][:a], naive_scale])
    e = G.split_backward(ref, "critic", case[1], R.RELU)
    names = {b[0]: (b[1], b[2]) for b in G.block_names(n_in, 64, R.KIND_CATEGORICAL, 2)}
    lo, hi = names["critic.W2"]
    r_naive = R.violations(e["W2"].T.ravel(), naive["grad"][lo:hi], naive["scale"][lo:hi]).max()
    assert e["dP2_max"] < 2.0 ** -3, e["dP2_max"]          # lo ~ 2^-11 of the operand < 2^-14: an fp16 subnormal
    assert r_naive > 1.0, r_naive


VARIANTS = {
    "gemm3-no-hi*lo": dict(gemm3=("hh", "lh")),
    "gemm3-no-lo*hi": dict(gemm3=("hh", "hl")),
    "gemm3-no-hi*lo-last-k": dict(gemm3_lost_last_k=("hl",)),
    "db2-no-lo": dict(db2_lo=False),
    "gemm4-no-last-k": dict(gemm4_lost_last_k=G.ALL_TERMS),
    "gemm4-no-lo*hi": dict(gemm4=("hh", "hl")),
    "fp16": dict(gemm2=("hh",), gemm3=("hh",), gemm4=("hh",), db2_lo=False),
}


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("name,kind,n_out", [h for h in HEADS if h[2] <= 2], ids=[h[0] for h in HEADS if h[2] <= 2])
def test_degraded_split_fails_the_bar(name, kind, n_out, variant):
    n_in, case, ref = _case(kind, n_out, R.RELU, "split-structured", "a2c")
    assert G.split_ratio(ref, case[1], R.RELU, n_in, 64, kind, n_out) < 0.1
    r = G.split_ratio(ref, case[1], R.RELU, n_in, 64, kind, n_out, **VARIANTS[variant])
    assert r > 2.0, r
