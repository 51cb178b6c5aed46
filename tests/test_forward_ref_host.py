"""CPU checks of the float64 forward reference (ac_ref.py) and of the bar the forward kernels are held to.

- The reference agrees with the float32 oracle (act_discrete, act_gaussian, critic_values, q_values) and with torch float64
  forwards (q_ref, dueling_ref) on every shape and magnitude of the sweep: per sample and row, within 1e-5 (|ref| + scale).
- A NumPy emulation of the tensor-core forward's 3-term fp16 split meets the same bar on the whole sweep.
- The emulation with one cross term lost (everywhere, or in the last K = 16 step only) or with plain fp16 operands fails it, on
  the "split-structured" case.  With random operands the lo parts have random signs and a lost term largely cancels in the sums
  (one lost K step lands near the bar, plain fp16 ~3x over it); the structured case makes every lo part positive, so they add
  up: one lost K step is ~5x the bar there, a whole lost term ~20x, while the correct split stays below 0.03 of it.  The GPU
  sweep carries the same case."""
import numpy as np
import pytest
import torch

import ac_ref as R
import dueling_ref
import oracle_lib as O
import q_ref

HEADS = [("cat", R.KIND_CATEGORICAL, n) for n in (1, 2, 3, 4)] + [("gauss", R.KIND_GAUSSIAN, 1)] + \
        [("q", R.KIND_Q, n) for n in (1, 2, 3, 4)] + [("duel", R.KIND_DUELING, n) for n in (1, 2, 3)]
HEAD_IDS = [f"{name}{n}" for name, _, n in HEADS]
MAG_CASES = [(m, a) for m, act in R.MAGNITUDES.items() for a in ((R.RELU, R.TANH) if act is None else (act,))]
MAG_IDS = [f"{m}-{'relu' if a == R.RELU else 'tanh'}" for m, a in MAG_CASES]
N = 256


def _nin(mag, default=4):
    return R.ENV_NIN.get(mag, default)


def _oracle_rows(kind, n_in, H, n_out, act, p, x):
    """the float32 oracle's outputs: dict name -> array, named as ac_ref.forward names them"""
    if kind == R.KIND_Q:
        return dict(q=O.q_values(O.ac_desc(n_in, H, n_out, act), p, x))
    if kind == R.KIND_DUELING:
        return dict(q=dueling_ref.oracle_q(p, n_in, H, n_out, act, x))
    seeds = O.splitmix_states_fast(x.shape[1], 7)
    if kind == R.KIND_GAUSSIAN:
        o = O.act_gaussian(O.ac_desc(n_in, H, 1, act, True), O.hyper_array(), p, x, seeds)
        return dict(mu=o["mu"], value=o["value"])
    o = O.act_discrete(O.ac_desc(n_in, H, n_out, act), p, x, seeds)
    return dict(heads=o["logits"], value=o["value"])


@pytest.mark.parametrize("mag,act", MAG_CASES, ids=MAG_IDS)
@pytest.mark.parametrize("name,kind,n_out", HEADS, ids=HEAD_IDS)
@pytest.mark.parametrize("H", [64, 128])
def test_reference_matches_the_oracle_and_torch(oracle, H, name, kind, n_out, mag, act):
    n_in = _nin(mag, 1 + (n_out + kind) % 4)
    p, x = R.make_case(kind, n_in, n_out, act, H, mag, N, seed=3 + n_out)
    ref = R.forward(p, n_in, H, kind, n_out, act, x)
    got = _oracle_rows(kind, n_in, H, n_out, act, p, x)
    for k, v in got.items():
        if k == "mu":
            R.check(v, ref["heads"][0][0], ref["heads"][1][0], f"oracle mu {mag}")
        else:
            R.check(v, *ref[k], f"oracle {k} {mag}")
    # torch float64 forwards: every head row, and the value network
    rows = R.head_rows(kind, n_out)
    na = R.nparams(n_in, H, rows)
    pa = p if kind in (R.KIND_Q, R.KIND_DUELING) else p[:na]
    if kind == R.KIND_DUELING:
        q64 = dueling_ref._torch_net(torch.tensor(pa, dtype=torch.float64), n_in, H, n_out, act)(torch.tensor(x.T, dtype=torch.float64))
        np.testing.assert_allclose(q64.numpy().T, ref["q"][0], rtol=1e-12, atol=1e-12 * np.abs(ref["q"][1]).max())
    else:
        fwd, _ = q_ref.unpack_mlp(torch.tensor(pa, dtype=torch.float64), n_in, H, [1, 1] if kind == R.KIND_GAUSSIAN else [rows], act)
        z = fwd(torch.tensor(x.T, dtype=torch.float64)).numpy().T
        zr = ref["q"] if kind == R.KIND_Q else ref["heads"]
        np.testing.assert_allclose(z, zr[0], rtol=1e-12, atol=1e-12 * np.abs(zr[1]).max())
    if "value" in ref:
        np.testing.assert_allclose(q_ref.q_values(p[na:], n_in, H, 1, act, x)[:, 0], ref["value"][0], rtol=1e-12,
                                   atol=1e-12 * np.abs(ref["value"][1]).max())
    if kind == R.KIND_CATEGORICAL:
        lp = torch.log_softmax(torch.tensor(ref["heads"][0]), 0).numpy()
        np.testing.assert_allclose(lp, ref["logp"][0], rtol=1e-12, atol=1e-12)


def test_gaussian_logp_matches_the_oracle_logpdf(oracle):
    rng = np.random.default_rng(5)
    mu, raw, a = rng.normal(0, 2, 300), rng.uniform(-3, 3, 300), rng.normal(0, 3, 300)
    lp, S = R.gaussian_logp(mu, raw, np.abs(mu), np.abs(raw), a)
    sigma = R.softplus(raw).astype(np.float32)
    got = np.array([O.lib().orc_normlogpdf1(float(m), float(s), float(b)) for m, s, b in zip(mu.astype(np.float32), sigma, a.astype(np.float32))])
    lp32, _ = R.gaussian_logp(mu.astype(np.float32), raw, 0 * S, 0 * S, a.astype(np.float32))
    R.check(got, lp32, S, "oracle normlogpdf1")
    assert np.all(np.isfinite(lp))


def _split_ratio(kind, n_in, n_out, act, mag, **kw):
    p, x = R.make_case(kind, n_in, n_out, act, 64, mag, N, seed=11 + n_out)
    rows = R.head_rows(kind, n_out)
    pa = p if kind in (R.KIND_Q, R.KIND_DUELING) else p[:R.nparams(n_in, 64, rows)]
    z, S = R.mlp(pa, n_in, 64, kind, n_out, act, x)
    got = R.split_mlp(pa, n_in, 64, kind, n_out, act, x, **kw)
    return R.violations(got, z, S).max()


@pytest.mark.parametrize("mag,act", MAG_CASES, ids=MAG_IDS)
@pytest.mark.parametrize("name,kind,n_out", HEADS, ids=HEAD_IDS)
def test_split_emulation_meets_the_bar(name, kind, n_out, mag, act):
    """the full 3-term split, on the head rows (the ones the kernels expose), at every shape and magnitude"""
    r = _split_ratio(kind, _nin(mag, 1 + (n_out + kind) % 4), n_out, act, mag)
    assert r <= 1.0, r


@pytest.mark.parametrize("variant", [dict(terms=("hh", "lh")), dict(terms=("hh", "hl")), dict(terms=("hh",)),
                                     dict(lost_last_k=("hl",)), dict(lost_last_k=("lh",))],
                         ids=["no-hi*lo", "no-lo*hi", "fp16", "no-hi*lo-last-k", "no-lo*hi-last-k"])
@pytest.mark.parametrize("name,kind,n_out", [h for h in HEADS if h[1] != R.KIND_DUELING],
                         ids=[i for i, h in zip(HEAD_IDS, HEADS) if h[1] != R.KIND_DUELING])
def test_degraded_split_fails_the_bar(name, kind, n_out, variant):
    """a lost term shows on every categorical, Gaussian and Q head of the structured case, by more than a factor 2 (the
    dueling combination Q_i = v + a_i - mean(a) cancels the advantage rows' common shift; only v carries it there)"""
    r = _split_ratio(kind, 4, n_out, R.RELU, "split-structured", **variant)
    assert r > 2.0, r
