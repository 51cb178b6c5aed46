"""Float64 restatement of the PPO / A2C loss + backward (policy.cuh sample_loss, the oracle's ac_loss_grad) with a magnitude scale
per gradient entry, and a NumPy emulation of the tensor-core backward's 3-term fp16 split (nn_tc.cu GEMM1-GEMM4).  Shared by the
CPU checks of the bar (test_backward_ref_host.py) and the GPU checks of the loss + backward kernels (test_backward_tc_gpu.py).

Scales.  Every quantity q carries a scale S_q >= |q| that bounds what float32 rounding can do to it (the forward's convention,
ac_ref.py), built by the rules
    a +- b: S_a + S_b          a * b: S_a |b| + |a| S_b          a / b: S_a / |b| + |a / b| S_b / |b|
    f(a):   |f'(a)| S_a + |f(a)|   (the argument's error through f, plus f's own rounding)
    a float32 input or constant c: |c|
applied to sample_loss operation by operation.  Each head output's dz so gets its own scale: the critic's
S = 2 w_critic inv_B (|R| + S_V) (the rounding of V rides on R - V), the actor's from the log-softmax / Gaussian log-density scales
of ac_ref (log-probabilities plus 1: the rounding of the sum of exps, whose largest term is 1) plus |terms|.  Backward through the layers (W exact, act' = relu mask or 1 - h^2 with scale 2 |h| S_h + 1 + h^2):
    S_dh2 = |W3|^T S_dz      S_dz2 = |d2| S_dh2 + |dh2| S_d2      S_dh1 = |W2|^T S_dz2      S_dz1 = |d1| S_dh1 + |dh1| S_d1
    S(dW3) = sum_s S_dz |h2| + |dz| S_h2    S(dW2) = sum_s S_dz2 |h1| + |dz2| S_h1    S(dW1) = sum_s S_dz1 |x|
    S(db3) = sum_s S_dz                      S(db2) = sum_s S_dz2                       S(db1) = sum_s S_dz1
The kernels are held to BAR (|g| + S) per gradient entry.  The losses: the means of the per-sample terms' scales.

Near-ties.  A sample whose float64 PPO ratio lies within BAR S_ratio of an edge 1 +- clip_range where the two sides select
different gradients, whose Gaussian softplus lies that close to min_sigma / max_sigma, or whose relu pre-activation lies that
close to 0, may legitimately take the other branch in float32.  ``loss_grad`` reports them (``ties``); the tests build batches
without them (or assert there are none) instead of widening the bar."""
import numpy as np

import ac_ref as R

BAR = R.BAR
f32 = np.float32


# ---------------------------------------------------------------------------------------------------------------------------
# value + scale arithmetic
class V:
    __slots__ = ("v", "s")

    def __init__(self, v, s=None):
        self.v = np.asarray(v, np.float64)
        self.s = np.abs(self.v) if s is None else np.asarray(s, np.float64)

    def __add__(a, b):
        b = _v(b); return V(a.v + b.v, a.s + b.s)
    __radd__ = __add__

    def __sub__(a, b):
        b = _v(b); return V(a.v - b.v, a.s + b.s)

    def __rsub__(a, b):
        return _v(b) - a

    def __mul__(a, b):
        b = _v(b); return V(a.v * b.v, a.s * np.abs(b.v) + np.abs(a.v) * b.s)
    __rmul__ = __mul__

    def __truediv__(a, b):
        b = _v(b)
        q = a.v / b.v
        return V(q, a.s / np.abs(b.v) + np.abs(q) * b.s / np.abs(b.v))

    def __rtruediv__(a, b):
        return _v(b) / a

    def __neg__(a):
        return V(-a.v, a.s)

    def __getitem__(a, k):
        return V(a.v[k], a.s[k])


def _v(x):
    return x if isinstance(x, V) else V(x)


def fn(f, df, a):
    y = f(a.v)
    return V(y, np.abs(df(a.v)) * a.s + np.abs(y))


def where(c, a, b):
    a, b = _v(a), _v(b)
    return V(np.where(c, a.v, b.v), np.where(c, a.s, b.s))


def vsum(xs):
    out = xs[0]
    for x in xs[1:]:
        out = out + x
    return out


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


# ---------------------------------------------------------------------------------------------------------------------------
# hyper-parameters as onpolicy_config / the oracle's hyper_array take them
def hyper(algo="ppo", clip_range=0.1, w_actor=1.0, w_critic=0.5, w_entropy=0.001, min_sigma=0.0, max_sigma=float("inf"),
          normalize_adv=True):
    return dict(algo=algo, clip_range=clip_range, w_actor=w_actor, w_critic=w_critic, w_entropy=w_entropy, min_sigma=min_sigma,
                max_sigma=max_sigma, normalize_adv=bool(normalize_adv))


def _c(x):
    """a float32 constant as the kernels hold it"""
    return float(np.float32(x))


def _trunk(p, n_in, H, kind, n_out, act, x):
    """forward intermediates of one network (ac_ref.mlp with the layers kept)"""
    W1, b1, W2, b2, W3, b3 = R.unpack(p, n_in, H, kind, n_out)
    z1 = W1 @ x + b1[:, None]; S1 = np.abs(W1) @ np.abs(x) + np.abs(b1)[:, None]
    h1, d1 = R._act(act, z1); Sh1 = d1 * S1 + (np.abs(h1) if act == R.TANH else 0.0)
    z2 = W2 @ h1 + b2[:, None]; S2 = np.abs(W2) @ Sh1 + np.abs(b2)[:, None]
    h2, d2 = R._act(act, z2); Sh2 = d2 * S2 + (np.abs(h2) if act == R.TANH else 0.0)
    z3 = W3 @ h2 + b3[:, None]; S3 = np.abs(W3) @ Sh2 + np.abs(b3)[:, None]
    ties = np.zeros(x.shape[1], bool)
    if act == R.RELU:
        ties = (np.abs(z1) <= BAR * S1).any(0) | (np.abs(z2) <= BAR * S2).any(0)
    return dict(W1=W1, W2=W2, W3=W3, z1=z1, S1=S1, h1=h1, d1=d1, Sh1=Sh1, z2=z2, h2=h2, d2=d2, Sh2=Sh2, z=V(z3, S3), ties=ties)


def _dact(act, d, h, Sh):
    """act'(z) as the kernels evaluate it (relu: the mask, exact; tanh: 1 - h^2) and its scale"""
    if act == R.RELU:
        return d, np.zeros_like(d)
    return d, 2.0 * np.abs(h) * Sh + 1.0 + h * h


def _backward(t, x, dz, act):
    """gradient blocks of one network from dz (rows, B) as V: dict block -> (value, scale), and the per-sample dP2 / dP1
    (the gradients of the layer-2 and layer-1 pre-activations)"""
    W1, W2, W3 = t["W1"], t["W2"], t["W3"]
    ax = np.abs(x)
    dh2 = W3.T @ dz.v; Sdh2 = np.abs(W3).T @ dz.s
    d2, Sd2 = _dact(act, t["d2"], t["h2"], t["Sh2"])
    dz2 = dh2 * d2; Sdz2 = Sdh2 * np.abs(d2) + np.abs(dh2) * Sd2
    dh1 = W2.T @ dz2; Sdh1 = np.abs(W2).T @ Sdz2
    d1, Sd1 = _dact(act, t["d1"], t["h1"], t["Sh1"])
    dz1 = dh1 * d1; Sdz1 = Sdh1 * np.abs(d1) + np.abs(dh1) * Sd1
    h1, Sh1, h2, Sh2 = t["h1"], t["Sh1"], t["h2"], t["Sh2"]
    g = dict(
        W1=(dz1 @ x.T, Sdz1 @ ax.T), b1=(dz1.sum(1), Sdz1.sum(1)),
        W2=(dz2 @ h1.T, Sdz2 @ np.abs(h1).T + np.abs(dz2) @ Sh1.T), b2=(dz2.sum(1), Sdz2.sum(1)),
        W3=(dz.v @ h2.T, dz.s @ np.abs(h2).T + np.abs(dz.v) @ Sh2.T), b3=(dz.v.sum(1), dz.s.sum(1)))
    return g, dict(dP2=dz2, dP1=dz1)


def pack(g, kind):
    """gradient blocks -> flat Flux order (the inverse of ac_ref.unpack), value and scale"""
    def flat(k):
        W3, b3 = g["W3"][k], g["b3"][k]
        if kind == R.KIND_GAUSSIAN:
            head = [W3[0], b3[:1], W3[1], b3[1:]]
        else:
            head = [W3.T.ravel(), b3]
        return np.concatenate([g["W1"][k].T.ravel(), g["b1"][k], g["W2"][k].T.ravel(), g["b2"][k]] + head)
    return flat(0), flat(1)


def block_names(n_in, H, kind, n_out):
    """(name, start, stop) of every parameter block of an actor-critic parameter vector, in flat order"""
    def one(pre, k, rows):
        sizes = [("W1", H * n_in), ("b1", H), ("W2", H * H), ("b2", H)]
        if k == R.KIND_GAUSSIAN:
            sizes += [("Wmu", H), ("bmu", 1), ("Wsigma", H), ("bsigma", 1)]
        else:
            sizes += [("W3", rows * H), ("b3", rows)]
        return [(f"{pre}.{n}", s) for n, s in sizes]
    out, o = [], 0
    for name, s in one("actor", kind, R.head_rows(kind, n_out)) + one("critic", R.KIND_Q, 1):
        out.append((name, o, o + s)); o += s
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# the loss
def _surrogate(hp, inv_B, logp_a, lp_old, A):
    """policy.cuh surrogate: (l0, d loss / d logp_a, ties)"""
    n = A.v.shape
    if hp["algo"] == "a2c":
        return -(logp_a * A), A * _c(-hp["w_actor"] * np.float32(inv_B)), np.zeros(n, bool)
    c = _c(hp["clip_range"])
    lo_e, hi_e = _c(1.0 - np.float32(c)), _c(1.0 + np.float32(c))
    ratio = fn(np.exp, np.exp, logp_a - lp_old)
    u = ratio * A
    rc = where(ratio.v < lo_e, lo_e, where(ratio.v > hi_e, hi_e, ratio))
    cc = rc * A
    l0 = -where(u.v <= cc.v, u, cc)
    inside = (ratio.v >= lo_e) & (ratio.v <= hi_e)
    gsel = where((u.v < cc.v) | inside, u, 0.0)
    band = BAR * ratio.s
    ties = ((np.abs(ratio.v - hi_e) <= band) & (A.v > 0)) | ((np.abs(ratio.v - lo_e) <= band) & (A.v < 0))
    return l0, gsel * _c(-hp["w_actor"] * np.float32(inv_B)), ties


def _actor_dz(hp, inv_B, kind, n_out, z, actions, lp_old, A):
    """(dz as V (rows, B), l0 V, entropy V, ties) of the actor head"""
    we = _c(hp["w_entropy"] * np.float32(inv_B))
    if kind == R.KIND_CATEGORICAL:
        lpv, lps = R.log_softmax(z.v, z.s)
        lp = V(lpv, lps + 1.0)      # + the float32 rounding of the sum of exps (its largest term is 1) through the log
        p = fn(np.exp, np.exp, lp)
        Hent = -vsum([p[o] * lp[o] for o in range(n_out)])
        a = np.asarray(actions, np.int64) - 1
        cols = np.arange(a.size)
        logp_a = V(lpv[a, cols], lps[a, cols])
        l0, dlogp, ties = _surrogate(hp, inv_B, logp_a, lp_old, A)
        rows = []
        for o in range(n_out):
            onehot = (a == o).astype(np.float64)
            rows.append(dlogp * (V(onehot) - p[o]) + we * (p[o] * (lp[o] + Hent)))
        return V(np.stack([r.v for r in rows]), np.stack([r.s for r in rows])), l0, Hent, ties
    mu, raw = z[0], z[1]
    sp = fn(R.softplus, sigmoid, raw)
    lo_s, hi_s = _c(hp["min_sigma"]), _c(hp["max_sigma"])
    clamped = (sp.v < lo_s) | (sp.v > hi_s)
    sigma = where(sp.v < lo_s, lo_s, where(sp.v > hi_s, hi_s, sp))
    ties = (np.abs(sp.v - lo_s) <= BAR * sp.s) | (np.abs(sp.v - hi_s) <= BAR * sp.s)
    a = V(np.asarray(actions, np.float64))
    s = sigma + _c(1e-8)
    var = s * s
    dd = a - mu
    logp_a = -0.5 * ((fn(np.log, lambda v: 1.0 / v, var) + dd * dd / var) + R.LOG2PI)
    Hent = fn(np.log, lambda v: 1.0 / v, sigma) + 0.5 * (R.LOG2PI + 1.0)
    l0, dlogp, t2 = _surrogate(hp, inv_B, logp_a, lp_old, A)
    dz0 = dlogp * (dd / (s * s))
    dsig = dlogp * (-1.0 / s + (dd * dd) / (s * s * s)) - we * (1.0 / sigma)
    dz1 = where(clamped, 0.0, dsig * fn(sigmoid, lambda r: sigmoid(r) * (1 - sigmoid(r)), raw))
    return V(np.stack([dz0.v, dz1.v]), np.stack([dz0.s, dz1.s])), l0, Hent, ties | t2


def loss_grad(p, n_in, H, kind, n_out, act, x, actions, logp_old, adv, ret, hp, adv_mean=0.0, adv_inv_std=1.0, B=None):
    """float64 losses and gradient of one minibatch (columns of x are the samples, in any order), as the kernels define them.
    Returns dict(grad, scale (flat, Flux order), losses {name: (value, scale)}, ties (B,), intermediates per role).
    B: the minibatch size when x holds only a slice of it (the gradient and losses are then that slice's share)."""
    p = np.asarray(p, np.float64)
    x = np.asarray(x, np.float64)
    B = x.shape[1] if B is None else B
    inv_B = float(np.float32(1.0) / np.float32(B))
    rows = R.head_rows(kind, n_out)
    na = R.nparams(n_in, H, rows)
    ta = _trunk(p[:na], n_in, H, kind, n_out, act, x)
    tc = _trunk(p[na:], n_in, H, R.KIND_Q, 1, act, x)
    adv = np.asarray(adv, np.float32)
    if hp["normalize_adv"]:
        A = (V(adv) - _c(adv_mean)) * _c(adv_inv_std)
    else:
        A = V(adv)
    lp_old = V(np.asarray(logp_old, np.float32) if logp_old is not None else np.zeros(B))
    dza, l0, Hent, ties = _actor_dz(hp, inv_B, kind, n_out, ta["z"], actions, lp_old, A)
    Rt = V(np.asarray(ret, np.float32))
    err = Rt - tc["z"][0]
    dzc = err * _c(-2.0 * hp["w_critic"] * np.float32(inv_B))
    dzc = V(dzc.v[None, :], dzc.s[None, :])
    ga, ia = _backward(ta, x, dza, act)
    gc, ic = _backward(tc, x, dzc, act)
    gav, gas = pack(ga, kind)
    gcv, gcs = pack(gc, R.KIND_Q)
    sq = err * err
    mean = lambda q: (q.v.sum() / B, q.s.sum() / B)
    la, lc, le = mean(l0), mean(sq), mean(Hent)
    wa, wc, we = _c(hp["w_actor"]), _c(hp["w_critic"]), _c(hp["w_entropy"])
    losses = dict(actor_loss=la, critic_loss=lc, entropy=le,
                  loss=(wa * la[0] + wc * lc[0] - we * le[0], wa * la[1] + wc * lc[1] + we * le[1]))
    return dict(grad=np.concatenate([gav, gcv]), scale=np.concatenate([gas, gcs]), losses=losses,
                ties=ties | ta["ties"] | tc["ties"], actor=dict(ta, dz=dza, **ia), critic=dict(tc, dz=dzc, **ic), inv_B=inv_B)


def check_grad(got, ref, n_in, H, kind, n_out, what, bar=BAR, blocks=None):
    """every gradient entry within bar (|g| + scale); the message names the block, the entry and err / tol of the worst entry
    of every failing block.  blocks: names to check (default all)."""
    got = np.asarray(got, np.float64)
    msgs = []
    for name, a, b in block_names(n_in, H, kind, n_out):
        if blocks is not None and name not in blocks:
            continue
        r = R.violations(got[a:b], ref["grad"][a:b], ref["scale"][a:b], bar)
        bad = ~(r <= 1.0)
        if bad.any():
            i = int(np.argmax(np.where(bad, r, -1.0)))
            msgs.append(f"{name}: {int(bad.sum())} of {b - a} entries, worst entry {i}: got {got[a + i]!r}, ref {ref['grad'][a + i]!r}, "
                        f"scale {ref['scale'][a + i]!r}, err / tol {r[i]:.3g}")
    if msgs:
        raise AssertionError(f"{what}: gradient outside {bar:g} (|g| + scale):\n  " + "\n  ".join(msgs))


def worst(got, ref, bar=BAR):
    return float(R.violations(got, ref["grad"], ref["scale"], bar).max())


def check_losses(got, ref, what, bar=BAR):
    for k, (v, s) in ref["losses"].items():
        tol = bar * (abs(v) + s)
        assert abs(float(got[k]) - v) <= tol, f"{what}: {k} = {float(got[k])!r}, float64 {v!r}, err / tol {abs(float(got[k]) - v) / tol:.3g}"


# ---------------------------------------------------------------------------------------------------------------------------
# the tensor-core backward (nn_tc.cu) in NumPy: GEMM2-GEMM4 on 3-term fp16 splits, per 128-sample tile, FP32 accumulators
TM = 128
K_SCALE = 64.0
ALL_TERMS = ("hh", "hl", "lh")     # A_hi*B_hi, A_hi*B_lo, A_lo*B_hi


def _split(v):
    return R._fp16_split(np.asarray(v, f32))


def _gemm_k(Ah, Al, Bh, Bl, terms, lost_last_k, k):
    """sum over the sample axis (K) of one 128-sample tile: A (M, k) x B (N, k)^T, the 3 terms in FP32; lost_last_k: terms that
    skip the last K = 16 step (samples 112..127 of the tile)"""
    ops = dict(hh=(Ah, Bh), hl=(Ah, Bl), lh=(Al, Bh))
    D = np.zeros((Ah.shape[0], Bh.shape[0]), f32)
    for t in terms:
        a, b = ops[t]
        kk = min(k, TM - 16) if t in lost_last_k else k
        D = (D + a[:, :kk] @ b[:, :kk].T).astype(f32)
    return D


def split_backward(ref, role, x, act, gemm3=ALL_TERMS, gemm3_lost_last_k=(), db2_lo=True, gemm2=ALL_TERMS, gemm4=ALL_TERMS,
                   gemm4_lost_last_k=()):
    """dW2, db2, dW1, db1 of one role ("actor" / "critic") as the tensor-core kernel computes them from float32 dz, H1, H2, x.
    Variants: gemm3 / gemm2 / gemm4: the split terms kept; *_lost_last_k: terms that skip the last K step of every tile; db2_lo:
    whether GEMM3's 1.0 column adds the dP2 lo part.  gemm*=("hh",) everywhere is plain fp16 operands."""
    t = ref[role]
    B = x.shape[1]
    inv_B = np.float32(ref["inv_B"])
    scale_base = np.float32(2.0 ** np.floor(np.log2(1.0 / inv_B)))
    sp = np.float32(scale_base * (4.0 if role == "critic" else 64.0))
    W2, W3 = t["W2"].astype(f32), t["W3"].astype(f32)
    dz = t["dz"].v.astype(f32)
    h2 = t["h2"].astype(f32)
    relu = act == R.RELU
    d2 = (t["z2"] > 0).astype(f32) if relu else (1 - h2 * h2).astype(f32)
    P = ((W3.T @ (dz * sp)).astype(f32) * d2).astype(f32)                       # dP2 operand (H, B)
    H1op = (np.maximum(t["z1"], 0) * K_SCALE).astype(f32) if relu else (np.tanh(t["z1"]).astype(f32) * f32(K_SCALE)).astype(f32)
    Ph, Pl = _split(P); Hh, Hl = _split(H1op)
    Wh, Wl = _split(W2 * f32(K_SCALE))
    # GEMM2: dH1 = W2^T dP2 (operand scale sp * 64), / 64, times act'(H1) from the signs / the split H1
    ops2 = dict(hh=(Wh, Ph), hl=(Wl, Ph), lh=(Wh, Pl))
    D2 = np.zeros((W2.shape[1], B), f32)
    for term in gemm2:
        w, a = ops2[term]
        D2 = (D2 + w.T @ a).astype(f32)
    D2 = (D2 * f32(1.0 / K_SCALE)).astype(f32)
    if relu:
        Q = np.where(t["z1"] > 0, D2, f32(0)).astype(f32)
    else:
        hs = ((Hh + Hl) * f32(1.0 / K_SCALE)).astype(f32)
        Q = (D2 * (f32(1) - hs * hs)).astype(f32)
    Qh, Ql = _split(Q)
    xs = np.asarray(x, f32)
    Xh, Xl = _split(xs * f32(K_SCALE))
    one = np.ones((1, B), f32)
    AccW2 = np.zeros((W2.shape[0], W2.shape[1]), f32)
    Accb2 = np.zeros(W2.shape[0], f32)
    AccW1 = np.zeros((W2.shape[1], xs.shape[0]), f32)
    Accb1 = np.zeros(W2.shape[1], f32)
    for t0 in range(0, B, TM):
        c = slice(t0, min(t0 + TM, B))
        k = c.stop - c.start
        AccW2 = (AccW2 + _gemm_k(Ph[:, c], Pl[:, c], Hh[:, c], Hl[:, c], gemm3, gemm3_lost_last_k, k)).astype(f32)
        Accb2 = (Accb2 + _gemm_k(Ph[:, c], Pl[:, c] if db2_lo else 0 * Pl[:, c], one[:, c], 0 * one[:, c], ("hh", "lh"), (), k)[:, 0]).astype(f32)
        AccW1 = (AccW1 + _gemm_k(Qh[:, c], Ql[:, c], Xh[:, c], Xl[:, c], gemm4, gemm4_lost_last_k, k)).astype(f32)
        Accb1 = (Accb1 + _gemm_k(Qh[:, c], Ql[:, c], one[:, c], 0 * one[:, c], tuple(x_ for x_ in gemm4 if x_ != "hl"), gemm4_lost_last_k, k)[:, 0]).astype(f32)
    return dict(W2=(AccW2 * f32(1.0 / (sp * K_SCALE))).astype(f32), b2=(Accb2 * f32(1.0 / sp)).astype(f32),
                W1=(AccW1 * f32(1.0 / (sp * K_SCALE))).astype(f32), b1=(Accb1 * f32(1.0 / sp)).astype(f32),
                dP2_max=float(np.abs(P).max()), dP1_max=float(np.abs(Q).max()))


def split_ratio(ref, x, act, n_in, H, kind, n_out, **variant):
    """max err / tol of the emulated W1, b1, W2, b2 blocks of both roles against the float64 reference"""
    names = {b[0]: (b[1], b[2]) for b in block_names(n_in, H, kind, n_out)}
    worst_r = 0.0
    for role in ("actor", "critic"):
        e = split_backward(ref, role, x, act, **variant)
        for blk, flat in (("W1", e["W1"].T.ravel()), ("b1", e["b1"]), ("W2", e["W2"].T.ravel()), ("b2", e["b2"])):
            a, b = names[f"{role}.{blk}"]
            worst_r = max(worst_r, float(R.violations(flat, ref["grad"][a:b], ref["scale"][a:b]).max()))
    return worst_r


# ---------------------------------------------------------------------------------------------------------------------------
# batches of the magnitude sweep
# name -> what it exercises
MAGNITUDES = {
    "unit": "N(0, 1) advantages and returns, near-uniform policy",
    "critic-1e-2": "returns R = V + N(0, 1e-2): a critic that fits its returns",
    "critic-1e-3": "returns R = V + N(0, 1e-3)",
    "critic-1e-2-v50": "|V| ~ 50, R = V + N(0, 1e-2)",
    "critic-1e-3-v50": "|V| ~ 50, R = V + N(0, 1e-3)",
    "deterministic": "p_max ~ 0.999: a near-deterministic policy (categorical)",
    "adv-100": "normalize_adv = 0, |A| up to ~100",
    "adv-0": "advantages exactly 0: only the entropy term",
    "clip-high": "PPO ratios all above 1 + clip_range",
    "clip-low": "PPO ratios all below 1 - clip_range",
    "clip-inside": "PPO ratios all inside the clip range",
    "clip-straddle": "PPO ratios on both sides of both edges",
    "sigma-min": "Gaussian sigma clamped at min_sigma",
    "sigma-max": "Gaussian sigma clamped at max_sigma",
    "pendulum": "Pendulum observations and returns down to ~-1600, tanh",
    "split-structured": "one state repeated, every split lo part of one sign (a lost term adds up instead of cancelling), most of\n"
                        "                        the critic's gradient in the last 16 samples of every tile",
}
# magnitudes that only make sense for one head (categorical / Gaussian) or one algorithm
GAUSS_ONLY = {"sigma-min", "sigma-max"}
CAT_ONLY = {"deterministic"}
PPO_ONLY = {"clip-high", "clip-low", "clip-inside", "clip-straddle"}


def _values(p, n_in, H, kind, n_out, act, x):
    rows = R.head_rows(kind, n_out)
    na = R.nparams(n_in, H, rows)
    z, _ = R.mlp(np.asarray(p, np.float64)[:na], n_in, H, kind, n_out, act, x)
    v, _ = R.mlp(np.asarray(p, np.float64)[na:], n_in, H, R.KIND_Q, 1, act, x)
    return z, v[0]


def make_batch(kind, n_in, n_out, act, H, mag, B, seed, algo="ppo"):
    """(params, x (n_in, B), actions, logp_old, adv, ret, hyper, adv_mean, adv_inv_std) of one sweep case, float32, with no
    near-tie sample (drawn with spares; the samples the float64 reference flags are dropped)"""
    rng = np.random.default_rng(seed)
    fmag = {"pendulum": "pendulum", "split-structured": "split-structured"}.get(mag, "unit")
    n = B + B // 8 + 16
    p, x = R.make_case(kind, n_in, n_out, act, H, fmag, n, seed)
    p = p.astype(np.float64)
    rows = R.head_rows(kind, n_out)
    na = R.nparams(n_in, H, rows)
    hp = hyper(algo=algo, clip_range=0.2, w_entropy=0.01)
    if mag == "split-structured":
        x = np.repeat(x[:, :1], n, axis=1)
        # grid-aligned positive observations: the x operand's lo parts all of one sign too
        x[:] = R._on_fp16_grid_plus(rng, n_in, 32.0, 36.0)[:, None]
        hp.update(normalize_adv=False, algo="a2c" if algo == "a2c" else "ppo", clip_range=10.0)
    if mag == "critic-1e-2-v50" or mag == "critic-1e-3-v50":
        p[na + R._offsets(n_in, H, 1)["head"].stop - 1] = 50.0          # critic b3: |V| ~ 50
    if mag == "deterministic":
        o = R._offsets(n_in, H, rows)["head"]
        p[o.stop - n_out] += 7.0 + np.log(n_out)                         # b3[0]: p_max ~ 0.999
    p = p.astype(np.float32)
    if kind == R.KIND_GAUSSIAN and mag in ("sigma-min", "sigma-max"):
        z, _ = _values(p, n_in, H, kind, n_out, act, x)
        sp = R.softplus(z[1])
        if mag == "sigma-min":
            hp["min_sigma"] = float(np.float32(sp.max() * 1.5))
        else:
            hp["max_sigma"] = float(np.float32(sp.min() / 1.5))
    z, v = _values(p, n_in, H, kind, n_out, act, x)
    if kind == R.KIND_GAUSSIAN:
        sig = np.clip(R.softplus(z[1]), hp["min_sigma"], hp["max_sigma"])
        actions = (z[0] + sig * rng.standard_normal(n)).astype(np.float32)
    elif mag in ("deterministic", "split-structured"):
        actions = np.where(rng.uniform(size=n) < 0.9, 1, 1 + rng.integers(0, n_out, n)).astype(np.int32)
        if mag == "split-structured":
            actions[:] = 1
    else:
        actions = rng.integers(1, n_out + 1, n).astype(np.int32)
    # the log-probability of the action under the current parameters (float64), to place the PPO ratios
    if kind == R.KIND_GAUSSIAN:
        lp_now, _ = R.gaussian_logp(z[0], z[1], 0 * z[0], 0 * z[1], actions, hp["min_sigma"], hp["max_sigma"])
    else:
        lpv, _ = R.log_softmax(z, 0 * z)
        lp_now = lpv[actions - 1, np.arange(n)]
    log_r = {"clip-high": rng.uniform(np.log(1.3), np.log(2.0), n), "clip-low": rng.uniform(np.log(0.5), np.log(0.75), n),
             "clip-inside": rng.uniform(np.log(0.85), np.log(1.15), n),
             "clip-straddle": rng.uniform(np.log(0.6), np.log(1.5), n)}.get(mag, 0.2 * rng.standard_normal(n))
    if mag == "split-structured":
        log_r = np.zeros(n)
    logp_old = (lp_now - log_r).astype(np.float32)
    adv = rng.standard_normal(n)
    if mag == "adv-100":
        hp["normalize_adv"] = False
        adv = 100.0 * rng.uniform(-1, 1, n)
    elif mag == "adv-0":
        adv = np.zeros(n)
    elif mag == "split-structured":
        adv = np.ones(n)
    elif mag == "pendulum":
        adv = 50.0 * rng.standard_normal(n)
    adv = adv.astype(np.float32)
    resid = {"critic-1e-2": 1e-2, "critic-1e-3": 1e-3, "critic-1e-2-v50": 1e-2, "critic-1e-3-v50": 1e-3}.get(mag)
    if resid is not None:
        ret = v + resid * rng.standard_normal(n)
    elif mag == "pendulum":
        ret = -rng.uniform(0.0, 1600.0, n)
    elif mag == "split-structured":
        # residual 100 on samples 112..127 of every 128-sample tile (the last K = 16 step of GEMM3 / GEMM4), 1 elsewhere: the last
        # K step carries most of the gradient, so a term lost there alone shows too
        ret = v + np.where(np.arange(n) % 128 >= 112, 100.0, 1.0)
    else:
        ret = rng.standard_normal(n)
    ret = ret.astype(np.float32)
    mean, inv_std = 0.0, 1.0
    if hp["normalize_adv"]:
        a64 = adv.astype(np.float64)
        mean, inv_std = float(np.float32(a64.mean())), float(np.float32(1.0 / (a64.std() + 1e-8)))
    ref = loss_grad(p, n_in, H, kind, n_out, act, x, actions, logp_old, adv, ret, hp, mean, inv_std)
    keep = np.flatnonzero(~ref["ties"])[:B]
    assert keep.size == B, (mag, int(ref["ties"].sum()))
    return p, np.ascontiguousarray(x[:, keep], np.float32), actions[keep], logp_old[keep], adv[keep], ret[keep], hp, mean, inv_std


def loss_grad_chunked(p, n_in, H, kind, n_out, act, x, actions, logp_old, adv, ret, hp, adv_mean=0.0, adv_inv_std=1.0, chunk=65536):
    """loss_grad of a large minibatch in slices of samples (bounded host memory): gradient, scale, losses and ties"""
    B = x.shape[1]
    out = None
    for a in range(0, B, chunk):
        c = slice(a, min(a + chunk, B))
        r = loss_grad(p, n_in, H, kind, n_out, act, x[:, c], actions[c], logp_old[c], adv[c], ret[c], hp, adv_mean, adv_inv_std, B=B)
        if out is None:
            out = dict(grad=r["grad"], scale=r["scale"], losses=r["losses"], ties=[r["ties"]])
        else:
            out["grad"] = out["grad"] + r["grad"]; out["scale"] = out["scale"] + r["scale"]
            out["losses"] = {k: (v[0] + r["losses"][k][0], v[1] + r["losses"][k][1]) for k, v in out["losses"].items()}
            out["ties"].append(r["ties"])
    out["ties"] = np.concatenate(out["ties"])
    return out


def ref_of(case, n_in, H, kind, n_out, act, idx=None):
    """the float64 reference of a make_batch case (columns idx of it, when given)"""
    p, x, a, lp, adv, ret, hp, mean, inv_std = case
    if idx is not None:
        x, a, lp, adv, ret = x[:, idx], a[idx], lp[idx], adv[idx], ret[idx]
    return loss_grad(p, n_in, H, kind, n_out, act, x, a, lp, adv, ret, hp, mean, inv_std)
