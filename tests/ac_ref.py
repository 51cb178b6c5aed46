"""Float64 restatement of the forward pass of every network kind the kernels run, with a magnitude scale per output, and a NumPy
emulation of the tensor-core forward's 3-term fp16 split (tc_fwd.cuh).  Shared by the CPU checks of the bar itself
(test_forward_ref_host.py) and the GPU checks of the forward kernels (test_forward_tc_gpu.py).

Network = Dense(in, H, act) -> Dense(H, H, act) -> head rows, flat in Flux.destructure order (nn.cuh):
  categorical / value / Q: W3 (n_out x H), b3;  Gaussian: Wmu, bmu, Wsig, bsig;  dueling: Wv, bv, Wa (n x H), ba.
An actor-critic parameter vector is the actor's followed by the critic's (value head).

``forward`` returns, for each output, its float64 value and a **magnitude scale**: the same sum with every term in absolute
value, carried through the layers with the activation derivative (S_h = act'(z) S_z, plus |h| for tanh, whose evaluation rounds;
relu is exact).  A float32 computation whose every operation is accurate to a few ulp of its operands stays within
~1e-6 (|ref| + scale); the forward kernels are held to ``BAR`` = 1e-5 of it, per sample and per output row (``check``)."""
import numpy as np

BAR = 1e-5
LOG2PI = float(np.log(2.0 * np.pi))
RELU, TANH = 0, 1
KIND_CATEGORICAL, KIND_GAUSSIAN, KIND_Q, KIND_DUELING = 0, 1, 2, 3   # learners.KIND_*


def head_rows(kind, n_out):
    """rows of the head: categorical / Q n_out, Gaussian 2 {mu, raw sigma}, dueling n_out + 1 {v, a_1 .. a_n}"""
    return {KIND_GAUSSIAN: 2, KIND_DUELING: n_out + 1}.get(kind, n_out)


def nparams(n_in, H, rows):
    return H * n_in + H + H * H + H + rows * H + rows


def unpack(p, n_in, H, kind, n_out):
    """one network's flat parameters -> (W1 (H, n_in), b1, W2 (H, H), b2, W3 (rows, H), b3) in float64"""
    p = np.asarray(p, np.float64)
    o = 0

    def take(n):
        nonlocal o
        v = p[o:o + n]; o += n
        return v
    W1 = take(H * n_in).reshape(n_in, H).T; b1 = take(H)
    W2 = take(H * H).reshape(H, H).T; b2 = take(H)
    if kind == KIND_GAUSSIAN:                   # Wmu (1 x H), bmu, Wsig (1 x H), bsig
        wm, bm, ws, bs = take(H), take(1), take(H), take(1)
        W3, b3 = np.stack([wm, ws]), np.concatenate([bm, bs])
    elif kind == KIND_DUELING:                  # Wv (1 x H), bv, Wa (n x H), ba
        wv, bv = take(H), take(1)
        wa, ba = take(n_out * H).reshape(H, n_out).T, take(n_out)
        W3, b3 = np.concatenate([wv[None, :], wa]), np.concatenate([bv, ba])
    else:
        W3, b3 = take(n_out * H).reshape(H, n_out).T, take(n_out)
    assert o == p.size, (o, p.size)
    return W1, b1, W2, b2, W3, b3


def _act(act, z):
    """h = act(z) and the scale factor of its input: act'(z) (relu: 1 where z > 0)"""
    if act == RELU:
        return np.maximum(z, 0.0), (z > 0).astype(np.float64)
    h = np.tanh(z)
    return h, 1.0 - h * h


def mlp(p, n_in, H, kind, n_out, act, x):
    """x (n_in, N) -> head rows z (rows, N) and their scale S (rows, N), float64"""
    W1, b1, W2, b2, W3, b3 = unpack(p, n_in, H, kind, n_out)
    x = np.asarray(x, np.float64)
    z1 = W1 @ x + b1[:, None]; S1 = np.abs(W1) @ np.abs(x) + np.abs(b1)[:, None]
    h1, d1 = _act(act, z1); Sh1 = d1 * S1 + (np.abs(h1) if act == TANH else 0.0)
    z2 = W2 @ h1 + b2[:, None]; S2 = np.abs(W2) @ Sh1 + np.abs(b2)[:, None]
    h2, d2 = _act(act, z2); Sh2 = d2 * S2 + (np.abs(h2) if act == TANH else 0.0)
    z3 = W3 @ h2 + b3[:, None]; S3 = np.abs(W3) @ Sh2 + np.abs(b3)[:, None]
    return z3, S3


def dueling_q(z, S):
    """head rows {v, a_1 .. a_n} -> Q_i = (v + a_i) - mean(a) and its scale"""
    v, a, Sv, Sa = z[0], z[1:], S[0], S[1:]
    return (v + a) - a.mean(0), Sv + Sa + Sa.mean(0)


def log_softmax(z, S):
    """log-softmax of the rows of z and its scale: the logits' scales through d lp_o / d z_k = [o == k] - p_k, and the size of
    the terms the kernel rounds, |z_o - max z| and log Σ exp(z - max z)"""
    m = z.max(0)
    ls = np.log(np.exp(z - m).sum(0))
    lp = (z - m) - ls
    p = np.exp(lp)
    return lp, S + (p * S).sum(0) + np.abs(z - m) + np.abs(ls)


def softplus(x):
    return np.logaddexp(0.0, x)


def gaussian_logp(mu, raw, Smu, Sraw, a, min_sigma=0.0, max_sigma=np.inf):
    """log-density of the given action a under N(mu, sigma), sigma = clamp(softplus(raw), min_sigma, max_sigma), as policy.cuh's
    normlogpdf1 (eps = 1e-8), and its scale: the head scales through d logp / d mu and d logp / d raw, and the size of its terms"""
    sp = softplus(raw)
    sigma = np.clip(sp, min_sigma, max_sigma)
    clamped = (sp < min_sigma) | (sp > max_sigma)
    a = np.asarray(a, np.float64)
    s = sigma + 1e-8
    v = s * s
    d = a - mu
    lp = -0.5 * (np.log(v) + d * d / v + LOG2PI)
    dsig = np.where(clamped, 0.0, np.abs(-1.0 / s + d * d / (s * s * s)) / (1.0 + np.exp(-raw)))
    return lp, np.abs(d) / v * Smu + dsig * Sraw + 0.5 * (np.abs(np.log(v)) + d * d / v + LOG2PI)


def forward(p, n_in, H, kind, n_out, act, x):
    """float64 outputs of a network given as learners.Network takes it: dict of (value, scale) pairs.
    categorical: heads (logits), logp (log-softmax rows), value;  Gaussian: heads {mu, raw sigma}, value;  Q / dueling: q"""
    p = np.asarray(p, np.float64)
    rows = head_rows(kind, n_out)
    if kind in (KIND_Q, KIND_DUELING):
        z, S = mlp(p, n_in, H, kind, n_out, act, x)
        return dict(q=dueling_q(z, S) if kind == KIND_DUELING else (z, S))
    na = nparams(n_in, H, rows)
    z, S = mlp(p[:na], n_in, H, kind, n_out, act, x)
    v, Sv = mlp(p[na:], n_in, H, KIND_Q, 1, act, x)
    out = dict(heads=(z, S), value=(v[0], Sv[0]))
    if kind == KIND_CATEGORICAL:
        out["logp"] = log_softmax(z, S)
    return out


def violations(got, ref, scale, bar=BAR):
    """|got - ref| / (bar (|ref| + scale)) elementwise (NaN / inf in got: inf)"""
    got = np.asarray(got, np.float64)
    tol = bar * (np.abs(ref) + scale)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.abs(got - ref) / np.where(tol > 0, tol, np.finfo(np.float64).tiny)
    return np.where(np.isfinite(got), r, np.inf)


def check(got, ref, scale, what, bar=BAR):
    """assert every output within bar (|ref| + scale), per sample and per row; the message names the worst element"""
    r = violations(got, ref, scale, bar)
    bad = ~(r <= 1.0)
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, r, -1.0)), r.shape)
        g = np.asarray(got, np.float64)[i]
        raise AssertionError(f"{what}: {int(bad.sum())} of {r.size} outputs outside {bar:g} (|ref| + scale); worst at "
                             f"{'(row, sample) ' if r.ndim == 2 else 'sample '}{tuple(int(k) for k in i)}: got {g!r}, ref {ref[i]!r}, "
                             f"scale {scale[i]!r}, err / tol {r[i]:.3g}")


def margin_of(rows, tol):
    """top-1 minus top-2 of rows (k, N), and whether the first maximum is decided by more than 4x the rows' largest tolerance"""
    if rows.shape[0] == 1:
        return np.full(rows.shape[1], np.inf), np.ones(rows.shape[1], bool)
    top = np.sort(rows, 0)
    m = top[-1] - top[-2]
    return m, m > 4.0 * tol.max(0)


# ---------------------------------------------------------------------------------------------------------------------------
# the 3-term fp16 split of tc_fwd.cuh in NumPy
K_SCALE = np.float32(64.0)


def _fp16_split(v):
    """split2 / fill_w2_image: hi = fp16(v), lo = fp16(v - hi) (v float32, the subtraction in float32)"""
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float32), lo.astype(np.float32)


def split_mlp(p, n_in, H, kind, n_out, act, x, terms=("hh", "hl", "lh"), lost_last_k=()):
    """head rows (rows, N) as the tensor-core forward computes them, in float32:
      layer 1 in float32 with the relu scale folded into W1 / b1 (tanh: fp32(64 tanh(z))), H1 and W2 as x_hi = fp16(64 x),
      x_lo = fp16(64 x - x_hi), the products of ``terms`` (hh = H1_hi*W2_hi, hl = H1_hi*W2_lo, lh = H1_lo*W2_hi) accumulated in
      float32, the 1/4096 undone before b2, then act and the head in float32.
    terms=("hh",) is fp16 in place of the split.  lost_last_k: terms that skip the last K = 16 step (inputs 48..63 of layer 2)."""
    f32 = np.float32
    W1, b1, W2, b2, W3, b3 = (a.astype(f32) for a in unpack(p, n_in, H, kind, n_out))
    x = np.asarray(x, f32)
    s1 = K_SCALE if act == RELU else f32(1.0)
    z1 = ((W1 * s1) @ x + (b1 * s1)[:, None]).astype(f32)
    h1 = np.maximum(z1, f32(0.0)) if act == RELU else (np.tanh(z1).astype(f32) * K_SCALE).astype(f32)
    ah, al = _fp16_split(h1)
    wh, wl = _fp16_split((W2 * K_SCALE).astype(f32))
    ops = dict(hh=(wh, ah), hl=(wl, ah), lh=(wh, al))
    D = np.zeros((H, x.shape[1]), f32)
    for t in terms:
        w, a = ops[t]
        k = H - 16 if t in lost_last_k else H
        D += w[:, :k] @ a[:k]
    z2 = (D * f32(1.0 / 4096.0) + b2[:, None]).astype(f32)
    h2 = np.maximum(z2, f32(0.0)) if act == RELU else np.tanh(z2).astype(f32)
    return (W3 @ h2 + b3[:, None]).astype(f32)


# ---------------------------------------------------------------------------------------------------------------------------
# parameters and observations of the magnitude sweep
# name -> activation it runs with (None: both) and what it exercises
MAGNITUDES = {
    "unit": None,               # glorot + 0.05 noise, N(0, 1) observations
    "h1-500": RELU,             # relu H1 peaks near 500 (the operand 64 H1 near 32 000, inside fp16's 65504)
    "tanh-saturated": TANH,     # |z| of both tanh layers up to ~40: the trunk saturates
    "w2-8": None,               # max |W2| = 8 (the operand 64 W2 = 512)
    "tiny": None,               # |obs|, H1 and |W2| ~ 1e-3: the operands' lo parts are fp16 subnormals
    "pendulum": TANH,           # Pendulum observations: cos, sin, angular velocity up to 8
    "mountaincar": RELU,        # MountainCar observations: position -1.2 .. 0.6, velocity up to 0.07
    "split-structured": RELU,   # every lo part positive (below), so a lost split term shifts every output the same way
}
ENV_NIN = {"pendulum": 3, "mountaincar": 2}


def _offsets(n_in, H, rows):
    o1 = H * n_in
    o2 = o1 + H
    o3 = o2 + H * H
    return dict(W1=slice(0, o1), b1=slice(o1, o2), W2=slice(o2, o3), b2=slice(o3, o3 + H), head=slice(o3 + H, nparams(n_in, H, rows)))


def _glorot(rng, n_in, H, rows):
    parts = []
    for o, i in ((H, n_in), (H, H), (rows, H)):
        lim = np.sqrt(6.0 / (i + o))
        parts += [rng.uniform(-lim, lim, o * i), np.zeros(o)]
    return np.concatenate(parts)


def _on_fp16_grid_plus(rng, n, lo, hi, frac=0.45):
    """n values v with 64 v = g + frac ulp(g), g an fp16 value in [lo, hi) (the bottom of a binade: lo part / value ~ 4e-4)"""
    g = rng.uniform(lo, hi, n).astype(np.float16).astype(np.float64)
    ulp = np.spacing(g.astype(np.float16)).astype(np.float64)
    return ((g + frac * ulp) / 64.0).astype(np.float32)


def _one_net(rng, n_in, H, kind, n_out, act, mag, x):
    rows = head_rows(kind, n_out)
    p = _glorot(rng, n_in, H, rows) + 0.05 * rng.standard_normal(nparams(n_in, H, rows))
    s = _offsets(n_in, H, rows)
    if mag == "h1-500" or mag == "tanh-saturated":
        top = 500.0 if mag == "h1-500" else 40.0
        z1 = np.abs(unpack(p, n_in, H, kind, n_out)[0] @ x + p[s["b1"]][:, None]).max()
        p[s["W1"]] *= top / z1; p[s["b1"]] *= top / z1
        if mag == "tanh-saturated":
            p[s["W2"]] *= 40.0 / np.sqrt(H)
    elif mag == "w2-8":
        p[s["W2"]] *= 8.0 / np.abs(p[s["W2"]]).max()
    elif mag == "tiny":
        p[s["b1"]] *= 1e-3 / np.abs(p[s["b1"]]).max()
        p[s["W2"]] *= 1e-3 / np.abs(p[s["W2"]]).max()
        p[s["b2"]] *= 1e-6
    elif mag == "split-structured":
        # relu H1 ~ b1 with 64 b1 = g + 0.45 ulp(g) on [32, 36), W2 > 0 with 64 W2 on [1, 1.125) the same way, W1 ~ 1e-7 (H1's lo
        # parts stay put), b2 = 0, head weights >= 0: both cross terms are ~4e-4 of hi*hi and add up instead of cancelling
        p[s["W1"]] = 1e-7 * rng.standard_normal(H * n_in)
        p[s["b1"]] = _on_fp16_grid_plus(rng, H, 32.0, 36.0)
        p[s["W2"]] = _on_fp16_grid_plus(rng, H * H, 1.0, 1.125)
        p[s["b2"]] = 0.0
        p[s["head"]] = np.abs(p[s["head"]])
    p = p.astype(np.float32)
    if kind == KIND_GAUSSIAN:   # raw sigma scaled into [-3, 3]: sigma = softplus(raw) neither underflows nor dwarfs the action
        z, _ = mlp(p, n_in, H, kind, n_out, act, x)
        c = 3.0 / max(np.abs(z[1]).max(), 1e-30)
        o = s["head"].start
        p[o + H + 1:o + 2 * H + 2] *= np.float32(c)
    return p


def observations(mag, n_in, N, seed):
    rng = np.random.default_rng(seed)
    if mag == "pendulum":
        th = rng.uniform(-np.pi, np.pi, N)
        x = np.stack([np.cos(th), np.sin(th), rng.uniform(-8.0, 8.0, N)])
    elif mag == "mountaincar":
        x = np.stack([rng.uniform(-1.2, 0.6, N), rng.uniform(-0.07, 0.07, N)])
    else:
        x = rng.standard_normal((n_in, N)) * (1e-3 if mag == "tiny" else 1.0)
    return x.astype(np.float32)


def make_case(kind, n_in, n_out, act, H, mag, N, seed):
    """(params as learners.Network takes them, observations (n_in, N)) of one sweep case"""
    if mag in ENV_NIN:
        assert n_in == ENV_NIN[mag]
    x = observations(mag, n_in, N, seed)
    rng = np.random.default_rng(seed + 1)
    xs = x[:, :min(N, 4096)].astype(np.float64)
    if kind in (KIND_Q, KIND_DUELING):
        return _one_net(rng, n_in, H, kind, n_out, act, mag, xs), x
    return np.concatenate([_one_net(rng, n_in, H, kind, n_out, act, mag, xs), _one_net(rng, n_in, H, KIND_Q, 1, act, mag, xs)]), x
