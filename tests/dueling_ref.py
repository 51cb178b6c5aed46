"""Test-side restatement of the dueling Q-network (DuelingNetwork, RLCore/src/utils/networks.jl:500-522) and its DQN loss.

- ``combine``: the forward of networks.jl:518-522 in Float32, one rounding per operation:
  μ = ((0f0 + a_1) + ... + a_n) / Float32(n), Q_i = (v + a_i) - μ.
- ``to_single_head``: the flat Flux.destructure vector of DuelingNetwork(trunk, val = Dense(H, 1), adv = Dense(H, n)) as the
  vector of a plain Q-network with n + 1 outputs {v, a_1 .. a_n}, so the oracle's MLP forward gives the head rows.
- ``dqn_loss_grad``: the TD loss of b200rl_dqn_update on a dueling network in float64 with torch autograd (loss = Σ w·ℓ / B).
- ``dqn_loss_grad_manual``: the same gradient by hand, through the backward the kernels implement (∂v = g,
  ∂a_j = (j == a ? g : 0) - g / n); the CPU suite checks it against autograd."""
import numpy as np

import oracle_lib as O


def nparams(ns, H, n):
    """Flux.destructure count of DuelingNetwork(Chain(Dense(ns, H), Dense(H, H)), Dense(H, 1), Dense(H, n))"""
    return H * ns + H + H * H + H + (H + 1) + n * (H + 1)


def glorot_params(ns, H, n, seed):
    """Flux's default Dense init (glorot_uniform weights, zero bias) in destructure order: W1 b1 W2 b2 Wv bv Wa ba"""
    rng = np.random.default_rng(seed)
    parts = []
    for o, i in ((H, ns), (H, H), (1, H), (n, H)):
        lim = np.sqrt(6.0 / (i + o))
        parts += [rng.uniform(-lim, lim, (o, i)).astype(np.float32).ravel(order="F"), np.zeros(o, np.float32)]
    return np.concatenate(parts)


def combine(z):
    """z (n + 1, N) head rows {v, a_1 .. a_n} (Float32) -> Q (n, N), networks.jl:518-522 with Float32 rounding per operation"""
    z = np.asarray(z, np.float32)
    n = z.shape[0] - 1
    s = np.zeros(z.shape[1:], np.float32)
    for j in range(1, n + 1):
        s = (s + z[j]).astype(np.float32)
    mu = (s / np.float32(n)).astype(np.float32)
    return np.stack([((z[0] + z[j]).astype(np.float32) - mu).astype(np.float32) for j in range(1, n + 1)])


def to_single_head(p, ns, H, n):
    trunk = H * ns + H + H * H + H
    head = p[trunk:]
    wv, bv = head[:H], head[H]
    wa = head[H + 1:H + 1 + n * H].reshape(H, n)            # Wa[o + n*j] -> [j, o]
    ba = head[H + 1 + n * H:]
    w3 = np.concatenate([wv[:, None], wa], axis=1)          # [j, o], o = 0 the value row
    return np.concatenate([p[:trunk], w3.ravel(), np.concatenate([[bv], ba])]).astype(np.float32)


def oracle_q(p, ns, H, n, act, obs):
    """Q (n, N) of a dueling network: the oracle's MLP forward for the head rows, then ``combine``"""
    z = O.q_values(O.ac_desc(ns, H, n + 1, act), to_single_head(np.asarray(p, np.float32), ns, H, n), obs)
    return combine(z)


def _torch_net(P, ns, H, n, act):
    import torch

    off = [0]

    def take(o, i):
        w = P[off[0]:off[0] + o * i].reshape(i, o).T
        off[0] += o * i
        b = P[off[0]:off[0] + o]
        off[0] += o
        return w, b

    (W1, b1), (W2, b2), (Wv, bv), (Wa, ba) = take(H, ns), take(H, H), take(1, H), take(n, H)
    f = torch.relu if act == 0 else torch.tanh

    def q(x):                                                  # x (B, ns) float64 -> Q (B, n)
        h2 = f(f(x @ W1.T + b1) @ W2.T + b2)
        v, a = h2 @ Wv.T + bv, h2 @ Wa.T + ba
        return (v + a) - a.mean(dim=1, keepdim=True)
    return q


def _target(q_t, q_o, r, t, disc, double_dqn):
    import torch

    qn = q_t.gather(1, q_o.argmax(1, keepdim=True))[:, 0] if double_dqn else q_t.max(1).values
    return r + disc * (1.0 - t) * qn


def dqn_loss_grad(p, pt, ns, H, n, act, s, a, r, t, s2, w=None, gamma=0.99, huber=True, double_dqn=False, disc=None):
    """float64 autograd: returns (grad of Σ w·ℓ / B, that loss, TD errors R - Q_a).  s, s2 (ns, B); a 1-based."""
    import torch

    dt = torch.float64
    P = torch.tensor(np.asarray(p, np.float64), dtype=dt, requires_grad=True)
    Pt = torch.tensor(np.asarray(pt, np.float64), dtype=dt)
    x, x2 = torch.tensor(np.asarray(s, np.float64).T), torch.tensor(np.asarray(s2, np.float64).T)
    B = x.shape[0]
    r_, t_ = torch.tensor(np.asarray(r, np.float64)), torch.tensor(np.asarray(t, np.float64))
    d_ = torch.tensor(np.asarray(disc, np.float64)) if disc is not None else torch.full((B,), float(np.float32(gamma)), dtype=dt)
    w_ = torch.tensor(np.asarray(w, np.float64)) if w is not None else torch.ones(B, dtype=dt)
    with torch.no_grad():
        R = _target(_torch_net(Pt, ns, H, n, act)(x2), _torch_net(P.detach(), ns, H, n, act)(x2), r_, t_, d_, double_dqn)
    qa = _torch_net(P, ns, H, n, act)(x).gather(1, torch.tensor(np.asarray(a, np.int64) - 1)[:, None])[:, 0]
    e = R - qa
    ae = e.abs()
    l = torch.where(ae < 1.0, 0.5 * e * e, ae - 0.5) if huber else e * e
    loss = (w_ * l).sum() / B
    loss.backward()
    return P.grad.numpy().copy(), float(loss.detach()), e.detach().numpy().copy()


def dqn_loss_grad_manual(p, pt, ns, H, n, act, s, a, r, t, s2, w=None, gamma=0.99, huber=True, double_dqn=False):
    """the same gradient in NumPy float64 through the dueling backward of the kernels (duel.cuh) and a plain MLP backward"""
    p = np.asarray(p, np.float64)
    B = s.shape[1]
    f = (lambda z: np.maximum(z, 0.0)) if act == 0 else np.tanh
    df = (lambda h: (h > 0).astype(np.float64)) if act == 0 else (lambda h: 1.0 - h * h)

    def unpack(q):
        o = 0
        out = []
        for (O_, I_) in ((H, ns), (H, H), (1, H), (n, H)):
            out.append(q[o:o + O_ * I_].reshape(I_, O_).T); o += O_ * I_
            out.append(q[o:o + O_]); o += O_
        return out

    def fwd(q, x):
        W1, b1, W2, b2, Wv, bv, Wa, ba = unpack(q)
        h1 = f(W1 @ x + b1[:, None]); h2 = f(W2 @ h1 + b2[:, None])
        v = Wv @ h2 + bv[:, None]; adv = Wa @ h2 + ba[:, None]
        return h1, h2, (v + adv) - adv.mean(0, keepdims=True)

    x, x2 = np.asarray(s, np.float64), np.asarray(s2, np.float64)
    qt, qo = fwd(np.asarray(pt, np.float64), x2)[2], fwd(p, x2)[2]
    qn = qt[qo.argmax(0), np.arange(B)] if double_dqn else qt.max(0)
    R = np.asarray(r, np.float64) + np.float64(np.float32(gamma)) * (1.0 - np.asarray(t, np.float64)) * qn
    h1, h2, q = fwd(p, x)
    ai = np.asarray(a, np.int64) - 1
    e = R - q[ai, np.arange(B)]
    wv = np.ones(B) if w is None else np.asarray(w, np.float64)
    if huber:
        l = np.where(np.abs(e) < 1.0, 0.5 * e * e, np.abs(e) - 0.5); dl = np.where(np.abs(e) < 1.0, -e, -np.sign(e))
    else:
        l = e * e; dl = -2.0 * e
    g = wv * dl / B                                          # ∂loss/∂Q_a per sample
    dv = g[None, :]
    dadv = -np.broadcast_to(g / n, (n, B)).copy()
    dadv[ai, np.arange(B)] += g
    W1, b1, W2, b2, Wv, bv, Wa, ba = unpack(p)
    dh2 = (Wv.T @ dv + Wa.T @ dadv) * df(h2)
    dh1 = (W2.T @ dh2) * df(h1)
    grads = [dh1 @ x.T, dh1.sum(1), dh2 @ h1.T, dh2.sum(1), dv @ h2.T, dv.sum(1), dadv @ h2.T, dadv.sum(1)]
    flat = np.concatenate([gr.T.ravel() if gr.ndim == 2 else gr for gr in grads])
    return flat, float((wv * l).sum() / B), e
