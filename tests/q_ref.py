"""Float64 restatements of the plain Q-network and the DQN TD loss, shared by the CPU check of the oracle's hand-written gradient
(test_oracle_nn.py) and the GPU checks of the TD loss + backward kernel (test_traj_dqn_gpu.py, test_n_step_gpu.py).

- ``unpack_mlp``: flat Flux.destructure parameters -> a torch forward (two hidden layers, one or more linear heads).
- ``dqn_loss_grad``: the loss of b200rl_dqn_update on a plain Q-network, Σ w·ℓ(R - Q_a) / B with R = r + d·(1 - t)·Q'(s'), in
  float64 with torch autograd; double DQN takes the arg-max of the online net's Q(s') (first maximum) and the target net's value.
- ``oracle_dqn_loss_grad``: the CPU oracle's gradient of the same loss for a sampled batch, per-sample discounts included.
- ``blocks``: the parameter blocks W1 b1 W2 b2 W3 b3 as slices of the flat vector.
- ``tie_actions``: parameters whose Q-values of two actions tie exactly (the double-DQN "first maximum wins" rule)."""
import numpy as np
import torch

import oracle_lib as O


def unpack_mlp(p, n_in, H, heads, act):
    """flat Flux-order params -> torch forward function"""
    o = 0
    def take(n):
        nonlocal o
        v = p[o:o + n]; o += n
        return v
    W1 = take(H * n_in).reshape(n_in, H).T; b1 = take(H)
    W2 = take(H * H).reshape(H, H).T; b2 = take(H)
    hs = []
    for d in heads:
        W = take(d * H).reshape(H, d).T; b = take(d)
        hs.append((W, b))
    f = torch.relu if act == O.ACT_RELU else torch.tanh
    def fwd(x):  # x (B, n_in)
        h = f(x @ W1.T + b1); h = f(h @ W2.T + b2)
        return torch.cat([h @ W.T + b for W, b in hs], dim=1)
    return fwd, o


def blocks(ns, H, na):
    """(name, slice) of W1 b1 W2 b2 W3 b3 in the flat parameter vector"""
    out, o = [], 0
    for name, n in (("W1", H * ns), ("b1", H), ("W2", H * H), ("b2", H), ("W3", na * H), ("b3", na)):
        out.append((name, slice(o, o + n))); o += n
    return out


def tie_actions(p, ns, H, na, a, b):
    """a copy of p whose head row and bias of action b equal those of action a (1-based): Q_a ≡ Q_b, bit for bit, in any forward"""
    p = np.array(p, np.float32)
    o = H * ns + H + H * H + H
    W3 = p[o:o + na * H]                                     # (na, H) column-major: W3[k + na * j] = row k, column j
    W3[b - 1::na] = W3[a - 1::na]
    p[o + na * H + b - 1] = p[o + na * H + a - 1]
    return p


def q_values(p, ns, H, na, act, x):
    """float64 Q (B, na) of the flat parameters p at the states x (ns, B)"""
    fwd, _ = unpack_mlp(torch.tensor(np.asarray(p, np.float64)), ns, H, [na], act)
    with torch.no_grad():
        return fwd(torch.tensor(np.asarray(x, np.float64).T)).numpy()


def dqn_loss_grad(p, pt, ns, H, na, act, s, a, r, t, s2, w=None, gamma=0.99, huber=True, double_dqn=False, disc=None):
    """float64 autograd: returns (grad of Σ w·ℓ / B, that loss, TD errors R - Q_a).  s, s2 (ns, B); a 1-based; disc (B) replaces
    Float32(gamma) per sample (an n-step window's γ^m)."""
    dt = torch.float64
    B = s.shape[1]
    P = torch.tensor(np.asarray(p, np.float64), requires_grad=True)
    q, _ = unpack_mlp(P, ns, H, [na], act)
    qt, _ = unpack_mlp(torch.tensor(np.asarray(pt, np.float64)), ns, H, [na], act)
    x, x2 = torch.tensor(np.asarray(s, np.float64).T), torch.tensor(np.asarray(s2, np.float64).T)
    d = torch.tensor(np.asarray(disc, np.float64)) if disc is not None else torch.full((B,), float(np.float32(gamma)), dtype=dt)
    with torch.no_grad():
        qn = qt(x2)
        qnext = qn[torch.arange(B), q(x2).argmax(1)] if double_dqn else qn.max(1).values
        R = torch.tensor(np.asarray(r, np.float64)) + d * (1 - torch.tensor(np.asarray(t, np.float64))) * qnext
    qv = q(x)[torch.arange(B), torch.tensor(np.asarray(a, np.int64) - 1)]
    e = R - qv
    l = torch.where(e.abs() < 1, 0.5 * e * e, e.abs() - 0.5) if huber else e * e
    W = torch.tensor(np.asarray(w, np.float64)) if w is not None else torch.ones(B, dtype=dt)
    L = (W * l).sum() / B
    L.backward()
    return P.grad.numpy().copy(), L.item(), e.detach().numpy().copy()


def oracle_dqn_loss_grad(desc, p, pt, b, w, huber, double_dqn):
    """the oracle's DQN loss of a sampled batch with R = G + discount·(1 - t)·q': one oracle call per window length (one discount
    each; a 1-step batch is one call with γ)"""
    B = b["reward"].size
    grad, loss, td = np.zeros(O.q_nparams(desc)), 0.0, np.empty(B, np.float32)
    for m in np.unique(b["horizon"]):
        i = np.flatnonzero(b["horizon"] == m)
        d = b["discount"][i[0]]
        assert np.all(b["discount"][i] == d)
        g, l, t = O.dqn_loss_grad(desc, p, pt, b["state"][:, i], b["action"][i], b["reward"][i], b["terminal"][i], b["next_state"][:, i],
                                  None if w is None else w[i], float(d), huber, double_dqn)
        grad += g * (i.size / B); loss += l * i.size / B; td[i] = t
    return grad, loss, td
