"""Host mirror of the reference's explorers for the DQN action path
(RLCore/src/policies/explorers/epsilon_greedy_explorer.jl:47-204, weighted_softmax_explorer.jl, gumbel_softmax_explorer.jl,
batch_explorer.jl:15-21; ReinforcementLearningFarm's EpsilonSpeedyExplorer).

The explorer object is host state in the reference too (a mutable struct holding the schedule and
the step counter); the per-column work — evaluating get_ϵ(step + i), the uniform draw and the
arg-max / random choice for every env of the batch — happens in ``b200rl_net_q_explore`` on the
device.  ``get_eps`` / ``prob`` are the reference's scalar Float64 formulas (Python floats are
IEEE doubles, evaluated left to right like the Julia code)."""
import math

import numpy as np

from . import _lib as L


class GreedyExplorer:
    """GreedyExplorer() (epsilon_greedy_explorer.jl:196-204): findmax(values)[2], no RNG."""
    is_break_tie = False

    def get_eps(self, step=None):
        return 0.0

    def prob(self, values, action=None):
        best = _findmax(values)
        p = [1.0 if i == best else 0.0 for i in range(len(values))]
        return p if action is None else p[action - 1]

    def plan_values(self, values):
        return _findmax(values) + 1


def _findmax(values):
    best = 0
    for i in range(1, len(values)):
        a, b = values[i], values[best]
        if (a != a and b == b) or a > b:
            best = i
    return best


class EpsilonGreedyExplorer:
    """EpsilonGreedyExplorer(; ϵ_stable, kind = :linear, ϵ_init = 1.0, warmup_steps = 0, decay_steps = 0, step = 1,
    is_break_tie = false) (epsilon_greedy_explorer.jl:47-67).  ``EpsilonGreedyExplorer(0.1)`` = ϵ_stable."""

    def __init__(self, eps_stable, kind="linear", eps_init=1.0, warmup_steps=0, decay_steps=0, step=1, is_break_tie=False):
        if kind not in ("linear", "exp"):
            raise ValueError("kind must be 'linear' or 'exp'")
        self.eps_stable, self.eps_init = float(eps_stable), float(eps_init)
        self.warmup_steps, self.decay_steps = int(warmup_steps), int(decay_steps)
        self.kind, self.step, self.is_break_tie = kind, int(step), bool(is_break_tie)

    def get_eps(self, step=None):
        """get_ϵ(s, step) (epsilon_greedy_explorer.jl:69-91)."""
        step = self.step if step is None else step
        if self.kind == "linear":
            if step <= self.warmup_steps:
                return self.eps_init
            if step >= self.warmup_steps + self.decay_steps:
                return self.eps_stable
            steps_left = self.warmup_steps + self.decay_steps - step
            return self.eps_stable + steps_left / self.decay_steps * (self.eps_init - self.eps_stable)
        if step <= self.warmup_steps:
            return self.eps_init
        n = step - self.warmup_steps
        scale = self.eps_init - self.eps_stable
        return self.eps_stable + scale * math.exp(-1.0 * n / self.decay_steps)

    def prob(self, values, action=None):
        """prob(s, values[, action]) (epsilon_greedy_explorer.jl:141-171): the Categorical's probability vector."""
        eps, n = self.get_eps(), len(values)
        probs = [eps / n] * n
        if self.is_break_tie:
            mx = max(values)
            inds = [i for i, v in enumerate(values) if v == mx]
            for i in inds:
                probs[i] += (1 - eps) / len(inds)
        else:
            probs[_findmax(values)] += 1 - eps
        return probs if action is None else probs[action - 1]

    def as_struct(self):
        return L.Explorer(self.eps_stable, self.eps_init, self.warmup_steps, self.decay_steps, self.step,
                          0 if self.kind == "linear" else 1, int(self.is_break_tie), 0.0)

    def advance(self, n):
        """The batch call planned n columns: the inner explorer's step moved n times (batch_explorer.jl:15-21)."""
        self.step += int(n)


class EpsilonSpeedyExplorer:
    """EpsilonSpeedyExplorer(β) (ReinforcementLearningFarm, explorers/epsilon_speedy_explorer.jl:19-53): ϵ-greedy with
    get_ϵ = exp(β_neg * step), β_neg = β * -1, step starting at 1; findmax without break-tie."""
    is_break_tie = False

    def __init__(self, beta, step=1):
        self.beta, self.step = float(beta), int(step)
        if not math.isfinite(self.beta):
            raise ValueError("beta must be finite")

    def get_eps(self, step=None):
        step = self.step if step is None else step
        return math.exp(self.beta * -1 * float(step))

    def prob(self, values, action=None):
        """prob(s, values[, action]): the Categorical's probability vector (ϵ/n everywhere, + 1 - ϵ at findmax)."""
        eps, n = self.get_eps(), len(values)
        probs = [eps / n] * n
        probs[_findmax(values)] += 1 - eps
        return probs if action is None else probs[action - 1]

    def as_struct(self):
        return L.Explorer(0.0, 0.0, 0, 0, self.step, 2, 0, self.beta)

    def advance(self, n):
        """The batch call planned n columns: the inner explorer's step moved n times (batch_explorer.jl:15-21)."""
        self.step += int(n)


def softmax(values):
    """NNlib's softmax of a Float32 vector as the device computes it: m = the largest non-NaN entry (-Inf if none),
    e_j = exp(Q_j - m) (or, m = +Inf, 1 where Q_j = +Inf and 0 elsewhere), p_j = e_j / (e_1 + e_2 + ...) left to right, every
    operation rounded once in Float32 (numpy's exp may differ from the device's in the last bit)."""
    q = np.asarray(values, np.float32)
    m = np.float32(-np.inf)
    for v in q:
        if v > m:
            m = v
    with np.errstate(invalid="ignore", over="ignore"):
        if m == np.inf:
            e = np.where(q == np.inf, np.float32(1), np.float32(0)).astype(np.float32)
        else:
            e = np.exp((q - m).astype(np.float32)).astype(np.float32)
        s = e[0]
        for v in e[1:]:
            s = np.float32(s + v)
        return (e / s).astype(np.float32)


class WeightedSoftmaxExplorer:
    """WeightedSoftmaxExplorer() (weighted_softmax_explorer.jl:20-21): sample(rng, Weights(softmax(values), 1f0)) per column
    (one Float64 draw); no step."""

    def prob(self, values):
        """prob(s, values) = softmax(values) (weighted_softmax_explorer.jl:28)"""
        return softmax(values)

    def as_struct(self):
        return L.Explorer(0.0, 0.0, 0, 0, 0, 3, 0, 0.0)

    def advance(self, n):
        pass


class GumbelSoftmaxExplorer:
    """GumbelSoftmaxExplorer() (gumbel_softmax_explorer.jl:12-16): argmax(logsoftmax(values) .- log.(-log.(u))) with
    u = rand(rng, Float32, n) per column; no step."""

    def as_struct(self):
        return L.Explorer(0.0, 0.0, 0, 0, 0, 4, 0, 0.0)

    def advance(self, n):
        pass
