"""NumPy restatement of the value-based explorers the device plans with (csrc/explore.cuh), one column at a time on the
column's own Xoshiro256++ stream — the test suite's second statement of the semantics, written from the reference and the
upstream libraries it calls, not from the header:

  kind 2  EpsilonSpeedyExplorer(β) (ReinforcementLearningFarm epsilon_speedy_explorer.jl:19-53):
          ϵ = exp((β * -1) * Float64(step)); rand(rng) >= ϵ ? findmax(Q)[2] : rand(rng, 1:n)
  kind 3  WeightedSoftmaxExplorer (weighted_softmax_explorer.jl:20-21): sample(rng, Weights(softmax(Q), 1f0))
          (NNlib softmax; StatsBase's inverse CDF: t = rand(rng) * 1f0, i = 1, cw = p_1, while cw < t && i < n ...)
  kind 4  GumbelSoftmaxExplorer (gumbel_softmax_explorer.jl:12-16): argmax(logsoftmax(Q) .- log.(-log.(rand(rng, Float32, n))))

Float32 operations are numpy float32 scalars (one rounding each); the Float32 exp / log are the Float64 evaluations the header
documents (plain Python float operations, rounded once to float32), since the selections must agree bit for bit."""
import math

import numpy as np

M64 = (1 << 64) - 1
F32 = np.float32
INF = F32(np.inf)


# ---- Xoshiro256++ and the Julia 1.10 samplers ------------------------------------------------------------------------------
def xo_next(s):
    tmp = (s[0] + s[3]) & M64
    res = ((((tmp << 23) | (tmp >> 41)) & M64) + s[0]) & M64
    t = (s[1] << 17) & M64
    s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3]; s[2] ^= t
    s[3] = ((s[3] << 45) | (s[3] >> 19)) & M64
    return res


def rand_f64(s):
    return (xo_next(s) >> 11) * 2.0 ** -53


def rand_f32(s):
    return F32(((xo_next(s) >> 32) & 0xFFFFFFFF) >> 8) * F32(2.0 ** -24)


def rand_oneto(s, n):
    """rand(rng, 1:n): Lemire nearly-divisionless on UInt64 (SamplerRangeNDL)"""
    x = xo_next(s)
    m = x * n
    lo = m & M64
    if lo < n:
        t = ((1 << 64) - n) % n
        while lo < t:
            x = xo_next(s)
            m = x * n
            lo = m & M64
    return (m >> 64) + 1


# ---- Float32 exp / log (header: Float64 evaluation rounded once) ------------------------------------------------------------
_EXP_INV = [1.0 / 479001600.0, 1.0 / 39916800.0, 1.0 / 3628800.0, 1.0 / 362880.0, 1.0 / 40320.0, 1.0 / 5040.0, 1.0 / 720.0,
            1.0 / 120.0, 1.0 / 24.0, 1.0 / 6.0, 0.5, 1.0, 1.0]
_LOG_INV = [1.0 / 21.0, 1.0 / 19.0, 1.0 / 17.0, 1.0 / 15.0, 1.0 / 13.0, 1.0 / 11.0, 1.0 / 9.0, 1.0 / 7.0, 1.0 / 5.0, 1.0 / 3.0, 1.0]
LN2_HI, LN2_LO = 6.93147180369123816490e-01, 1.90821492927058770002e-10


def f32_exp(x):
    x = F32(x)
    if x != x:
        return x
    if x < F32(-104.0):
        return F32(0.0)
    if x > F32(89.0):
        return INF
    xd = float(x)
    k = (xd * 1.4426950408889634 + 6755399441055744.0) - 6755399441055744.0
    r = (xd - k * LN2_HI) - k * LN2_LO
    p = 1.0 / 6227020800.0
    for c in _EXP_INV:
        p = p * r + c
    with np.errstate(over="ignore"):
        return F32(p * math.ldexp(1.0, int(k)))


def f32_log(x):
    x = F32(x)
    if x != x:
        return x
    if x < 0:
        return F32(np.nan)
    if x == 0:
        return -INF
    if x == INF:
        return x
    m, e = math.frexp(float(x))          # x = m 2^e, m in [0.5, 1)
    m, e = m * 2.0, e - 1                # m in [1, 2)
    if m > 1.4142135623730951:
        m, e = m * 0.5, e + 1
    f = m - 1.0
    s = f / (2.0 + f)
    s2 = s * s
    p = 1.0 / 23.0
    for c in _LOG_INV:
        p = p * s2 + c
    ed = float(e)
    return F32(ed * LN2_HI + (ed * LN2_LO + (2.0 * s) * p))


# ---- NNlib softmax / logsoftmax ------------------------------------------------------------------------------------------
def fast_maximum(q):
    """@fastmath reduce(max, q; init = -Inf32): NaN never wins"""
    m = -INF
    for v in q:
        if v > m:
            m = v
    return m


def softmax(q):
    q = [F32(v) for v in q]
    m = fast_maximum(q)
    with np.errstate(invalid="ignore", over="ignore"):
        if not (m - m == 0) and m == INF:
            e = [F32(1.0) if v == INF else F32(0.0) for v in q]
        else:
            e = [f32_exp(F32(v - m)) for v in q]
        s = e[0]
        for v in e[1:]:
            s = F32(s + v)
        return [F32(v / s) for v in e]


def logsoftmax_parts(q):
    """(out = x .- max_ or NNlib's non-finite branch, log(sum(exp, out)))"""
    q = [F32(v) for v in q]
    m = fast_maximum(q)
    with np.errstate(invalid="ignore", over="ignore"):
        if not (m - m == 0) and m == INF:
            d = [F32(0.0) if v == INF else -INF for v in q]
        else:
            d = [F32(v - m) for v in q]
        s = f32_exp(d[0])
        for v in d[1:]:
            s = F32(s + f32_exp(v))
        return d, f32_log(s)


# ---- the three columns ---------------------------------------------------------------------------------------------------
def findmax_gt(q):
    """explore::select's findmax (the ϵ-greedy code): first maximum, NaN ranks highest"""
    best = 0
    for o in range(1, len(q)):
        a, b = q[o], q[best]
        if (a != a and b == b) or a > b:
            best = o
    return best


def isless(a, b):
    """Base.isless on Float32: NaN above everything, -0.0 below 0.0"""
    if a != a:
        return False
    if b != b:
        return True
    if a == b:
        return bool(np.signbit(a)) and not bool(np.signbit(b))
    return a < b


def findmax_base(z):
    best, m = 0, z[0]
    for o in range(1, len(z)):
        if isless(m, z[o]):
            m, best = z[o], o
    return best


def speedy_eps(beta, step):
    return math.exp((beta * -1.0) * float(step))


def speedy_column(beta, step, q, s):
    eps = speedy_eps(beta, step)
    u = rand_f64(s)
    return findmax_gt(q) + 1 if u >= eps else rand_oneto(s, len(q))


def weighted_softmax_column(q, s):
    p = softmax(q)
    t = rand_f64(s) * 1.0
    i, cw = 0, p[0]
    while float(cw) < t and i < len(q) - 1:
        i += 1
        cw = F32(cw + p[i])
    return i + 1


def gumbel_softmax_column(q, s):
    d, lse = logsoftmax_parts(q)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        g = [F32(F32(d[o] - lse) - f32_log(-f32_log(rand_f32(s)))) for o in range(len(q))]
    return findmax_base(g) + 1


def plan(kind, q, rng, step0=1, beta=0.0):
    """BatchExplorer over the columns of q (n, N) with column i at step0 + i (kind 2); rng (N, 4) uint64 advanced in place.
    Returns the (N,) int32 actions."""
    q = np.asarray(q, np.float32)
    N = q.shape[1]
    out = np.empty(N, np.int32)
    for i in range(N):
        s = [int(v) for v in rng[i]]
        col = [q[o, i] for o in range(q.shape[0])]
        if kind == 2:
            out[i] = speedy_column(beta, step0 + i, col, s)
        elif kind == 3:
            out[i] = weighted_softmax_column(col, s)
        elif kind == 4:
            out[i] = gumbel_softmax_column(col, s)
        else:
            raise ValueError(kind)
        rng[i] = np.array(s, np.uint64)
    return out
