"""Host side of the softmax and speedy explorers (no GPU).

csrc/explore.cuh compiled for the host, bit for bit against the NumPy restatement in explorers_ref.py — actions and advanced
streams for EpsilonSpeedyExplorer (kind 2), WeightedSoftmaxExplorer (kind 3) and GumbelSoftmaxExplorer (kind 4): n = 1 to 4,
ties and ±0, ±Inf entries, spreads that underflow exp to 0, sums that round, NaN and a stream whose next output is 0 (u = 0).
The header's Float32 exp / log against correctly rounded values (a long double evaluation rounded once): exhaustively over
the Float32 inputs of [-104, 0] (exp) and of [2^-30, 32] (log), every 61st bit pattern over the rest of (-Inf, 0] / [0, +Inf],
and the special values.  The reference's pinned EpsilonSpeedyExplorer numbers through the header and explorers.py; chi-square
of both softmax kinds over 2^20 seeded columns; the C struct's layout against _lib.Explorer; kinds 0 and 1 unchanged."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import explorers_ref as R
import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))
HD = os.path.join(HERE, "hostdev")
CSRC = os.path.join(os.path.dirname(HERE), "reinforcementlearning.jl_b200", "csrc")

DRIVER = r"""
#include <cuda_runtime.h>
#include <cstddef>
#include <thread>
#include <vector>
#include "explore.cuh"
#include "jl_device.cuh"

extern "C" {
// BatchExplorer over the columns of qv (na, n) with column i at step0 + i; rng (n, 4) advanced in place
void hd_plan(const b200rl_explorer* e, long long step0, const float* qv, int na, long long n, unsigned long long* rng, int* out) {
    for (long long i = 0; i < n; ++i) {
        unsigned long long st[4] = {rng[4 * i], rng[4 * i + 1], rng[4 * i + 2], rng[4 * i + 3]};
        out[i] = explore::select(*e, step0 + i, qv + (long long)na * i, na, st);
        for (int k = 0; k < 4; ++k) rng[4 * i + k] = st[k];
    }
}
// the same Q column for every one of n streams
void hd_plan_fixed(const b200rl_explorer* e, const float* q, int na, long long n, unsigned long long* rng, int* out) {
    for (long long i = 0; i < n; ++i) {
        unsigned long long st[4] = {rng[4 * i], rng[4 * i + 1], rng[4 * i + 2], rng[4 * i + 3]};
        out[i] = explore::select(*e, 1 + i, q, na, st);
    }
}
double hd_speedy_eps(double beta, long long step) { return explore::speedy_eps(beta, step); }
void hd_exp(const float* x, long long n, float* y) { for (long long i = 0; i < n; ++i) y[i] = explore::f32_exp(x[i]); }
void hd_log(const float* x, long long n, float* y) { for (long long i = 0; i < n; ++i) y[i] = explore::f32_log(x[i]); }
float hd_rand_f32_explore(unsigned long long* s) {
    unsigned long long st[4] = {s[0], s[1], s[2], s[3]};
    float u = explore::xo_f32(st);
    for (int k = 0; k < 4; ++k) s[k] = st[k];
    return u;
}
float hd_rand_f32_jld(unsigned long long* s) {
    jld::Xo g{s[0], s[1], s[2], s[3]};
    float u = jld::rand_f32(g);
    s[0] = g.s0; s[1] = g.s1; s[2] = g.s2; s[3] = g.s3;
    return u;
}
long long hd_explorer_layout(long long* off) {
    off[0] = offsetof(b200rl_explorer, eps_stable); off[1] = offsetof(b200rl_explorer, eps_init);
    off[2] = offsetof(b200rl_explorer, warmup_steps); off[3] = offsetof(b200rl_explorer, decay_steps);
    off[4] = offsetof(b200rl_explorer, step); off[5] = offsetof(b200rl_explorer, kind);
    off[6] = offsetof(b200rl_explorer, is_break_tie); off[7] = offsetof(b200rl_explorer, beta);
    return (long long)sizeof(b200rl_explorer);
}
// fn 0: exp, 1: log over the bit patterns lo, lo + stride, ... <= hi (as uint32) against the long double value rounded once:
// out = {checked, differing, largest distance in ulps (bit patterns of the same sign), a pattern at that distance}
static long long ulps(float a, float b) {
    if (a != a || b != b) return (a != a && b != b) ? 0 : (1ll << 40);
    uint32_t ua, ub;
    memcpy(&ua, &a, 4); memcpy(&ub, &b, 4);
    long long ia = (ua >> 31) ? -(long long)(ua & 0x7fffffffu) : (long long)ua, ib = (ub >> 31) ? -(long long)(ub & 0x7fffffffu) : (long long)ub;
    return ia > ib ? ia - ib : ib - ia;
}
void hd_sweep(int fn, uint32_t lo, uint32_t hi, uint32_t stride, long long* out) {
    unsigned nt = std::thread::hardware_concurrency();
    if (nt < 1) nt = 1;
    if (nt > 32) nt = 32;
    std::vector<long long> res(4 * nt, 0);
    std::vector<std::thread> th;
    const unsigned long long count = ((unsigned long long)hi - lo) / stride + 1;
    for (unsigned t = 0; t < nt; ++t) th.emplace_back([&, t] {
        long long* r = &res[4 * t];
        for (unsigned long long j = t; j < count; j += nt) {
            uint32_t b = (uint32_t)(lo + j * stride);
            float x;
            memcpy(&x, &b, 4);
            float got = fn == 0 ? explore::f32_exp(x) : explore::f32_log(x);
            float ref = fn == 0 ? (float)expl((long double)x) : (float)logl((long double)x);
            long long d = ulps(got, ref);
            r[0] += 1;
            if (d) r[1] += 1;
            if (d > r[2]) { r[2] = d; r[3] = b; }
        }
    });
    for (auto& t : th) t.join();
    out[0] = out[1] = out[2] = out[3] = 0;
    for (unsigned t = 0; t < nt; ++t) {
        out[0] += res[4 * t]; out[1] += res[4 * t + 1];
        if (res[4 * t + 2] > out[2]) { out[2] = res[4 * t + 2]; out[3] = res[4 * t + 3]; }
    }
}
}
"""


@pytest.fixture(scope="module")
def xh(tmp_path_factory):
    d = tmp_path_factory.mktemp("explorers")
    src, so = d / "explorers_driver.cpp", d / "libexplorers.so"
    src.write_text(DRIVER)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wno-unknown-pragmas",
                           "-pthread", "-I", HD, "-I", CSRC, "-shared", "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    vp = C.c_void_p
    L.hd_plan.restype, L.hd_plan.argtypes = None, [vp, C.c_longlong, vp, C.c_int, C.c_longlong, vp, vp]
    L.hd_plan_fixed.restype, L.hd_plan_fixed.argtypes = None, [vp, vp, C.c_int, C.c_longlong, vp, vp]
    L.hd_speedy_eps.restype, L.hd_speedy_eps.argtypes = C.c_double, [C.c_double, C.c_longlong]
    for f in (L.hd_exp, L.hd_log):
        f.restype, f.argtypes = None, [vp, C.c_longlong, vp]
    for f in (L.hd_rand_f32_explore, L.hd_rand_f32_jld):
        f.restype, f.argtypes = C.c_float, [vp]
    L.hd_explorer_layout.restype, L.hd_explorer_layout.argtypes = C.c_longlong, [vp]
    L.hd_sweep.restype, L.hd_sweep.argtypes = None, [C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _struct(pkg, kind, beta=0.0, step=1):
    ex = {2: pkg.EpsilonSpeedyExplorer(beta, step=step) if kind == 2 else None, 3: pkg.WeightedSoftmaxExplorer(),
          4: pkg.GumbelSoftmaxExplorer()}[kind]
    return ex.as_struct()


def header_plan(xh, pkg, kind, q, rng, step0=1, beta=0.0):
    q = np.asfortranarray(np.asarray(q, np.float32))
    na, n = q.shape
    st = _struct(pkg, kind, beta, step0)
    a, r = np.empty(n, np.int32), np.ascontiguousarray(rng, np.uint64).copy()
    xh.hd_plan(C.byref(st), step0, _p(q), na, n, _p(r), _p(a))
    return a, r


def check_plan(xh, pkg, kind, q, seed, step0=1, beta=0.0):
    q = np.asarray(q, np.float32)
    rng = O.splitmix_states_fast(q.shape[1], seed)
    a, r = header_plan(xh, pkg, kind, q, rng, step0, beta)
    rr = rng.copy()
    ref = R.plan(kind, q, rr, step0, beta)
    assert np.array_equal(a, ref), (kind, np.nonzero(a != ref)[0][:10], q[:, np.nonzero(a != ref)[0][:3]])
    assert np.array_equal(r, rr)
    return a


F = np.float32
INF, NAN = np.inf, np.nan
SPECIAL = [  # columns of 4; the first n rows are used
    [0.0, 0.0, 0.0, 0.0], [-0.0, 0.0, -0.0, 0.0], [1.0, 1.0, 0.5, 1.0],          # ties and ±0
    [INF, 1.0, INF, -INF], [-INF, -INF, -INF, -INF], [INF, INF, INF, INF], [-INF, 2.0, -INF, 3.0], [1.0, INF, -1.0, 0.0],
    [0.0, -200.0, -1e30, -3e38], [3e38, -3e38, 0.0, 1.0],                             # spreads that underflow exp to 0
    [1e-8, 0.0, -1e-8, 2e-8], [0.1, 0.2, 0.3, 0.4], [1 / 3, 2 / 3, 1.0, 4 / 3], [16.0, 16.0, 15.999999, 0.0],   # sums that round
    [NAN, 1.0, 2.0, 3.0], [1.0, NAN, 2.0, INF], [NAN, NAN, NAN, NAN],
    [-87.0, -88.0, -103.9, -104.5], [88.0, 0.0, -1.0, 5.0],
]


@pytest.mark.parametrize("kind", [2, 3, 4])
@pytest.mark.parametrize("na", [1, 2, 3, 4])
def test_header_matches_the_restatement(xh, pkg, kind, na):
    rng = np.random.default_rng(10 * kind + na)
    n = 1500
    q = (rng.standard_normal((na, n)) * 10.0 ** rng.integers(-4, 3, (na, n))).astype(np.float32)
    q[:, ::9] = q[0, ::9]                                            # all-tie columns
    q[:, 5::13] = np.float32(0.0) * np.sign(rng.standard_normal((na, 1)))   # ±0
    sp = np.array(SPECIAL, np.float32).T[:na]
    q = np.hstack([sp, np.repeat(sp, 40, axis=1), q])                # each special column under 41 streams
    with np.errstate(invalid="ignore"):
        check_plan(xh, pkg, kind, q, 3 + kind, step0=1 if kind != 2 else 17, beta=0.02)


@pytest.mark.parametrize("beta", [0.0, 1e-5, 0.1, 3.0, -1e-4])
def test_speedy_schedules(xh, pkg, beta):
    q = np.random.default_rng(1).standard_normal((3, 2000)).astype(np.float32)
    a = check_plan(xh, pkg, 2, q, 7, step0=1, beta=beta)
    if beta == 0.0:                                                  # ϵ = 1: rand(1:n) every column
        assert len(set(a.tolist())) == 3


def test_a_zero_uniform(xh, pkg):
    """s0 = s3 = 0 makes the next Xoshiro256++ output 0: u = 0f0 (Gumbel: log(0) = -Inf, that entry becomes -Inf) and
    rand(rng) = 0.0 (weighted softmax: t = 0, the first action; speedy: u < ϵ, a random action)"""
    s = np.array([[0, 0x123456789ABCDEF, 0xFEDCBA987654321, 0]], np.uint64)
    st = [int(v) for v in s[0]]
    assert R.xo_next(list(st)) == 0
    for na in (1, 2, 3, 4):
        for q in ([0.0, 0.0, 0.0, 0.0], [5.0, 1.0, 2.0, 3.0], [1.0, 5.0, 2.0, 3.0], [INF, 1.0, 2.0, 3.0]):
            qq = np.array(q, np.float32)[:na, None]
            for kind in (2, 3, 4):
                a, r = header_plan(xh, pkg, kind, qq, s, beta=0.1)
                rr = s.copy()
                with np.errstate(invalid="ignore"):
                    ref = R.plan(kind, qq, rr, 1, 0.1)
                assert np.array_equal(a, ref) and np.array_equal(r, rr), (kind, na, q)
    # the Gumbel draw of column 1 is u = 0: action 1 can only win when it is the only action
    a, _ = header_plan(xh, pkg, 4, np.array([[9.0], [0.0]], np.float32), s)
    assert a[0] == 2
    a, _ = header_plan(xh, pkg, 3, np.array([[-9.0], [0.0]], np.float32), s)
    assert a[0] == 1                                                 # t = 0: cw = p_1 >= 0 stops at once


def test_rand_f32_is_jl_device_sampler(xh):
    s1 = np.array([1, 2, 3, 4], np.uint64)
    s2 = s1.copy()
    rs = [1, 2, 3, 4]
    for _ in range(1000):
        u1, u2 = xh.hd_rand_f32_explore(_p(s1)), xh.hd_rand_f32_jld(_p(s2))
        assert np.float32(u1) == np.float32(u2) == R.rand_f32(rs)
    assert np.array_equal(s1, s2)


def test_exp_log_special_values(xh):
    x = np.array([-INF, -0.0, 0.0, NAN, -104.5, -103.98, -103.97, -87.5, -1e-45, -1e-30, 88.7, 89.5, INF], np.float32)
    y = np.empty_like(x)
    xh.hd_exp(_p(x), x.size, _p(y))
    assert y[0] == 0 and y[1] == 1 and y[2] == 1 and np.isnan(y[3]) and y[4] == 0 and y[-2] == INF and y[-1] == INF
    assert y[5] == 0 and y[6] == np.float32(2.0 ** -149)            # exp(-103.97) > 2^-150 rounds up to the smallest subnormal
    assert 0 < y[7] < np.finfo(np.float32).tiny                      # a subnormal result
    assert y[8] == 1 and y[9] == 1
    x = np.array([0.0, -0.0, INF, NAN, -1.0, 1.0, 2.0 ** -149, 2.0 ** -126, np.finfo(np.float32).max, 2.0 ** -24], np.float32)
    y = np.empty_like(x)
    xh.hd_log(_p(x), x.size, _p(y))
    assert y[0] == -INF and y[1] == -INF and y[2] == INF and np.isnan(y[3]) and np.isnan(y[4]) and y[5] == 0
    assert y[6] == np.float32(-149 * math.log(2)) and y[7] == np.float32(-126 * math.log(2)) and y[9] == np.float32(-24 * math.log(2))
    for fn, ref in ((xh.hd_exp, R.f32_exp), (xh.hd_log, R.f32_log)):  # the restatement's Float32 exp / log are the header's
        xs = np.random.default_rng(2).standard_normal(20000).astype(np.float32) * np.float32(30)
        xs = -np.abs(xs) if fn is xh.hd_exp else np.abs(xs)
        ys = np.empty_like(xs)
        fn(_p(xs), xs.size, _p(ys))
        assert all(np.float32(ys[i]).view(np.uint32) == ref(xs[i]).view(np.uint32) for i in range(xs.size))


def _sweep(xh, fn, lo, hi, stride):
    out = np.zeros(4, np.int64)
    xh.hd_sweep(fn, lo, hi, stride, _p(out))
    return out


def _bits(x):
    return int(np.float32(x).view(np.uint32))


def test_exp_within_one_ulp_of_correctly_rounded(xh):
    """exp on (-Inf, 0]: every Float32 in [-104, 0] (below, every result rounds to 0), then every 61st bit pattern to -Inf"""
    full = _sweep(xh, 0, 0x80000000, _bits(-104.0), 1)
    assert full[0] == _bits(-104.0) - 0x80000000 + 1
    tail = _sweep(xh, 0, _bits(-104.0), 0xFF800000, 61)
    for out in (full, tail):
        assert out[2] <= 1, (out, np.uint32(out[3]).view(np.float32))
    assert full[1] < 1e-6 * full[0]                                  # off by one ulp only next to a halfway point
    assert tail[1] == 0


def test_log_within_one_ulp_of_correctly_rounded(xh):
    """log on [0, +Inf]: every Float32 in [2^-30, 32] (u, -log(u) and the softmax sums live there), every 61st bit pattern
    over the rest"""
    for lo, hi, stride in ((_bits(2.0 ** -30), _bits(32.0), 1), (0, _bits(2.0 ** -30), 61), (_bits(32.0), 0x7F800000, 61)):
        out = _sweep(xh, 1, lo, hi, stride)
        assert out[2] <= 1, (out, np.uint32(out[3]).view(np.float32))
        assert out[1] < 1e-6 * out[0] + 1


def test_pinned_speedy_numbers(xh, pkg):
    """RLFarm test/algorithms/explorers/epsilon_speedy_explorer.jl:17-21, 52, 71"""
    ex = pkg.EpsilonSpeedyExplorer(0.1)
    assert ex.step == 1 and ex.beta == 0.1
    assert ex.get_eps() == pytest.approx(math.exp(-0.1), rel=1e-15) and xh.hd_speedy_eps(0.1, 1) == ex.get_eps()
    ex.step = 10
    assert ex.get_eps() == pytest.approx(math.exp(-1.0), rel=1e-15) and xh.hd_speedy_eps(0.1, 10) == ex.get_eps()
    ex2 = pkg.EpsilonSpeedyExplorer(1e-5, step=10 ** 5)
    assert ex2.get_eps() == pytest.approx(0.36787944117144233, rel=1e-15) and xh.hd_speedy_eps(1e-5, 10 ** 5) == ex2.get_eps()
    p = pkg.EpsilonSpeedyExplorer(0.1).prob([1, 2, 3, 4, 5])
    np.testing.assert_allclose(p, [0.1809674836071919] * 4 + [0.2761300655712324], rtol=1e-15)
    assert pkg.EpsilonSpeedyExplorer(0.1).prob([1, 2, 3, 4, 5], 5) == p[4]
    assert R.speedy_eps(0.1, 1) == ex.get_eps(1) and R.speedy_eps(1e-5, 10 ** 5) == ex2.get_eps()


def test_weighted_softmax_prob_is_softmax(pkg):
    q = [1.0, 2.0, 3.0, 4.0, 5.0]
    p = pkg.WeightedSoftmaxExplorer().prob(q)
    e = np.exp(np.array(q) - 5.0)
    np.testing.assert_allclose(p, e / e.sum(), rtol=2e-7)
    np.testing.assert_allclose(p, np.array(R.softmax(q), np.float32), rtol=2e-7)
    assert pkg.WeightedSoftmaxExplorer().prob([INF, 0.0, INF]).tolist() == [0.5, 0.0, 0.5]


@pytest.mark.parametrize("kind", [3, 4])
def test_action_frequencies_chi_square(xh, pkg, kind):
    from scipy.stats import chisquare
    q = np.array([0.3, -1.2, 1.1, 0.05], np.float32)
    n = 1 << 20
    rng = O.splitmix_states_fast(n, 40 + kind)
    a = np.empty(n, np.int32)
    st = _struct(pkg, kind)
    xh.hd_plan_fixed(C.byref(st), _p(q), 4, n, _p(rng), _p(a))
    counts = np.bincount(a, minlength=5)[1:]
    p = np.exp(q.astype(np.float64) - q.max())
    p /= p.sum()
    assert chisquare(counts, p * n).pvalue > 1e-4, counts


def test_explorer_struct_layout(xh, pkg):
    off = np.zeros(8, np.int64)
    size = xh.hd_explorer_layout(_p(off))
    E = pkg._lib.Explorer
    assert size == C.sizeof(E) == 56
    names = ["eps_stable", "eps_init", "warmup_steps", "decay_steps", "step", "kind", "is_break_tie", "beta"]
    assert [f[0] for f in E._fields_] == names
    assert off.tolist() == [getattr(E, n).offset for n in names]


@pytest.mark.parametrize("brk", [False, True])
def test_kinds_zero_and_one_unchanged(xh, pkg, brk):
    """the ϵ-greedy kinds through the same entry point: explorers.py's schedule and the oracle's selection"""
    n, na = 3000, 3
    q = np.asfortranarray(np.random.default_rng(5).standard_normal((na, n)).astype(np.float32))
    q[:, ::7] = q[0, ::7]
    for kind in ("linear", "exp"):
        ex = pkg.EpsilonGreedyExplorer(0.05, kind=kind, eps_init=0.9, warmup_steps=500, decay_steps=1500, step=200, is_break_tie=brk)
        st = ex.as_struct()
        assert st.beta == 0.0 and st.kind == (0 if kind == "linear" else 1)
        rng = O.splitmix_states_fast(n, 9)
        a, r = np.empty(n, np.int32), rng.copy()
        xh.hd_plan(C.byref(st), 200, _p(q), na, n, _p(r), _p(a))
        rr = rng.copy()
        ref = O.egreedy_plan(O.explorer6(0.05, 0.9, 500, 1500, kind, brk), 200, q, rr)
        assert np.array_equal(a, ref) and np.array_equal(r, rr)


def test_python_explorers(pkg):
    s = pkg.EpsilonSpeedyExplorer(0.5, step=3)
    st = s.as_struct()
    assert (st.kind, st.beta, st.step) == (2, 0.5, 3)
    s.advance(10)
    assert s.step == 13
    assert pkg.WeightedSoftmaxExplorer().as_struct().kind == 3 and pkg.GumbelSoftmaxExplorer().as_struct().kind == 4
    with pytest.raises(ValueError):
        pkg.EpsilonSpeedyExplorer(float("nan"))
    # the device agent loop takes the new explorers (the env side is checked per run)
    assert all(t in pkg.learners.DEVICE_EXPLORERS for t in (pkg.EpsilonSpeedyExplorer, pkg.WeightedSoftmaxExplorer, pkg.GumbelSoftmaxExplorer))
