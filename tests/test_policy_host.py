"""Host side of the policy head (no GPU).

csrc/policy.cuh (the sampler and the per-sample PPO / A2C loss gradient every learner kernel runs) compiled for the host:
sample_loss against torch float64 autograd of the reference formulas (PPO and A2C, categorical na = 1..4 and Gaussian heads, ratios
inside, outside and exactly on the clip edges, sigma clamped at either bound or free, the critic), the two head widths the kernels
instantiate agreeing bit for bit; sample_head advancing the policy stream exactly like the oracle's sampler, its categorical action
against a NumPy Gumbel-max restatement and the oracle, its Gaussian action and log-probability within float32 tolerance."""
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
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
// what policy.cuh uses beyond the stub: the rounded single-precision intrinsics (g++ runs with -ffp-contract=off: each operation
// rounds once), the bit casts, and the out-of-line qualifier of gumbel64 (defined here, after the standard headers)
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline int __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
static inline unsigned __float_as_uint(float f) { unsigned i; std::memcpy(&i, &f, 4); return i; }
#define __noinline__ __attribute__((noinline))
#include "policy.cuh"

static AcHyper hyper(const float* h, int algo) { return AcHyper{h[0], h[1], h[2], h[3], h[4], h[5], 0, algo}; }

// per sample k: z (4), {a_bits, lp_old, A, ret} -> out (6) = {dz[0..3], l0, l1}
template <int NO>
static void loss(int heads2, int na, int role, const float* h, int algo, float inv_B, const float* z, const float* aux, long long N, float* out) {
    const AcHyper hp = hyper(h, algo);
    for (long long k = 0; k < N; ++k) {
        float zz[NO];
        for (int o = 0; o < NO; ++o) zz[o] = z[4 * k + o];
        const float* x = aux + 4 * k;
        const policy::LossOut<NO> r = policy::sample_loss(heads2, na, role, hp, inv_B, zz, x[0], x[1], x[2], x[3]);
        for (int o = 0; o < 4; ++o) out[6 * k + o] = o < NO ? r.dz[o] : 0.f;
        out[6 * k + 4] = r.l0;
        out[6 * k + 5] = r.l1;
    }
}
extern "C" void hd_loss4(int heads2, int na, int role, const float* h, int algo, float inv_B, const float* z, const float* aux, long long N,
                         float* out) { loss<4>(heads2, na, role, h, algo, inv_B, z, aux, N, out); }
extern "C" void hd_loss2(int heads2, int na, int role, const float* h, int algo, float inv_B, const float* z, const float* aux, long long N,
                         float* out) { loss<2>(heads2, na, role, h, algo, inv_B, z, aux, N, out); }
extern "C" float hd_expf(float x) { return expf(x); }
// per sample k: z (4), stream st (4 words, advanced) -> action bits, logp
extern "C" void hd_sample(int heads2, int na, const float* h, const float* z, long long N, unsigned long long* st, uint32_t* a, float* logp) {
    const AcHyper hp = hyper(h, 0);
    for (long long k = 0; k < N; ++k) {
        float zz[4] = {z[4 * k], z[4 * k + 1], z[4 * k + 2], z[4 * k + 3]};
        unsigned long long s[4];
        explore::xo_load(st, k, s);
        a[k] = policy::sample_head(heads2, na, hp, zz, s, logp[k]);
        explore::xo_store(st, k, s);
    }
}
"""

LOG2PI = math.log(2.0 * math.pi)


@pytest.fixture(scope="module")
def ph(tmp_path_factory):
    d = tmp_path_factory.mktemp("policy")
    src, so = d / "policy_driver.cpp", d / "libpolicy.so"
    src.write_text(DRIVER)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wno-unknown-pragmas",
                           "-I", HD, "-I", CSRC, "-shared", "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    vp = C.c_void_p
    for f in (L.hd_loss4, L.hd_loss2):
        f.restype = None
        f.argtypes = [C.c_int, C.c_int, C.c_int, vp, C.c_int, C.c_float, vp, vp, C.c_longlong, vp]
    L.hd_expf.restype, L.hd_expf.argtypes = C.c_float, [C.c_float]
    L.hd_sample.restype = None
    L.hd_sample.argtypes = [C.c_int, C.c_int, vp, vp, C.c_longlong, vp, vp, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def hyper(clip_range=0.2, w_actor=1.0, w_critic=0.5, w_entropy=0.01, min_sigma=0.0, max_sigma=np.inf):
    return np.array([clip_range, w_actor, w_critic, w_entropy, min_sigma, max_sigma], np.float32)


def header_loss(ph, heads2, na, role, h, algo, inv_B, z, aux, width=4):
    z4 = np.zeros((len(z), 4), np.float32)
    z4[:, :np.shape(z)[1]] = z
    aux = np.ascontiguousarray(aux, np.float32)
    out = np.full((len(z), 6), np.nan, np.float32)
    (ph.hd_loss4 if width == 4 else ph.hd_loss2)(heads2, na, role, _p(h), algo, inv_B, _p(z4), _p(aux), len(z), _p(out))
    return out


def action_bits(a, gaussian):
    return np.asarray(a, np.float32) if gaussian else np.asarray(a, np.int32).view(np.float32)


def ref_loss(heads2, na, role, h, algo, inv_B, z, aux, ratio0=None):
    """torch float64 autograd of one sample's weighted loss w_actor/B * surrogate - w_entropy/B * entropy (actor) or
    w_critic/B * (ret - V)^2 (critic) -> (dz, l0, l1).  ratio0 (optional): the ratio's value at z, its derivative that of
    exp(logp_a(z)) (puts the ratio exactly where the header's float32 ratio is, for the clip-edge cases)."""
    import torch
    clip, w_a, w_c, w_e, smin, smax = [float(x) for x in h]
    zt = torch.tensor(np.asarray(z, np.float64), requires_grad=True)
    a_bits, lp_old, A, ret = [float(x) for x in np.asarray(aux, np.float32)]
    if role == 1:
        l0 = (ret - zt[0]) ** 2
        (w_c * inv_B * l0).backward()
        return zt.grad.numpy(), l0.item(), 0.0
    if not heads2:
        a = int(np.float32(a_bits).view(np.int32)) - 1
        lp = torch.log_softmax(zt[:na], 0)
        ent = -(lp.exp() * lp).sum()
        logp_a = lp[a]
    else:
        mu, raw = zt[0], zt[1]
        sigma = torch.clamp(torch.nn.functional.softplus(raw), smin, smax)
        s = sigma + 1e-8
        logp_a = -0.5 * ((torch.log(s * s) + (a_bits - mu) ** 2 / (s * s)) + LOG2PI)
        ent = torch.log(sigma) + 0.5 * (LOG2PI + 1.0)
    if algo == 0:
        ratio = torch.exp(logp_a - lp_old) if ratio0 is None else ratio0 * torch.exp(logp_a - logp_a.detach())
        l0 = -torch.minimum(ratio * A, torch.clamp(ratio, 1.0 - clip, 1.0 + clip) * A)
    else:
        l0 = -(logp_a * A)
    (w_a * inv_B * l0 - w_e * inv_B * ent).backward()
    g = zt.grad.numpy()
    return g, l0.item(), ent.item()


def check_loss(ph, heads2, na, role, h, algo, z, aux, inv_B=1.0 / 64, ratio0=None, rtol=1e-4):
    got = header_loss(ph, heads2, na, role, h, algo, inv_B, z, aux)
    nz = 1 if role else (2 if heads2 else na)
    for k in range(len(z)):
        r0 = None if ratio0 is None else ratio0[k]
        dz, l0, l1 = ref_loss(heads2, na, role, h, algo, inv_B, z[k][:nz], aux[k], r0)
        scale = inv_B * max(1.0, abs(float(aux[k][2])), abs(l0))
        np.testing.assert_allclose(got[k, :nz], dz, rtol=rtol, atol=1e-6 * scale, err_msg=f"dz sample {k}")
        assert np.all(got[k, nz:4] == 0)
        assert got[k, 4] == pytest.approx(l0, rel=rtol, abs=1e-6 * max(1.0, abs(l0)))
        assert got[k, 5] == pytest.approx(l1, rel=rtol, abs=1e-6)
    if nz <= 2:   # the tensor-core kernel's width: the same bits
        got2 = header_loss(ph, heads2, na, role, h, algo, inv_B, z, aux, width=2)
        assert np.array_equal(got2[:, :2].view(np.uint32), got[:, :2].view(np.uint32))
        assert np.array_equal(got2[:, 4:].view(np.uint32), got[:, 4:].view(np.uint32))
    return got


def logp_of(ph, heads2, na, h, z, a):
    """the header's own float32 log-probability of each action: A2C with A = 1 makes l0 = -logp_a exactly"""
    aux = np.zeros((len(z), 4), np.float32)
    aux[:, 0] = action_bits(a, heads2)
    aux[:, 2] = 1.0
    return -header_loss(ph, heads2, na, 0, h, 1, 1.0, z, aux)[:, 4]


def cases(rng, heads2, na, n):
    if heads2:
        z = np.stack([rng.normal(0, 1, n), rng.normal(0, 1.5, n)], 1).astype(np.float32)
        a = (z[:, 0] + rng.normal(0, 1, n)).astype(np.float32)
    else:
        z = rng.normal(0, 2, (n, na)).astype(np.float32)
        a = rng.integers(1, na + 1, n)
    return z, a


@pytest.mark.parametrize("heads2,na", [(0, 1), (0, 2), (0, 3), (0, 4), (1, 2)])
@pytest.mark.parametrize("algo", [0, 1])
def test_actor_loss_inside_and_outside_the_clip_range(ph, heads2, na, algo):
    rng = np.random.default_rng(10 * na + heads2 + 100 * algo)
    n, clip = 48, 0.2
    h = hyper(clip_range=clip)
    z, a = cases(rng, heads2, na, n)
    lp = logp_of(ph, heads2, na, h, z, a)
    # log-ratios well inside (-0.1 .. 0.1) and well outside on both sides (|log r| in 0.3 .. 1.5), advantages of both signs
    lr = np.concatenate([rng.uniform(-0.1, 0.1, n // 3), rng.uniform(0.3, 1.5, n // 3), -rng.uniform(0.3, 1.5, n - 2 * (n // 3))])
    aux = np.zeros((n, 4), np.float32)
    aux[:, 0] = action_bits(a, heads2)
    aux[:, 1] = (lp - lr).astype(np.float32)
    aux[:, 2] = rng.normal(0, 2, n).astype(np.float32)
    check_loss(ph, heads2, na, 0, h, algo, z, aux)


@pytest.mark.parametrize("heads2,na", [(0, 2), (0, 3), (1, 2)])
def test_ppo_ratio_exactly_on_the_clip_edges(ph, heads2, na):
    """ratio == 1 + clip and ratio == 1 - clip in float32 (the clip range is made from the header's own ratio), and
    clip = 0 with ratio 1 (both edges at once): the unclipped branch's gradient, like autograd's inclusive clamp"""
    rng = np.random.default_rng(7 + na + heads2)
    n = 12
    z, a = cases(rng, heads2, na, n)
    h0 = hyper()
    lp = logp_of(ph, heads2, na, h0, z, a)
    for k in range(n):
        d = np.float32([0.125, -0.125, 0.0][k % 3])
        lp_old = np.float32(lp[k] - d)
        dd = np.float32(lp[k] - lp_old)
        r = np.float32(ph.hd_expf(float(dd)))
        clip = np.float32(r - np.float32(1)) if d > 0 else (np.float32(np.float32(1) - r) if d < 0 else np.float32(0))
        edge = np.float32(np.float32(1) + clip) if d >= 0 else np.float32(np.float32(1) - clip)
        assert edge == r
        for A in (np.float32(1.5), np.float32(-0.75)):
            aux = np.array([[action_bits([a[k]], heads2)[0], lp_old, A, 0.0]], np.float32)
            got = check_loss(ph, heads2, na, 0, hyper(clip_range=clip), 0, z[k:k + 1], aux, ratio0=[float(r)])
            assert got[0, 4] == -(r * A)


@pytest.mark.parametrize("algo", [0, 1])
def test_gaussian_sigma_clamped_and_free(ph, algo):
    rng = np.random.default_rng(3 + algo)
    n = 30
    z, a = cases(rng, 1, 2, n)
    z[:, 1] = np.linspace(-3, 3, n, dtype=np.float32)          # softplus(raw) from 0.049 to 3.05
    for smin, smax in ((0.0, np.inf), (0.5, np.inf), (0.0, 1.0), (0.3, 1.2)):
        h = hyper(min_sigma=smin, max_sigma=smax)
        lp = logp_of(ph, 1, 2, h, z, a)
        aux = np.zeros((n, 4), np.float32)
        aux[:, 0] = a
        aux[:, 1] = (lp - rng.uniform(-0.05, 0.05, n)).astype(np.float32)
        aux[:, 2] = rng.normal(0, 1, n).astype(np.float32)
        got = check_loss(ph, 1, 2, 0, h, algo, z, aux)
        sp = np.log1p(np.exp(z[:, 1].astype(np.float64)))
        clamped = (sp < smin) | (sp > smax)
        assert np.all(got[clamped, 1] == 0) and np.all(got[~clamped, 1] != 0)
        if smin > 0 or np.isfinite(smax):
            assert clamped.any()


@pytest.mark.parametrize("heads2,na", [(0, 2), (1, 2), (0, 1)])
def test_critic_squared_error(ph, heads2, na):
    rng = np.random.default_rng(5)
    n = 20
    z = rng.normal(0, 3, (n, 1)).astype(np.float32)
    aux = np.zeros((n, 4), np.float32)
    aux[:, 3] = rng.normal(0, 10, n).astype(np.float32)
    got = check_loss(ph, heads2, na, 1, hyper(w_critic=0.5), 0, z, aux)
    err = aux[:, 3] - z[:, 0]
    assert np.array_equal(got[:, 4], err * err) and np.all(got[:, 5] == 0)


# ---- sample_head ---------------------------------------------------------------------------------------------------------
def header_sample(ph, heads2, na, h, z, st):
    z4 = np.zeros((len(z), 4), np.float32)
    z4[:, :np.shape(z)[1]] = z
    st = np.ascontiguousarray(st, np.uint64).copy()
    a = np.zeros(len(z), np.uint32)
    lp = np.zeros(len(z), np.float32)
    ph.hd_sample(heads2, na, _p(h), _p(z4), len(z), _p(st), _p(a), _p(lp))
    return a, lp, st


@pytest.mark.parametrize("heads2,na", [(0, 1), (0, 2), (0, 3), (0, 4), (1, 2)])
def test_stream_advance_matches_the_oracle(ph, heads2, na):
    """na Float64 draws (categorical) or two Float32 draws (Gaussian): the streams end where the oracle's sampler leaves them"""
    n = 256
    desc = O.ac_desc(4, 64, 1 if heads2 else na, gaussian=bool(heads2))
    params = O.glorot_params(desc, 1)
    obs = np.random.default_rng(2).standard_normal((4, n)).astype(np.float32)
    st0 = O.splitmix_states_fast(n, 99 + na + heads2)
    if heads2:
        ref = O.act_gaussian(desc, O.hyper_array(), params, obs, st0)
    else:
        ref = O.act_discrete(desc, params, obs, st0)
    z = np.random.default_rng(4).normal(0, 1, (n, 2 if heads2 else na)).astype(np.float32)
    _, _, st = header_sample(ph, heads2, na, hyper(), z, st0)
    assert np.array_equal(st, ref["rng"])
    if not heads2:   # fed the oracle's logits, the same action wherever the oracle's Gumbel-max is not a near-tie
        a, lp, _ = header_sample(ph, 0, na, hyper(), ref["logits"].T.copy(), st0)
        far = ref["margin"] > 1e-6
        assert far.sum() > n // 2
        assert np.array_equal(a[far].astype(np.int32), ref["action"][far])
        np.testing.assert_allclose(lp[far], ref["logp"][far], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("na", [1, 2, 3, 4])
def test_categorical_matches_numpy_gumbel_max(ph, na):
    n = 2000
    rng = np.random.default_rng(na)
    z = (rng.normal(0, 1.5, (n, na)) * rng.choice([0.1, 1.0, 5.0], (n, 1))).astype(np.float32)
    st0 = O.splitmix_states_fast(n, 1234 + na)
    a, lp, st = header_sample(ph, 0, na, hyper(), z, st0)
    checked = 0
    for k in range(n):
        s = [int(x) for x in st0[k]]
        lpk = z[k].astype(np.float64) - np.logaddexp.reduce(z[k].astype(np.float64))
        g = np.array([-math.log(-math.log(R.rand_f64(s))) + lpk[o] for o in range(na)])
        assert s == [int(x) for x in st[k]]
        order = np.sort(g)
        if na > 1 and order[-1] - order[-2] < 1e-4:
            continue
        checked += 1
        best = int(np.argmax(g))
        assert a[k] == best + 1, k
        assert lp[k] == pytest.approx(lpk[best], rel=1e-5, abs=1e-6)
    assert checked > 0.95 * n


def test_gaussian_matches_box_muller(ph):
    n = 2000
    rng = np.random.default_rng(8)
    z = np.stack([rng.normal(0, 2, n), rng.normal(0, 1.5, n)], 1).astype(np.float32)
    for smin, smax in ((0.0, np.inf), (0.4, 1.1)):
        h = hyper(min_sigma=smin, max_sigma=smax)
        st0 = O.splitmix_states_fast(n, 77)
        a, lp, st = header_sample(ph, 1, 2, h, z, st0)
        a = a.view(np.float32)
        for k in range(n):
            s = [int(x) for x in st0[k]]
            u1, u2 = float(R.rand_f32(s)), float(R.rand_f32(s))
            assert s == [int(x) for x in st[k]]
            mu = float(z[k, 0])
            sigma = min(max(math.log1p(math.exp(float(z[k, 1]))), smin), smax)
            nn = math.sqrt(-2.0 * math.log(1.0 - u1)) * math.cos(float(np.float32(6.2831855)) * u2)
            ak = mu + sigma * nn
            assert a[k] == pytest.approx(ak, rel=1e-5, abs=1e-5 * (1 + abs(sigma * nn)))
            sg = sigma + 1e-8
            lpk = -0.5 * (math.log(sg * sg) + (float(a[k]) - mu) ** 2 / (sg * sg) + LOG2PI)
            assert lp[k] == pytest.approx(lpk, rel=1e-5, abs=1e-5)
