// policy.cuh — the policy head of the actor-critic learners, once for every kernel that samples from it or differentiates it:
//   sample_head  the action and its log-probability on the env's policy stream: sample_categorical (networks.jl:425-432, Gumbel-max
//                on Float64 uniforms) or GaussianNetwork (networks.jl:64-116, Box–Muller on two Float32 uniforms)
//   sample_loss  one sample's PPO clipped surrogate / A2C term, entropy and their gradient with respect to the head outputs, or the
//                critic's squared error (SURVEY Appendix B)
// The FFMA kernels (nn.cu: forward_kernel, ac_loss_grad_kernel) use them with NO = kOutMax head rows, the tensor-core kernels
// (fwd_tc.cu: policy inference, rollout, sampled evaluate; nn_tc.cu: K7) with NO = kOutMax and NO = 2.
// Plain C++ once the CUDA qualifiers are defined away, so the CPU suite compiles this file for the host (tests/hostdev/cuda_runtime.h,
// g++ -ffp-contract=off) and checks it against torch autograd, the oracle's Xoshiro and a NumPy Gumbel-max.
// Rounding: the Gaussian sample spells every operation out (__fmul_rn / __fadd_rn: no FMA, the reference's Julia semantics). The rest
// is plain arithmetic whose contraction follows the including translation unit (nn.cu / nn_tc.cu contract, fwd_tc.cu does not), so
// each kernel computes exactly what its own copy of this code computed.
#pragma once
#include <cmath>
#include <cstdint>

#include "explore.cuh"

struct AcHyper {  // scalars of the actor-critic losses (SURVEY Appendix B)
    float clip_range, w_actor, w_critic, w_entropy, min_sigma, max_sigma;
    int normalize_adv;
    int algo;  // 0 PPO clipped surrogate, 1 A2C (logp * advantage)
};

namespace policy {

constexpr float kLog2Pi = 1.8378770664093453f;

__device__ __forceinline__ float softplus_f(float x) { return x > 0.f ? x + log1pf(expf(-x)) : log1pf(expf(x)); }
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }
// diagnormlogpdf with d = 1 (distributions.jl:18-21, eps = 1f-8)
__device__ __forceinline__ float normlogpdf1(float mu, float sigma, float x) {
    float s = sigma + 1e-8f, v = s * s, dd = x - mu;
    return -0.5f * ((logf(v) + (dd * dd) / v) + kLog2Pi);
}
// log-softmax of the first na rows of z: lp[o] = (z[o] - m) - ls
template <int NO>
__device__ __forceinline__ void logsoftmax_shift(const float (&z)[NO], int na, float& m, float& ls) {
    m = -3.4e38f;
#pragma unroll
    for (int o = 0; o < NO; ++o) if (o < na) m = fmaxf(m, z[o]);
    float se = 0.f;
#pragma unroll
    for (int o = 0; o < NO; ++o) if (o < na) se += expf(z[o] - m);
    ls = logf(se);
}
// clamp(softplus(raw), min_sigma, max_sigma) of the Gaussian head
__device__ __forceinline__ float gaussian_sigma(const AcHyper& hp, float sp) { return fminf(fmaxf(sp, hp.min_sigma), hp.max_sigma); }

// one Gumbel(0, 1) draw in Float64 (one out-of-line copy: the double-precision log is ~150 instructions)
inline __device__ __noinline__ double gumbel64(double u) { return -log(-log(u)); }

// policy head: sample an action and its log-probability from the head outputs z (na rows, or {mu, raw sigma} when heads2) on
// the env's policy stream.  Categorical: na Float64 draws; Gaussian: two Float32 draws.  Returns the action as raw 32 bits
// (int32 1-based | float).
template <int NO>
__device__ __forceinline__ uint32_t sample_head(int heads2, int na, const AcHyper& hp, const float (&z)[NO], unsigned long long (&st)[4],
                                                float& logp) {
    if (!heads2) {
        float m, ls;
        logsoftmax_shift(z, na, m, ls);
        int best = 0;
        double bv = 0.0;
        float blp = 0.f;
#pragma unroll
        for (int o = 0; o < NO; ++o) {
            if (o < na) {
                const float lp = (z[o] - m) - ls;
                double u = explore::xo_f64(st);
                double gv = gumbel64(u) + (double)lp;
                if (o == 0 || gv > bv) { bv = gv; best = o; blp = lp; }
            }
        }
        logp = blp;
        return (uint32_t)(best + 1);
    }
    float mu = z[0], raw = z[1];
    float sigma = gaussian_sigma(hp, softplus_f(raw));
    float u1 = explore::xo_f32(st), u2 = explore::xo_f32(st);
    float n = __fmul_rn(sqrtf(__fmul_rn(-2.0f, logf(1.0f - u1))), cosf(__fmul_rn(6.2831855f, u2)));
    float a = __fadd_rn(mu, __fmul_rn(sigma, n));
    logp = normlogpdf1(mu, sigma, a);
    return __float_as_uint(a);
}

// The actor's surrogate term l0 (PPO: -min(r A, clip(r) A); A2C: -logp_a A) and dloss/dlogp_a, scaled by w_actor / B
__device__ __forceinline__ float surrogate(const AcHyper& hp, float inv_B, float logp_a, float lp_old, float A, float& l0) {
    float gsel;   // d(surrogate)/d(logp_a)
    if (hp.algo == 0) {
        float ratio = expf(logp_a - lp_old);
        float u = ratio * A;
        float rc = fminf(fmaxf(ratio, 1.0f - hp.clip_range), 1.0f + hp.clip_range);
        float cc = rc * A;
        l0 = -fminf(u, cc);
        bool inside = ratio >= 1.0f - hp.clip_range && ratio <= 1.0f + hp.clip_range;
        gsel = (u < cc || inside) ? u : 0.f;
    } else {
        l0 = -(logp_a * A);
        gsel = A;
    }
    return -hp.w_actor * inv_B * gsel;
}

// Per-sample loss and d(loss)/d(head outputs), gradients scaled by inv_B = 1 / (global minibatch size).
//   actor (role 0): l0 = surrogate term, l1 = entropy; a_bits = the action's raw 32 bits (int32 1-based | float), lp_old, A
//   critic (role 1): l0 = (ret - z[0])^2
template <int NO> struct LossOut { float dz[NO]; float l0, l1; };
template <int NO>
__device__ __forceinline__ LossOut<NO> sample_loss(int heads2, int na, int role, const AcHyper& hp, float inv_B, const float (&z)[NO],
                                                   float a_bits, float lp_old, float A, float ret) {
    LossOut<NO> r;
#pragma unroll
    for (int o = 0; o < NO; ++o) r.dz[o] = 0.f;
    r.l0 = 0.f; r.l1 = 0.f;
    if (role == 1) {
        float err = ret - z[0];
        r.l0 = err * err;
        r.dz[0] = -2.0f * hp.w_critic * inv_B * err;
        return r;
    }
    if (!heads2) {
        float lp[NO], pr[NO];
        float m, ls;
        logsoftmax_shift(z, na, m, ls);
        float Hent = 0.f;
#pragma unroll
        for (int o = 0; o < NO; ++o) {
            lp[o] = (z[o] - m) - ls;
            pr[o] = o < na ? expf(lp[o]) : 0.f;
            if (o < na) Hent -= pr[o] * lp[o];
        }
        int a = __float_as_int(a_bits) - 1;
        float logp_a = 0.f;
#pragma unroll
        for (int o = 0; o < NO; ++o) if (o == a) logp_a = lp[o];
        r.l1 = Hent;
        float dlogp = surrogate(hp, inv_B, logp_a, lp_old, A, r.l0);
#pragma unroll
        for (int o = 0; o < NO; ++o)
            if (o < na) r.dz[o] = dlogp * ((o == a ? 1.f : 0.f) - pr[o]) + hp.w_entropy * inv_B * pr[o] * (lp[o] + Hent);
    } else {
        float mu = z[0], raw = z[1];
        float sp = softplus_f(raw);
        float sigma = gaussian_sigma(hp, sp);
        bool clamped = sp < hp.min_sigma || sp > hp.max_sigma;
        float a = a_bits;
        float logp_a = normlogpdf1(mu, sigma, a);
        float Hent = logf(sigma) + 0.5f * (kLog2Pi + 1.0f);
        r.l1 = Hent;
        float dlogp = surrogate(hp, inv_B, logp_a, lp_old, A, r.l0);
        float sgm = sigma + 1e-8f, dd = a - mu;
        r.dz[0] = dlogp * (dd / (sgm * sgm));
        float dsig = dlogp * (-1.0f / sgm + (dd * dd) / (sgm * sgm * sgm)) - hp.w_entropy * inv_B * (1.0f / sigma);
        r.dz[1] = clamped ? 0.f : dsig * sigmoid_f(raw);
    }
    return r;
}

}  // namespace policy
