// explore.cuh — one column of BatchExplorer(inner explorer) (explorers/batch_explorer.jl:15-21) on the column's own Xoshiro256++
// stream, for the value-based explorers a QBasedPolicy plans with:
//   kinds 0 / 1  EpsilonGreedyExplorer{:linear | :exp} (epsilon_greedy_explorer.jl:69-112): get_ϵ(step), the uniform draw, the
//                arg-max / random choice
//   kind 2       EpsilonSpeedyExplorer(β) (RLFarm epsilon_speedy_explorer.jl:19-53): the same selection with ϵ = exp(-β·step)
//   kind 3       WeightedSoftmaxExplorer (weighted_softmax_explorer.jl:20-21): sample(rng, Weights(softmax(Q), 1f0))
//   kind 4       GumbelSoftmaxExplorer (gumbel_softmax_explorer.jl:12-16): argmax(logsoftmax(Q) .- log.(-log.(rand(rng, Float32, n))))
// q_explore_kernel (b200rl_net_q_explore), the replay driver's staged collect and the fused collect run this code; on a sharded
// ctx they number the columns globally (column_step).
// Plain C++ once the CUDA qualifiers are defined away, so the CPU suite compiles this file for the host
// (tests/hostdev/cuda_runtime.h, g++ -ffp-contract=off) and checks it against explorers.py, the oracle and a NumPy restatement.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#include "../../include/b200rl.h"
#include "greedy.cuh"

namespace explore {

// Float64 operations with explicit rounding on the device (no FMA contraction, like the reference's Julia code); the host
// build gets the same rounding points from -ffp-contract=off
#ifdef __CUDA_ARCH__
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ unsigned long long mul64hi(unsigned long long a, unsigned long long b) { return __umul64hi(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float d2f(double a) { return __double2float_rn(a); }
#else
inline unsigned long long mul64hi(unsigned long long a, unsigned long long b) { return (unsigned long long)(((unsigned __int128)a * b) >> 64); }
inline double dadd(double a, double b) { return a + b; }
inline double dsub(double a, double b) { return a - b; }
inline double dmul(double a, double b) { return a * b; }
inline double ddiv(double a, double b) { return a / b; }
inline float fadd(float a, float b) { return a + b; }
inline float fsub(float a, float b) { return a - b; }
inline float fdiv(float a, float b) { return a / b; }
inline float d2f(double a) { return (float)a; }
#endif

// Xoshiro256++ on a 4-word state held in registers.  Streams live in memory as 4 consecutive words per column (rng + 4 i),
// moved as two 16-byte vectors.
__host__ __device__ __forceinline__ void xo_load(const unsigned long long* rng, int64_t i, unsigned long long (&s)[4]) {
    const ulonglong2* p = reinterpret_cast<const ulonglong2*>(rng + 4 * i);
    ulonglong2 a = p[0], b = p[1];
    s[0] = a.x; s[1] = a.y; s[2] = b.x; s[3] = b.y;
}
__host__ __device__ __forceinline__ void xo_store(unsigned long long* rng, int64_t i, const unsigned long long (&s)[4]) {
    ulonglong2* p = reinterpret_cast<ulonglong2*>(rng + 4 * i);
    p[0] = make_ulonglong2(s[0], s[1]);
    p[1] = make_ulonglong2(s[2], s[3]);
}
__host__ __device__ __forceinline__ unsigned long long xo_next(unsigned long long (&s)[4]) {
    unsigned long long tmp = s[0] + s[3];
    unsigned long long res = ((tmp << 23) | (tmp >> 41)) + s[0];
    unsigned long long t = s[1] << 17;
    s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3]; s[2] ^= t;
    s[3] = (s[3] << 45) | (s[3] >> 19);
    return res;
}
// rand(rng, Float64)
__host__ __device__ __forceinline__ double xo_f64(unsigned long long (&s)[4]) { return (double)(xo_next(s) >> 11) * 0x1p-53; }
// rand(rng, Float32): jl_device.cuh's rand_f32 on this stream layout (an output of 0 happens: its top 24 bits all zero)
__host__ __device__ __forceinline__ float xo_f32(unsigned long long (&s)[4]) { return (float)((unsigned)(xo_next(s) >> 32) >> 8) * 0x1p-24f; }

// rand(rng, Base.OneTo(n)) - 1 — Lemire nearly-divisionless on UInt64 (Julia 1.10 SamplerRangeNDL), 0-based, n up to 2^64 - 1
__host__ __device__ __forceinline__ unsigned long long xo_below(unsigned long long (&s)[4], unsigned long long n) {
    unsigned long long x = xo_next(s);
    unsigned long long hi = mul64hi(x, n), lo = x * n;
    if (lo < n) {
        unsigned long long t = (0ull - n) % n;
        while (lo < t) {
            x = xo_next(s);
            hi = mul64hi(x, n);
            lo = x * n;
        }
    }
    return hi;
}
// rand(rng, Base.OneTo(n)), 1-based, for n within int (action counts)
__host__ __device__ __forceinline__ int xo_oneto(unsigned long long (&s)[4], unsigned long long n) { return (int)xo_below(s, n) + 1; }

// get_ϵ(s::EpsilonGreedyExplorer{:linear | :exp}, step) (epsilon_greedy_explorer.jl:69-91): Float64, left to right
// Ex: b200rl_explorer, or any struct with its schedule fields (the fused collect's kernel argument)
template <class Ex>
__host__ __device__ __forceinline__ double explorer_eps(const Ex& e, long long step) {
    if (step <= e.warmup_steps) return e.eps_init;
    if (e.kind == 0) {
        if (step >= e.warmup_steps + e.decay_steps) return e.eps_stable;
        long long steps_left = e.warmup_steps + e.decay_steps - step;
        return dadd(e.eps_stable, dmul(ddiv((double)steps_left, (double)e.decay_steps), dsub(e.eps_init, e.eps_stable)));
    }
    long long n = step - e.warmup_steps;
    double scale = dsub(e.eps_init, e.eps_stable);
    return dadd(e.eps_stable, dmul(scale, exp(ddiv(dmul(-1.0, (double)n), (double)e.decay_steps))));
}

// get_ϵ(s::EpsilonSpeedyExplorer) at `step` (epsilon_speedy_explorer.jl:35-37): exp(β_neg * step), β_neg = β * -1, in Float64 with
// the device's exp
__host__ __device__ __forceinline__ double speedy_eps(double beta, long long step) { return exp(dmul(dmul(beta, -1.0), (double)step)); }

// rand(rng) >= ϵ ? (findmax | rand(rng, find_all_max)) : rand(rng, 1:na) on Q-values v[0 .. na); 1-based.  The uniform draw
// happens even when ϵ = 0, exactly like the reference.
__host__ __device__ __forceinline__ int eps_select(double eps, bool break_tie, const float* v, int na, unsigned long long (&st)[4]) {
    const double u = xo_f64(st);
    int action;
    if (u >= eps) {
        int best = 0;
        for (int o = 1; o < na; ++o) {
            const float a = v[o], b = v[best];
            if ((a != a && b == b) || a > b) best = o;     // findmax: first maximum, NaN ranks highest
        }
        action = best + 1;
        if (break_tie) {
            float mx = v[0];
            for (int o = 1; o < na; ++o) mx = v[o] > mx ? v[o] : mx;
            int cnt = 0;
            for (int o = 0; o < na; ++o) cnt += v[o] == mx;
            int pick = xo_oneto(st, (unsigned long long)(cnt > 0 ? cnt : 1));
            for (int o = 0; o < na; ++o) {
                if (v[o] == mx && --pick == 0) { action = o + 1; break; }
            }
        }
    } else {
        action = xo_oneto(st, (unsigned long long)na);
    }
    return action;
}

// ---- Float32 exp / log of the softmax explorers ---------------------------------------------------------------------------
// Each is a Float64 evaluation made of single IEEE operations (no FMA, no library call) rounded once to Float32, so the host and
// device builds give the same bits.  The Float64 result is within 2^-50 (relative) of the true value, so the Float32 result is the
// correctly rounded one except where the true value lies within that distance of a halfway point, and then one ulp away.
// (Julia's own Float32 exp / log are table-driven Float32 kernels that are not restated here: like the rest of DESIGN.md §2 these
// semantics are recalled, and the two agree wherever both round correctly.)
constexpr int kMaxActions = 4;     // n_out of a Q-network
__host__ __device__ __forceinline__ double bits_to_f64(unsigned long long b) { double d; memcpy(&d, &b, 8); return d; }
__host__ __device__ __forceinline__ unsigned long long f64_to_bits(double d) { unsigned long long b; memcpy(&b, &d, 8); return b; }
__host__ __device__ __forceinline__ float bits_to_f32(uint32_t b) { float f; memcpy(&f, &b, 4); return f; }

// exp(x::Float32).  x = k·ln2 + r with k = round(x / ln2) (|k| <= 151: k·LN2_HI is exact), |r| <= 0.35, exp(r) by its Taylor series
// to r^13 (truncation < 2^-57), times 2^k (a normal Float64: exact).  exp(-Inf) = 0, exp(+Inf) = Inf, exp(NaN) = NaN.
__host__ __device__ __forceinline__ float f32_exp(float x) {
    if (x != x) return x;
    if (x < -104.0f) return 0.0f;                   // exp(-104) < 2^-150: rounds to 0
    if (x > 89.0f) return bits_to_f32(0x7f800000u);
    const double xd = (double)x;
    const double k = dsub(dadd(dmul(xd, 1.4426950408889634), 0x1.8p52), 0x1.8p52);     // round to nearest
    const double r = dsub(dsub(xd, dmul(k, 6.93147180369123816490e-01)), dmul(k, 1.90821492927058770002e-10));
    double p = 1.0 / 6227020800.0;                   // 1/13!
    const double inv[13] = {1.0 / 479001600.0, 1.0 / 39916800.0, 1.0 / 3628800.0, 1.0 / 362880.0, 1.0 / 40320.0, 1.0 / 5040.0,
                            1.0 / 720.0, 1.0 / 120.0, 1.0 / 24.0, 1.0 / 6.0, 0.5, 1.0, 1.0};
#pragma unroll
    for (int j = 0; j < 13; ++j) p = dadd(dmul(p, r), inv[j]);
    return d2f(dmul(p, bits_to_f64((unsigned long long)((long long)k + 1023) << 52)));
}

// log(x::Float32) for x >= 0.  x = 2^e·m with m in [√2/2, √2) (subnormal x are normal Float64), log m = 2 atanh(s) with
// s = (m - 1)/(m + 1), |s| < 0.172, by its series to s^23 (truncation < 2^-60), plus e·ln2 in two parts.  log(0) = -Inf,
// log(+Inf) = +Inf, log(x < 0) = NaN, log(NaN) = NaN.
__host__ __device__ __forceinline__ float f32_log(float x) {
    if (x != x) return x;
    if (x < 0.0f) return bits_to_f32(0x7fc00000u);
    if (x == 0.0f) return bits_to_f32(0xff800000u);
    if (x == bits_to_f32(0x7f800000u)) return x;
    const unsigned long long b = f64_to_bits((double)x);
    int e = (int)((b >> 52) & 0x7ff) - 1023;
    double m = bits_to_f64((b & 0x000fffffffffffffull) | 0x3ff0000000000000ull);
    if (m > 1.4142135623730951) { m = dmul(m, 0.5); e += 1; }
    const double f = dsub(m, 1.0);                   // exact
    const double s = ddiv(f, dadd(2.0, f));
    const double s2 = dmul(s, s);
    double p = 1.0 / 23.0;
    const double inv[11] = {1.0 / 21.0, 1.0 / 19.0, 1.0 / 17.0, 1.0 / 15.0, 1.0 / 13.0, 1.0 / 11.0, 1.0 / 9.0, 1.0 / 7.0, 1.0 / 5.0,
                            1.0 / 3.0, 1.0};
#pragma unroll
    for (int j = 0; j < 11; ++j) p = dadd(dmul(p, s2), inv[j]);
    const double ed = (double)e;
    const double lm = dmul(dmul(2.0, s), p);
    return d2f(dadd(dmul(ed, 6.93147180369123816490e-01), dadd(dmul(ed, 1.90821492927058770002e-10), lm)));
}

// NNlib's max_ = fast_maximum(x) (@fastmath reduce(max, x; init = -Inf32)): NaN entries never win, so m = -Inf when every
// entry is NaN or -Inf
__host__ __device__ __forceinline__ float fast_maximum(const float* v, int na) {
    float m = bits_to_f32(0xff800000u);
#pragma unroll
    for (int o = 0; o < kMaxActions; ++o)
        if (o < na && v[o] > m) m = v[o];
    return m;
}

// sample(rng, Weights(softmax(v), 1f0)) (NNlib softmax, StatsBase's inverse CDF): one Float64 draw; 1-based
__host__ __device__ __forceinline__ int weighted_softmax_select(const float* v, int na, unsigned long long (&st)[4]) {
    const float inf = bits_to_f32(0x7f800000u);
    const float m = fast_maximum(v, na);
    const bool finite = fsub(m, m) == 0.0f;
    float e[kMaxActions];
#pragma unroll
    for (int o = 0; o < kMaxActions; ++o)            // out .= exp.(x .- max_), or NNlib's branch for a non-finite max_
        e[o] = o < na ? ((finite || m != inf) ? f32_exp(fsub(v[o], m)) : (v[o] == inf ? 1.0f : 0.0f)) : 0.0f;
    float s = e[0];
#pragma unroll
    for (int o = 1; o < kMaxActions; ++o)
        if (o < na) s = fadd(s, e[o]);
    const double t = xo_f64(st);                     // rand(rng) * sum(wv), sum(wv) = 1f0
    int i = 0;
    float cw = fdiv(e[0], s);
    bool go = true;
#pragma unroll
    for (int o = 1; o < kMaxActions; ++o) {          // while cw < t && i < n: i += 1; cw += p_i
        go = go && o < na && (double)cw < t;
        if (go) { i = o; cw = fadd(cw, fdiv(e[o], s)); }
    }
    return i + 1;
}

// argmax(logsoftmax(v) .- log.(-log.(u))), u = rand(rng, Float32, na): na Float32 draws; findmax order (greedy.cuh); 1-based
__host__ __device__ __forceinline__ int gumbel_softmax_select(const float* v, int na, unsigned long long (&st)[4]) {
    const float inf = bits_to_f32(0x7f800000u);
    const float m = fast_maximum(v, na);
    const bool finite = fsub(m, m) == 0.0f;
    float d[kMaxActions];
#pragma unroll
    for (int o = 0; o < kMaxActions; ++o)            // out .= x .- max_, or NNlib's branch for a non-finite max_
        d[o] = o < na ? ((finite || m != inf) ? fsub(v[o], m) : (v[o] == inf ? 0.0f : -inf)) : 0.0f;
    float s = f32_exp(d[0]);
#pragma unroll
    for (int o = 1; o < kMaxActions; ++o)            // sum(exp, out), left to right
        if (o < na) s = fadd(s, f32_exp(d[o]));
    const float lse = f32_log(s);
    float g[kMaxActions] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
    for (int o = 0; o < kMaxActions; ++o)
        if (o < na) g[o] = fsub(fsub(d[o], lse), f32_log(-f32_log(xo_f32(st))));    // u = 0: log(0) = -Inf -> g = -Inf
    return greedy::findmax_index(g, na) + 1;
}

// The explorer step of local column i at plan k of a window that starts at explorer step `step`, for a batch sharded over the
// ranks of a communicator (DESIGN.md §3): rank r of G owns N columns, numbered globally r·N + i, and every plan! of the whole
// batch moves the step by G·N — what one BatchExplorer over the G·N columns does.  col0 = r·N, stride = G·N; on one GPU (col0 = 0,
// stride = N) this is step + k·N + i.
__host__ __device__ __forceinline__ long long column_step(long long step, long long col0, long long stride, long long k, long long i) {
    return step + col0 + k * stride + i;
}

// The column planned at explorer step `step` on Q-values v[0 .. na), 1-based.  EXT = false compiles kinds 0 and 1 only (the
// fused collect instantiations of the ϵ-greedy explorer); the caller routes kinds 2-4 to an EXT = true instantiation.
// Ex: b200rl_explorer, or (EXT = false) any struct with its schedule fields.
template <bool EXT = true, class Ex = b200rl_explorer>
__host__ __device__ __forceinline__ int select(const Ex& ex, long long step, const float* v, int na, unsigned long long (&st)[4]) {
    if constexpr (EXT) {
        if (ex.kind >= 2) {
            if (ex.kind == 3) return weighted_softmax_select(v, na, st);
            if (ex.kind == 4) return gumbel_softmax_select(v, na, st);
            return eps_select(speedy_eps(ex.beta, step), false, v, na, st);
        }
    }
    return eps_select(explorer_eps(ex, step), ex.is_break_tie != 0, v, na, st);
}

}  // namespace explore
