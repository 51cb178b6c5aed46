// explore.cuh — one column of BatchExplorer(EpsilonGreedyExplorer) (explorers/batch_explorer.jl:15-21,
// epsilon_greedy_explorer.jl:69-112): get_ϵ(step), the uniform draw and the arg-max / random choice on the column's own
// Xoshiro256++ stream.  q_explore_kernel (b200rl_net_q_explore) and the replay driver's staged collect run this code.
// Plain C++ once the CUDA qualifiers are defined away, so the CPU suite compiles this file for the host
// (tests/hostdev/cuda_runtime.h, g++ -ffp-contract=off) and checks it against explorers.py and the oracle.
#pragma once
#include <cmath>
#include <cstdint>

#include "../../include/b200rl.h"

namespace explore {

// Float64 operations with explicit rounding on the device (no FMA contraction, like the reference's Julia code); the host
// build gets the same rounding points from -ffp-contract=off
#ifdef __CUDA_ARCH__
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ unsigned long long mul64hi(unsigned long long a, unsigned long long b) { return __umul64hi(a, b); }
#else
inline unsigned long long mul64hi(unsigned long long a, unsigned long long b) { return (unsigned long long)(((unsigned __int128)a * b) >> 64); }
inline double dadd(double a, double b) { return a + b; }
inline double dsub(double a, double b) { return a - b; }
inline double dmul(double a, double b) { return a * b; }
inline double ddiv(double a, double b) { return a / b; }
#endif

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

// rand(rng, Base.OneTo(n)) — Lemire nearly-divisionless on UInt64 (Julia 1.10 SamplerRangeNDL), 1-based
__host__ __device__ __forceinline__ int xo_oneto(unsigned long long (&s)[4], unsigned long long n) {
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
    return (int)hi + 1;
}

// get_ϵ(s::EpsilonGreedyExplorer{:linear | :exp}, step) (epsilon_greedy_explorer.jl:69-91): Float64, left to right
__host__ __device__ __forceinline__ double explorer_eps(const b200rl_explorer& e, long long step) {
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

// The column planned with get_ϵ(step) on Q-values v[0 .. na): rand(rng) >= ϵ ? (findmax | rand(rng, find_all_max)) :
// rand(rng, 1:na); 1-based.  The uniform draw happens even when ϵ = 0, exactly like the reference.
__host__ __device__ __forceinline__ int select(const b200rl_explorer& ex, long long step, const float* v, int na, unsigned long long (&st)[4]) {
    const double eps = explorer_eps(ex, step);
    const double u = xo_f64(st);
    int action;
    if (u >= eps) {
        int best = 0;
        for (int o = 1; o < na; ++o) {
            const float a = v[o], b = v[best];
            if ((a != a && b == b) || a > b) best = o;     // findmax: first maximum, NaN ranks highest
        }
        action = best + 1;
        if (ex.is_break_tie) {
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

}  // namespace explore
