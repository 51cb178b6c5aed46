// greedy.cuh — the greedy policy head: plan! without sampling (b200rl_net_act_greedy, b200rl_evaluate mode 0).
//
//   categorical logits / Q-values : findmax(z)[2], 1-based (GreedyExplorer, explorers/epsilon_greedy_explorer.jl:196-204;
//                                   CategoricalNetwork without sampling, RLCore/src/utils/networks.jl:403-420)
//   Gaussian heads                : mu (GaussianNetwork(...; is_sampling = false), networks.jl:64-100)
//
// findmax follows Julia Base: a left-to-right reduction that keeps the current maximum unless isless(max, x), so the first
// maximum wins, NaN ranks above every number (and the first NaN wins) and -0.0 ranks below 0.0.  (Recalled from Base, like
// the other stdlib semantics of DESIGN.md §2; unpinned.)  Plain C++ once the CUDA qualifiers are defined away, so the CPU
// suite compiles this file for the host (tests/hostdev/cuda_runtime.h).
#pragma once
#include <cstdint>
#include <cstring>

namespace greedy {

__host__ __device__ __forceinline__ uint32_t f32_bits(float x) {
    uint32_t b;
    memcpy(&b, &x, 4);
    return b;
}

// Base.isless(a::Float32, b::Float32)
__host__ __device__ __forceinline__ bool jl_isless(float a, float b) {
    if (a != a) return false;                       // NaN is not less than anything
    if (b != b) return true;                        // every number is less than NaN
    if (a == b) return (f32_bits(a) >> 31) > (f32_bits(b) >> 31);   // -0.0 < 0.0
    return a < b;
}

// findmax(z[0 .. n))[2] - 1 (0-based), 1 <= n <= NMAX (unrolled over NMAX: z stays in registers)
template <int NMAX>
__host__ __device__ __forceinline__ int findmax_index(const float (&z)[NMAX], int n) {
    int best = 0;
    float m = z[0];
#pragma unroll
    for (int o = 1; o < NMAX; ++o)
        if (o < n && jl_isless(m, z[o])) { m = z[o]; best = o; }
    return best;
}

// the greedy action of one sample as raw 32 bits: int32 1-based for a single head (logits, Q-values), the Float32 mu of a
// Gaussian head pair.  Desc: anything with `nout` and `heads2` (MlpDesc).
template <class Desc, int NMAX>
__host__ __device__ __forceinline__ uint32_t greedy_action(const Desc& d, const float (&z)[NMAX]) {
    if (d.heads2) return f32_bits(z[0]);
    return (uint32_t)(findmax_index(z, d.nout) + 1);
}

}  // namespace greedy
