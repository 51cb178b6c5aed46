// duel.cuh — the combine of a dueling Q-network's heads and its backward (DuelingNetwork, RLCore/src/utils/networks.jl:500-522):
//
//   Q = val .+ adv .- mean(adv, dims = 1)     parsed as (val .+ adv) .- mean
//
// z = {v, a_1 .. a_n} (the head rows, val first), n = number of actions (1 <= n <= M - 1):
//   μ   = ((0f0 + a_1) + a_2 + ... + a_n) / Float32(n)      Statistics' _mean: sum(...; dims) ./= n, sequential for short columns
//   Q_i = (v + a_i) - μ
// every operation rounded once (explicit __fadd_rn / __fsub_rn / __fdiv_rn: no FMA, no reassociation, whatever the including
// translation unit's flags).  The summation order and divide are recalled from the Statistics stdlib (unpinned, DESIGN.md §3).
//
// Backward, g = ∂ℓ/∂Q_a (a 0-based): ∂ℓ/∂v = g, ∂ℓ/∂a_j = (j == a ? g : 0) - g / Float32(n).
//
// Plain C++ once the CUDA qualifiers are defined away; the CPU suite compiles it for the host with its own rounded intrinsics.
#pragma once

namespace duel {

// z (head rows) -> z (Q in rows 0 .. n-1, zeros above), in place
template <int M>
__device__ __forceinline__ void combine(float (&z)[M], int n) {
    float s = 0.f;
#pragma unroll
    for (int j = 1; j < M; ++j)
        if (j <= n) s = __fadd_rn(s, z[j]);
    const float mu = __fdiv_rn(s, (float)n);
    const float v = z[0];
#pragma unroll
    for (int o = 0; o < M; ++o) z[o] = o < n ? __fsub_rn(__fadd_rn(v, z[o + 1 < M ? o + 1 : 0]), mu) : 0.f;
}

// the head-row gradients dz = {∂ℓ/∂v, ∂ℓ/∂a_1 .. ∂ℓ/∂a_n, 0 ...} of ∂ℓ/∂Q_a = g
template <int M>
__device__ __forceinline__ void backward(float g, int a, int n, float (&dz)[M]) {
    const float gn = __fdiv_rn(g, (float)n);
    dz[0] = g;
#pragma unroll
    for (int j = 1; j < M; ++j) dz[j] = j <= n ? __fsub_rn(j - 1 == a ? g : 0.f, gn) : 0.f;
}

}  // namespace duel
