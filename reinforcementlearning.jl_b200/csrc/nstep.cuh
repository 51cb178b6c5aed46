// nstep.cuh — the n-step window of one sampled replay entry: NStepBatchSampler(n, γ) (ReinforcementLearningTrajectories 0.4,
// external and unpinned; DESIGN.md §3).  sample_gather_kernel<PRIO, true> (traj.cu) calls it once per batch slot after the key
// has been drawn, so which entries are drawn does not depend on n.
//
// Entry q = the sampled key (slot p, lane e).  The window takes entries q, q+1, ... of the same lane (slots mod cap + 1) and ends
// at the first of: n entries taken; the entry just taken is terminal; the next entry is not sampleable (flag bit 1 clear: the
// lane's newest state frame, the entry straddling a forced reset, or a destroyed slot).  m = its length, 1 <= m <= n.
//   G         = r[q+m-1], then G = r[q+j] + γ·G for j = m-2 .. 0   (Float32, every operation rounded, no FMA: discount_rewards' order)
//   terminal  = terminal bit of entry q+m-1
//   next slot = slot of state frame q+m
//   discount  = γ^m as the left-to-right Float32 product of m factors
// The walk reads flags forward and rewards backward, so it keeps no per-entry array.  Plain C++ once the CUDA qualifiers are
// defined away; the CPU suite compiles it for the host with its own __fadd_rn / __fmul_rn.
#pragma once
#include <cstdint>

#include "ring.cuh"

constexpr int kNStepMax = 32;

struct NStepWindow {
    float G, discount;
    int64_t next_slot;
    int m;
    uint8_t terminal;
};

namespace nstep {

__device__ __forceinline__ NStepWindow window(const Ring& r, int64_t key, int n, float gamma) {
    const int64_t F = r.frames();
    const int64_t e = key % r.lanes;
    int64_t s = key / r.lanes;
    uint8_t f = r.flag[key];
    int m = 1;
    while (m < n && !(f & kRingTerminal)) {
        const int64_t s1 = s + 1 == F ? 0 : s + 1;
        const uint8_t f1 = r.flag[s1 * r.lanes + e];
        if (!(f1 & kRingSampleable)) break;
        s = s1; f = f1; ++m;
    }
    NStepWindow w;
    w.m = m;
    w.terminal = f & kRingTerminal;
    w.next_slot = s + 1 == F ? 0 : s + 1;
    float G = r.reward[s * r.lanes + e];
    float d = gamma;
    for (int j = m - 2; j >= 0; --j) {
        s = s == 0 ? F - 1 : s - 1;
        G = __fadd_rn(r.reward[s * r.lanes + e], __fmul_rn(gamma, G));
        d = __fmul_rn(d, gamma);
    }
    w.G = G;
    w.discount = d;
    return w;
}

}  // namespace nstep
