// stop_episodes.cuh — StopAfterNEpisodes on the fused agent loops (b200rl_onpolicy_run_episodes, b200rl_replay_run_episodes).
//
// The stage loop checks StopAfterNEpisodes after every step: cur += count_t (lanes whose is_terminated is true after step t, a
// MaxTimeoutEnv cut included) and it stops once cur >= k.  The fused loops run a stretch of s steps ahead, reduce the terminal
// flags the stretch wrote to the per-step counts count_1 .. count_s, and find the step the stage loop would have stopped after:
//   s* = the first t in 1 .. s with  count_1 + ... + count_t >= k - cur,   0 when the stretch does not reach the budget.
// A budget already spent (k - cur <= 0) stops after the first step, as the stage loop does (it checks only after a step).
//
// stop::crossing is plain C++ once the CUDA qualifiers are defined away; the CPU suite compiles it for the host.  The kernels
// below it (count, crossing, shadow copy) are device code only.
#pragma once
#include <cstdint>

#include "ring.cuh"

struct StopCrossing {
    int64_t step;       // s* (1-based), 0 = no crossing inside the stretch
    int64_t episodes;   // count_1 + ... + count_{s*}, or the sum over the whole stretch when s* = 0
};

namespace stop {

__host__ __device__ inline StopCrossing crossing(const unsigned long long* counts, int64_t s, int64_t remaining) {
    int64_t sum = 0;
    for (int64_t t = 0; t < s; ++t) {
        sum += (int64_t)counts[t];
        if (sum >= remaining) return StopCrossing{t + 1, sum};
    }
    return StopCrossing{0, sum};
}

// The stretches of b200rl_eval_run_episodes (an evaluation policy under run(), one fused evaluation launch per stretch).
// kEvalStretchMax bounds every stretch: the counts buffer holds kEvalStretchMax + 2 entries, and one launch stays short (about
// 10 ms at 65 536 CartPole envs).  With an episode budget a stretch that cannot reach it (N · s < remaining) runs unmarked for as
// long as possible; once fewer than N · kEvalStretchMarked episodes remain, stretches of kEvalStretchMarked steps are marked, so a
// rollback re-runs at most that many steps.
constexpr int64_t kEvalStretchMax = 1024;
constexpr int64_t kEvalStretchMarked = 64;
__host__ __device__ inline int64_t eval_stretch(int64_t left, int64_t remaining, int64_t N, bool counting) {
    const int64_t s = left < kEvalStretchMax ? left : kEvalStretchMax;
    if (!counting) return s;
    const int64_t unmarked = remaining > 0 ? (remaining - 1) / N : 0;   // the longest stretch with N · s < remaining
    if (unmarked >= kEvalStretchMarked) return s < unmarked ? s : unmarked;
    return s < kEvalStretchMarked ? s : kEvalStretchMarked;
}

}  // namespace stop

#ifdef __CUDACC__
namespace stop {

constexpr int kCountBlock = 256;

// per-step terminal counts of the fused rollout's columns t0 .. t0 + s - 1 of terminals (N, T) u8: counts[j] += lanes terminal
// after step j + 1 of the stretch.  grid (ceil(N / kCountBlock), min(s, 65535)): blockIdx.y strides over the s columns.
__global__ void __launch_bounds__(kCountBlock) count_columns_kernel(const uint8_t* __restrict__ terminals, int64_t N, int t0, int s,
                                                                     unsigned long long* __restrict__ counts) {
    const int64_t i = (int64_t)blockIdx.x * kCountBlock + threadIdx.x;
    for (int j = blockIdx.y; j < s; j += gridDim.y) {
        const int term = i < N ? (terminals[(size_t)N * (t0 + j) + i] & 1) : 0;
        const int n = __syncthreads_count(term);
        if (threadIdx.x == 0 && n) atomicAdd(counts + j, (unsigned long long)n);
    }
}

// per-step terminal counts of the last s steps pushed into the replay ring.  Every step of an auto-reset env stores one
// transition per lane (flag bit kRingSampleable) in the slot of the state it was taken in; state frames without a transition
// (the newest one, the terminal observation before an episode-start frame) have the bit clear.  So walking a lane back from its
// newest frame, the k-th transition met is the one of step s + 1 - k; its terminal bit is the env's is_terminated after that
// step.  Needs 2 s + 1 <= cap + 1 frames (the longest a stretch of s steps can write), so that none of them is overwritten.
// counts: s entries; dynamic shared memory: s ints.
__global__ void __launch_bounds__(kCountBlock) count_ring_kernel(Ring r, int s, unsigned long long* __restrict__ counts) {
    extern __shared__ int hist[];
    for (int j = threadIdx.x; j < s; j += kCountBlock) hist[j] = 0;
    __syncthreads();
    const int64_t e = (int64_t)blockIdx.x * kCountBlock + threadIdx.x;
    if (e < r.lanes) {
        const int64_t F = r.frames();
        int64_t q = (r.head[e] + F - 1) % F;   // the newest state frame
        for (int j = s - 1, walked = 0; j >= 0 && walked < F - 1; ++walked) {
            q = q == 0 ? F - 1 : q - 1;
            const uint8_t f = r.flag[q * r.lanes + e];
            if (f & kRingSampleable) {
                if (f & kRingTerminal) atomicAdd(hist + j, 1);
                --j;
            }
        }
    }
    __syncthreads();
    for (int j = threadIdx.x; j < s; j += kCountBlock)
        if (hist[j]) atomicAdd(counts + j, (unsigned long long)hist[j]);
}

// the first crossing of `remaining` by the counts of a stretch of s steps -> out {s*, episodes}
__global__ void crossing_kernel(const unsigned long long* __restrict__ counts, int64_t s, int64_t remaining, long long* __restrict__ out) {
    const StopCrossing c = crossing(counts, s, remaining);
    out[0] = (long long)c.step;
    out[1] = (long long)c.episodes;
}

// Copies between the state a stretch changes and its shadow: region k is bytes[k] bytes at state[k] <-> shadow[k].  grid (x, n).
constexpr int kMaxRegions = 32;
struct Regions {
    int n;
    char* state[kMaxRegions];
    char* shadow[kMaxRegions];
    size_t bytes[kMaxRegions];
};
__global__ void __launch_bounds__(256) copy_regions_kernel(Regions g, int to_shadow) {
    const int k = blockIdx.y;
    char* dst = to_shadow ? g.shadow[k] : g.state[k];
    const char* src = to_shadow ? g.state[k] : g.shadow[k];
    const size_t nb = g.bytes[k];
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if ((((uintptr_t)dst | (uintptr_t)src | nb) & 15) == 0) {
        uint4* d = reinterpret_cast<uint4*>(dst);
        const uint4* s = reinterpret_cast<const uint4*>(src);
        for (size_t i = i0; i < nb / 16; i += stride) d[i] = s[i];
    } else if ((((uintptr_t)dst | (uintptr_t)src | nb) & 3) == 0) {
        uint32_t* d = reinterpret_cast<uint32_t*>(dst);
        const uint32_t* s = reinterpret_cast<const uint32_t*>(src);
        for (size_t i = i0; i < nb / 4; i += stride) d[i] = s[i];
    } else {
        for (size_t i = i0; i < nb; i += stride) dst[i] = src[i];
    }
}

}  // namespace stop
#endif
