// optim.cuh — the optimiser step of every learner, once for the three kernels that run it: clip_adam_kernel and K8
// reduce_clip_adam_kernel (nn.cu), and the tail of the tensor-core K7 (nn_tc.cu).
//   clip_scale    clip_by_global_norm! (basic.jl:19-29) as a factor on the gradient
//   adam_update   one element of Optimisers.jl Adam (SURVEY Appendix B); beta_advance moves beta^t on after the step
// Plain C++ once the CUDA qualifiers are defined away, so the CPU suite compiles this part for the host (tests/hostdev/cuda_runtime.h,
// g++ -ffp-contract=off) and checks it bit for bit against the oracle.  Contraction follows the including translation unit (nn.cu and
// nn_tc.cu contract), so each kernel computes what its own copy of this code computed.
// Below __CUDACC__: the grid barrier, the step's closing epilogue and the stats publication of the single-launch steps (K8, K7's tail).
#pragma once
#include <cmath>

namespace optim {

// the factor clip_by_global_norm! applies for global norm gn.  max_norm = 0 disables clipping (the DQN default), where the reference's
// rule would scale the gradient to zero
__host__ __device__ __forceinline__ float clip_scale(float gn, float max_norm) {
    return max_norm > 0.f && max_norm <= gn ? max_norm / fmaxf(max_norm, gn) : 1.0f;
}

struct AdamOut { float m, v, p; };
// Adam on one element: gradient g (already clipped), moments m, v and parameter p before the step, beta^t = {bt1, bt2} of this step
__host__ __device__ __forceinline__ AdamOut adam_update(float g, float m, float v, float p, float lr, float b1, float b2, float eps, float bt1,
                                                       float bt2) {
    const float mk = b1 * m + (1.0f - b1) * g;
    const float vk = b2 * v + (1.0f - b2) * (g * g);
    return {mk, vk, p - mk / (1.0f - bt1) / (sqrtf(vk / (1.0f - bt2)) + eps) * lr};
}
// beta^t after the step, once every element has used {bt1, bt2}
__host__ __device__ __forceinline__ void beta_advance(float* beta_t, float bt1, float bt2, float b1, float b2) {
    beta_t[0] = bt1 * b1;
    beta_t[1] = bt2 * b2;
}

#ifdef __CUDACC__
// Device-wide barrier of a single-launch step (all CTAs co-resident), called by one thread per CTA: everything the CTA wrote before it
// is visible to every CTA after it (fence cumulativity, as in cooperative groups).  A CTA that never arrives traps after 2^26 polls
// instead of hanging the GPU.
__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int G) {
    __threadfence();
    atomicAdd(counter, 1u);
    unsigned int spins = 0;
    while (*reinterpret_cast<volatile unsigned int*>(counter) < G)
        if (++spins > (1u << 26)) __trap();
    __threadfence();
}

// Closes a single-launch step, called by one thread per CTA once every thread of its CTA has read beta^t and the exchange sequence
// number: the last CTA through advances beta^t, re-arms the NC barrier counters (counters[NC - 1] is the one it arrives at), stores
// the sequence number `seq` of a peer exchange (xchg) and bumps the update tick (may be null).  Nothing depends on host-side launch
// counts, so the launch can be captured in a CUDA graph and replayed.  Step: OptStep (nn.cuh).
template <int NC, class Step>
__device__ __forceinline__ void close_step(const Step& st, float bt1, float bt2, bool xchg, unsigned seq) {
    __threadfence();
    if (atomicAdd(st.counters + NC - 1, 1u) + 1u == gridDim.x) {
        beta_advance(st.beta_t, bt1, bt2, st.b1, st.b2);
#pragma unroll
        for (int c = 0; c < NC; ++c) st.counters[c] = 0u;
        if (xchg) *st.seq_ptr = seq;
        if (st.tick) *st.tick += 1u;
    }
}

// the step's stats: loss sum i (0..3) to loss_out4[i] and stats_row[i]; the gradient norm to gnorm_out and stats_row[4] (each may be null)
template <class Step>
__device__ __forceinline__ void publish_loss(const Step& st, int i, float lsum) {
    if (st.loss_out4) st.loss_out4[i] = lsum;
    if (st.stats_row) st.stats_row[i] = lsum;
}
template <class Step>
__device__ __forceinline__ void publish_gnorm(const Step& st, float gn) {
    if (st.gnorm_out) *st.gnorm_out = gn;
    if (st.stats_row) st.stats_row[4] = gn;
}
#endif

}  // namespace optim
