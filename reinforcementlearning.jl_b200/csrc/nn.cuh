// nn.cuh — shared declarations of the learner kernels (nn.cu) for algo.cu.
//
// Network = Dense(in,H,act) -> Dense(H,H,act) -> head(s); parameters flat in
// Flux.destructure order, weights (out,in) column-major (W[o + out*i]):
//   W1 (H x in), b1 (H), W2 (H x H), b2 (H), then
//   single head:     W3 (n_out x H), b3 (n_out)                      [categorical logits / value / Q]
//   gaussian heads:  Wmu (1 x H), bmu (1), Wsig (1 x H), bsig (1)    [GaussianNetwork mu / sigma, 1-d action]
//   dueling heads:   Wv (1 x H), bv (1), Wa (n_out x H), ba (n_out)  [DuelingNetwork val / adv, combined by duel.cuh]
// (ActorCritic RLCore/src/utils/networks.jl:15-20, GaussianNetwork :44-116, DuelingNetwork :500-522.)
#pragma once
#include "common.cuh"
#include "optim.cuh"
#include "policy.cuh"   // AcHyper

constexpr int kInMax = 4;    // observation width <= 4 (CartPole 4, Pendulum 3, MountainCar 2)
constexpr int kOutMax = 4;   // head rows <= 4 (a dueling head has n_out + 1 rows: n_out <= 3)

enum { B200RL_ACT_RELU = 0, B200RL_ACT_TANH = 1 };

struct MlpDesc {
    int in, H, act, nout, heads2;  // heads2: two 1-wide heads (gaussian mu / sigma)
    int duel;                      // 1: dueling Q-network, head rows {val, adv_1 .. adv_nout}; nout stays the width of Q
    __host__ __device__ int rows() const { return nout + duel; }   // rows the head computes
    __host__ __device__ int64_t nparams() const { return (int64_t)H * in + H + (int64_t)H * H + H + (int64_t)rows() * H + rows(); }
};

// head row o (0 .. rows()-1), weight column j / bias, inside the flat parameter vector.  The one place that knows the head
// layouts: the FFMA kernels (nn.cu), the tensor-core forward (tc_fwd.cuh) and the tensor-core backward (nn_tc.cu) all use it.
// MAY_DUEL = false: a kernel that never sees a dueling network (the actor-critic ones) compiles without the dueling branch.
template <bool MAY_DUEL = true>
__host__ __device__ __forceinline__ int rows_of(const MlpDesc& d) { return MAY_DUEL ? d.rows() : d.nout; }
__host__ __device__ __forceinline__ int64_t head_base(const MlpDesc& d) { return (int64_t)d.H * d.in + d.H + (int64_t)d.H * d.H + d.H; }
template <bool MAY_DUEL = true>
__host__ __device__ __forceinline__ int64_t head_w(const MlpDesc& d, int o, int j) {
    if (MAY_DUEL && d.duel) return head_base(d) + (o == 0 ? (int64_t)j : (int64_t)(d.H + 1) + (o - 1) + (int64_t)d.nout * j);
    return head_base(d) + (d.heads2 ? (int64_t)o * (d.H + 1) + j : (int64_t)o + (int64_t)d.nout * j);
}
template <bool MAY_DUEL = true>
__host__ __device__ __forceinline__ int64_t head_b(const MlpDesc& d, int o) {
    if (MAY_DUEL && d.duel) return head_base(d) + (o == 0 ? (int64_t)d.H : (int64_t)(d.H + 1) + (int64_t)d.nout * d.H + (o - 1));
    return head_base(d) + (d.heads2 ? (int64_t)o * (d.H + 1) + d.H : (int64_t)d.nout * d.H + o);
}

// One minibatch of the on-policy update: sample j is flat index perm(j) into the rollout
// arrays (states (ns, total) column-major; actions / logp_old / adv / ret (total)).
struct AcBatch {
    const float* states; int ns;
    const void* actions;        // int32 (1-based) or float
    const float* logp_old; const float* adv; const float* ret;
    const int32_t* idx;         // explicit permutation slice, or null ->
    uint32_t perm_n, perm_key, perm_offset;  // ... Feistel permutation of [0, perm_n), slice start
    const uint32_t* perm_epoch; // device update counter (may be null): the key actually used is perm_key + *perm_epoch * 1000003
    const float4* rec;          // packed 32-byte rollout records (may be null): rec[2j] = state (zero padded), rec[2j+1] =
                                // {action bits, logp_old, advantage, return} — one DRAM sector per gathered sample instead of five
    int64_t B;                  // samples in this minibatch (local)
    float inv_B;                // 1 / (global minibatch size)  — gradients are sums * inv_B
    const float* norm2;         // device {mean, inv_std} for advantage normalisation
};

#ifdef __CUDACC__
__device__ __forceinline__ uint32_t ac_perm_key(const AcBatch& b) { return b.perm_key + (b.perm_epoch ? *b.perm_epoch * 1000003u : 0u); }
// the trunk activation, and its derivative from the activation's output h
__device__ __forceinline__ float act_f(int act, float z) { return act == B200RL_ACT_RELU ? fmaxf(z, 0.f) : tanhf(z); }
__device__ __forceinline__ float dact_f(int act, float h) { return act == B200RL_ACT_RELU ? (h > 0.f ? 1.f : 0.f) : 1.f - h * h; }
// sum of v over the NTHREADS threads of the CTA (warp shuffles, then the warp sums in order); valid on thread 0
template <int NTHREADS>
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x == 0)
        for (int k = 0; k < NTHREADS / 32; ++k) t += red[k];
    return t;
}
#endif
int nn_grid_ctas(b200rl_ctx* ctx, int H);  // persistent CTAs per role
int nn_dqn_max_partials(b200rl_ctx* ctx, int H);
// forward (rollout inference).  obs (in, N) column-major.  Any output may be null.
int nn_policy_act(b200rl_ctx* ctx, const MlpDesc& actor, const MlpDesc& critic, const float* params, const AcHyper& hp,
                  const float* obs, int64_t N, unsigned long long* rng, void* action_out, float* logp_out, float* value_out,
                  float* head_out /* (nout, N) raw head outputs, for tests */, float* state_copy /* (in, N) */);
int nn_mlp_forward(b200rl_ctx* ctx, const MlpDesc& net, const float* params, const float* obs, int64_t N, float* out /* (nout, N) */);
// loss + backward: writes per-CTA partial gradients/losses; nn_reduce sums them in CTA order.
// Returns the number of gradient partials written (> 0; loss rows = 2x that) or a negative status.
int nn_ac_loss_grad(b200rl_ctx* ctx, const MlpDesc& actor, const MlpDesc& critic, const float* params, const AcHyper& hp,
                    const AcBatch& b, float* partial /* [ctas][np] */, float* loss_partial /* [2*ctas][4] */);
int nn_reduce_partials(b200rl_ctx* ctx, const float* partial, int n_partials, int64_t np, float* grad, const float* loss_partial,
                       int n_loss_partials, float* loss_out4);

// ---- optimiser step: [reduce the per-CTA partials -> peer exchange ->] global norm -> clip_by_global_norm! -> Adam (optim.cuh) ----
// The operands of one step on a network's flat parameter vector.  The single-launch steps (K8, K7's tail) meet at self-resetting
// grid barriers on `counters` and keep their sequence numbers and tick in device memory, so they can be captured and replayed.
struct OptStep {
    float* params; float* grad; float* m; float* v; float* beta_t /* device [2]: {beta1^t, beta2^t} */;
    float* loss_out4; float* stats_row; float* gnorm_out;     // each may be null; stats_row receives {4 loss sums, grad norm}
    double* cta_sumsq;            // >= grid doubles (<= 256)
    unsigned int* counters;       // 4 zero-initialised uints (grid barriers: K8 uses 2, K7 3)
    unsigned int* tick;           // may be null: device update counter incremented once by the step (keys the permutation)
    unsigned int* seq_ptr;        // gradient-exchange sequence number (sharded run; set by the launcher)
    float max_norm, lr, b1, b2, eps;
    P2PTable tab;                 // nranks <= 1: single GPU (set by the launcher)
};
// clip_by_global_norm! + Adam on st.grad (single CTA, deterministic); writes st.gnorm_out
int nn_clip_adam(b200rl_ctx* ctx, int64_t np, const OptStep& st);
// reduce + [peer exchange +] clip + Adam in one launch, when its ceil(np / 256) CTAs are all co-resident (B200RL_ERR_UNSUPPORTED
// otherwise); the peer exchange runs when one is attached
int nn_reduce_clip_adam(b200rl_ctx* ctx, const float* partial, int n_partials, int64_t np, const float* loss_partial, int n_loss, const OptStep& st);
// K7 + optimiser step in one launch.  Returns the number of gradient partials (> 0) like nn_ac_loss_grad, or
// B200RL_ERR_UNSUPPORTED *without side effects* when the configuration is outside the fused path (the caller then runs
// nn_ac_loss_grad + nn_reduce_clip_adam).
int nn_ac_loss_grad_step(b200rl_ctx* ctx, const MlpDesc& actor, const MlpDesc& critic, const AcHyper& hp, const AcBatch& b, float* partial,
                         float* loss_partial, const OptStep& st);
int nn_target_sync(b200rl_ctx* ctx, float* target, const float* model, int64_t np, float rho);
// target sync every `freq` optimiser steps, counted on the device: *upd_dev += 1, sync when it is a multiple of freq
int nn_target_sync_counted(b200rl_ctx* ctx, float* target, const float* model, int64_t np, float rho, unsigned long long* upd_dev, int freq);
// DQN: TD loss + backward on a gathered batch (device arrays s (in,B), a, r, t, s2, w).  disc (may be null): per-sample discount
// (n-step γ^m) in place of the scalar gamma
int nn_dqn_loss_grad(b200rl_ctx* ctx, const MlpDesc& q, const float* params, const float* target, const float* s, const int32_t* a,
                     const float* r, const uint8_t* t, const float* s2, const float* w, int64_t B, float inv_B, float gamma, int huber,
                     int double_dqn, float* partial, float* loss_partial, float* td_out, const float* disc);
int nn_q_act(b200rl_ctx* ctx, const MlpDesc& q, const float* params, const float* obs, int64_t N, unsigned long long* rng, float epsilon,
             int32_t* action_out, float* q_out);
// step_dev (may be null): explorer step read from device memory instead of ex.step.  On a sharded ctx column i is global column
// rank · N + i (explore::column_step)
int nn_q_explore(b200rl_ctx* ctx, const MlpDesc& q, const float* params, const float* obs, int64_t N, unsigned long long* rng,
                 const b200rl_explorer& ex, int32_t* action_out, float* q_out, const long long* step_dev = nullptr);

// tensor-core (wgmma) variants, nn_tc.cu.  Used for H = 64 unless disabled (B200RL_TC=0 or b200rl_set_tensor_cores(0)).
bool nn_tc_enabled();
bool nn_tc_supported(const MlpDesc& d);
int nn_tc_forward(b200rl_ctx* ctx, int grid, const MlpDesc& actor, const MlpDesc& critic, const float* params, const AcHyper& hp, int mode,
                  const float* obs, int64_t N, unsigned long long* rng, void* action_out, float* logp_out, float* value_out, float* head_out,
                  float* state_copy);
// fused rollout (fwd_tc.cu): nsteps x {policy inference, env step, transition push} in one launch; B200RL_ERR_UNSUPPORTED =
// outside the fused envelope, step through nn_policy_act + b200rl_env_step instead
struct b200rl_env;
int nn_tc_rollout(b200rl_ctx* ctx, b200rl_env* env, const MlpDesc& actor, const MlpDesc& critic, const float* params, const AcHyper& hp,
                  unsigned long long* policy_rng, int t0, int nsteps, int T, int final_bootstrap, float* states, void* actions, float* logp,
                  float* values, float* rewards, uint8_t* terminals);
// fused evaluation window (fwd_tc.cu): nsteps x {actor -> greedy (mode 0) | sampled (mode 1) action | Q-network -> explorer column
// (mode 2; ex null: GreedyExplorer), env step, episode records}; B200RL_ERR_UNSUPPORTED = outside the fused envelope, step through
// staged launches instead
int nn_tc_evaluate(b200rl_ctx* ctx, b200rl_env* env, const MlpDesc& actor, const float* params, const AcHyper& hp, int mode, int nsteps,
                   int K, unsigned long long* policy_rng, float* returns, int32_t* lengths, int32_t* counts, const b200rl_explorer* ex = nullptr);
// the same window as a stretch of run(policy, env, stop) (b200rl_eval_run_episodes): from the env's current state, no records; the
// finished episodes go to the env's episode log when one is attached, and step_counts (may be null) gets, per window step j, the
// lanes terminal after step j + 1 added.  B200RL_ERR_UNSUPPORTED = outside the fused envelope
int nn_tc_eval_run(b200rl_ctx* ctx, b200rl_env* env, const MlpDesc& actor, const float* params, const AcHyper& hp, int mode, int nsteps,
                   unsigned long long* policy_rng, const b200rl_explorer* ex, unsigned long long* step_counts);
// fused DQN collect window (fwd_tc.cu): nsteps x {Q -> explorer column | findmax, env step, ring push} for H = 64; the touched
// sum-tree leaves of each lane go to keys / vals (stride, N) for one tree rebuild.  B200RL_ERR_UNSUPPORTED = outside the envelope
struct Ring;
int nn_tc_replay_collect(b200rl_ctx* ctx, b200rl_env* env, const MlpDesc& q, const float* params, const b200rl_explorer* ex,
                         const long long* step_dev, unsigned long long* xrng, const Ring& ring, float default_priority, int prioritized,
                         int nsteps, int64_t* keys, float* vals, int stride);
bool nn_tc_bwd_supported(const MlpDesc& actor, const MlpDesc& critic);
int nn_tc_partial_rows(int grid, const MlpDesc& actor, const AcHyper& hp, int64_t B);   // gradient-partial rows the tensor-core K7 writes with `grid` CTAs
// whether K7 with `grid` CTAs can run the optimiser step on np parameters in its tail (the launch geometry only; nn_ac_loss_grad_step
// decides the rest)
bool nn_tc_step_fits(b200rl_ctx* ctx, int grid, const MlpDesc& actor, const AcHyper& hp, int64_t B, int64_t np);
int nn_tc_ac_loss_grad(b200rl_ctx* ctx, int grid, const MlpDesc& actor, const MlpDesc& critic, const float* params, const AcHyper& hp,
                       const AcBatch& b, float* partial, float* loss_partial, int64_t np, const OptStep* step /* null: loss + backward only */);
