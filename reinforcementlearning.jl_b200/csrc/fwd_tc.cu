// fwd_tc.cu — K6 on tensor cores and the fused rollout kernel (K6 + K1 + K3 over a whole rollout in ONE launch).
//
//   forward_tc_kernel  : policy inference for one env batch (plan!): actor -> action + log-prob, critic -> value.
//   rollout_tc_kernel  : n_steps x { obs -> actor -> sample action -> critic -> value -> env step (+ fused auto-reset) ->
//                        write the transition into column t of the rollout tensors }.  A CTA owns up to two tiles of 128
//                        envs for the whole launch; their env state and both RNG streams stay in shared memory, the weights of
//                        both networks too.  Replaces 2 launches per env step (agent_base.jl:45-66 stage loop, run.jl:52-68).
//   evaluate_tc_kernel : n_steps x { obs -> actor -> greedy | sampled action (or Q -> explorer action) -> env step (+ fused
//                        auto-reset) -> per-env episode records }: one network, no rollout tensors (b200rl_evaluate,
//                        b200rl_evaluate_explore).
//   replay_collect_tc_kernel : n_steps x { obs -> Q -> explorer action -> env step (+ fused auto-reset) -> replay ring push }.
//
// The kernels share one tile forward (tile_forward), one resident env slot with its load / write-back (EnvSlot) and the act! step
// of env_device.cuh, and are compiled with the env flags (-fmad=false): stepping through plan!/act! one launch at a time or
// through a fused kernel gives bit-identical results.
#include "common.cuh"
#include "duel.cuh"
#include "env_device.cuh"
#include "explore.cuh"
#include "greedy.cuh"
#include "internal.h"
#include "policy.cuh"
#include "ring.cuh"
#include "tc_fwd.cuh"

using namespace tcfwd;
using namespace envdev;

namespace {

struct SmemFwd {
    alignas(128) uint8_t T[TILE_BYTES];   // A operand / accumulator image of the tile (tc_fwd.cuh)
    NetSm net;
    float X[kInMax * TM];                 // [i][s]
    float Zp[2 * kOutMax * TM];           // head partials [half][o][s]
};

// One tile of TM samples through one network: the observations in X ([i][s], published by a barrier before the call) -> layer 1 ->
// the GEMM of both warpgroups -> the head partial sums of both 32-feature halves in Zp ([half][o][s]).  Called by all NT threads;
// ends with a barrier, after which Zp may be read (tile_heads) and the next tile's X writes are ordered behind this tile's reads.
// UNROLL: as layer1_to_smem / head_partials.
template <int ACT, int UNROLL = (ACT == B200RL_ACT_RELU ? 2 : 1)>
__device__ __forceinline__ void tile_forward(const NetSm& net, int act_rt, int c, int s, uint8_t* T, const float* X, float* Zp) {
    {
        float x[kInMax];
#pragma unroll
        for (int k = 0; k < kInMax; ++k) x[k] = X[k * TM + s];
        layer1_to_smem<ACT, UNROLL>(net, act_rt, x, c, s, T);
    }
    wg::fence_proxy_async();
    __syncthreads();
    gemm_block(T + c * BLK, net, c);   // warpgroup c: samples 64c .. 64c+63
    __syncthreads();
    {
        float zp[kOutMax];
        head_partials<ACT, UNROLL>(net, act_rt, c, s, T, zp);
#pragma unroll
        for (int o = 0; o < kOutMax; ++o) Zp[(c * kOutMax + o) * TM + s] = zp[o];
    }
    __syncthreads();
}
// head outputs of sample s after tile_forward
__device__ __forceinline__ void tile_heads(const NetSm& net, const float* Zp, int s, float (&z)[kOutMax]) {
#pragma unroll
    for (int o = 0; o < kOutMax; ++o) z[o] = net.b3[o] + Zp[o * TM + s] + Zp[(kOutMax + o) * TM + s];
}

// mode 0: actor-critic rollout step (CTA role = blockIdx & 1), mode 1: plain forward of `actor` -> head_out
template <int ACT>
__global__ void __launch_bounds__(NT, 2)
forward_tc_kernel(MlpDesc actor, MlpDesc critic, const float* __restrict__ params, AcHyper hp, int mode, const float* __restrict__ obs,
                  int64_t N, unsigned long long* __restrict__ rng, void* __restrict__ action_out, float* __restrict__ logp_out,
                  float* __restrict__ value_out, float* __restrict__ head_out, float* __restrict__ state_copy) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    SmemFwd& sm = *reinterpret_cast<SmemFwd*>(smem_raw);
    const int nroles = mode == 0 ? 2 : 1;
    const int role = mode == 0 ? (blockIdx.x & 1) : 0;
    const int cta = blockIdx.x / nroles, nctas = gridDim.x / nroles;
    const MlpDesc d = role ? critic : actor;
    const int64_t poff = role ? actor.nparams() : 0;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q = warp & 3, c = warp >> 2;
    const int s = 32 * q + lane;
    load_net(sm.net, d, params + poff, (ACT >= 0 ? ACT : d.act) == B200RL_ACT_RELU && ACT >= 0 ? kScale : 1.0f);
    wg::fence_proxy_async();
    __syncthreads();
    const int64_t ntiles = (N + TM - 1) / TM;
    for (int64_t tile = cta; tile < ntiles; tile += nctas) {
        if (tid < TM) {
            int64_t i = tile * TM + tid;
            float x[kInMax] = {0.f, 0.f, 0.f, 0.f};
            if (i < N) {
                if (d.in == 4) {
                    float4 v4 = reinterpret_cast<const float4*>(obs)[i];
                    x[0] = v4.x; x[1] = v4.y; x[2] = v4.z; x[3] = v4.w;
                    if (state_copy && role == 0) reinterpret_cast<float4*>(state_copy)[i] = v4;
                } else {
#pragma unroll
                    for (int k = 0; k < kInMax; ++k) {
                        if (k < d.in) {
                            x[k] = obs[(int64_t)d.in * i + k];
                            if (state_copy && role == 0) state_copy[(int64_t)d.in * i + k] = x[k];
                        }
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < kInMax; ++k) sm.X[k * TM + tid] = x[k];
        }
        __syncthreads();
        tile_forward<ACT>(sm.net, d.act, c, s, sm.T, sm.X, sm.Zp);   // (its last barrier: the head reads are done before the next
        if (tid < TM) {                                              //  tile's layer 1 overwrites the image)
            int64_t i = tile * TM + tid;
            if (i < N) {
                float z[kOutMax];
                tile_heads(sm.net, sm.Zp, tid, z);
                if (mode == 1 && d.duel) duel::combine(z, d.nout);   // dueling Q-network: the combined Q, not the head rows
                if (head_out && (mode == 1 || role == 0))
                    for (int o = 0; o < d.nout; ++o) head_out[(int64_t)d.nout * i + o] = z[o];
                if (mode == 0 && role == 1) {
                    if (value_out) value_out[i] = z[0];
                } else if (mode == 0) {
                    unsigned long long st[4];
                    explore::xo_load(rng, i, st);
                    float lp;
                    uint32_t a = policy::sample_head(actor.heads2, actor.nout, hp, z, st, lp);
                    if (action_out) reinterpret_cast<uint32_t*>(action_out)[i] = a;
                    if (logp_out) logp_out[i] = lp;
                    explore::xo_store(rng, i, st);
                }
            }
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// resident env slots of the fused kernels: a CTA keeps up to kSlots tiles of 128 envs (tiles base + k * nctas) in shared memory,
// one entry per env, owned by thread s = the env's sample in the tile
constexpr int kSlots = 2;

// a 4-word stream of env s in a slot's transposed [word][env] layout
__device__ __forceinline__ void get_stream(const unsigned long long* w, int s, unsigned long long (&x)[4]) {
#pragma unroll
    for (int k = 0; k < 4; ++k) x[k] = w[k * TM + s];
}
__device__ __forceinline__ void put_stream(unsigned long long* w, int s, const unsigned long long (&x)[4]) {
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k * TM + s] = x[k];
}

template <class E> struct EnvSlot {   // the env part of a slot; each kernel's slot type adds its own fields
    using Env = E;
    using act_bits = typename std::conditional<sizeof(typename Env::act_t) == 8, unsigned long long, uint32_t>::type;
    typename Env::S st[TM];
    int t[TM];
    int flags[TM];
    float ep_ret[TM];
    typename Env::real last_rew[TM];
    act_bits last_act[TM];                 // env.action after the last act! (a reset may have redrawn it), raw bits
    unsigned long long erng[4 * TM];       // env stream
};

__device__ __forceinline__ int group_slots(int64_t base, int nctas, int64_t ntiles) {   // resident tiles of the group at `base`
    int n = 0;
    for (int k = 0; k < kSlots; ++k)
        if (base + (int64_t)k * nctas < ntiles) n = k + 1;
    return n;
}
// Owner thread s: loads the env part of env i of each resident tile into its slot; more(slot, i) loads the kernel's own fields.
template <class Slot, class More>
__device__ __forceinline__ void load_group(Slot* slot, int nslots, int64_t base, int nctas, const EnvArrays& ea, int64_t N, int s, More&& more) {
    for (int k = 0; k < nslots; ++k) {
        const int64_t i = (base + (int64_t)k * nctas) * TM + s;
        if (i < N) {
            Slot& sl = slot[k];
            sl.st[s] = Slot::Env::load(ea.state, i);
            sl.t[s] = ea.t[i];
            sl.flags[s] = ea.flags[i];
            sl.ep_ret[s] = ea.ep_ret[i];
            unsigned long long e[4];
            explore::xo_load(ea.rng, i, e);
            put_stream(sl.erng, s, e);
            more(sl, i);
        }
    }
}
// ... and writes it back: reward and action are the last step's, so only when the window stepped (`stepped`).
template <class Slot, class More>
__device__ __forceinline__ void store_group(const Slot* slot, int nslots, int64_t base, int nctas, const EnvArrays& ea, int64_t N, int s,
                                            bool stepped, More&& more) {
    using Env = typename Slot::Env;
    for (int k = 0; k < nslots; ++k) {
        const int64_t i = (base + (int64_t)k * nctas) * TM + s;
        if (i < N) {
            const Slot& sl = slot[k];
            Env::store(ea.state, i, sl.st[s]);
            if (!Env::kObsIsState) Env::write_obs(ea.obs, i, N, sl.st[s]);
            store_obs_f32<Env>(ea, i, N, sl.st[s]);
            ea.t[i] = sl.t[s];
            ea.flags[i] = (uint8_t)sl.flags[s];
            ea.ep_ret[i] = sl.ep_ret[s];
            unsigned long long e[4];
            get_stream(sl.erng, s, e);
            explore::xo_store(ea.rng, i, e);
            if (stepped) {
                reinterpret_cast<typename Env::real*>(ea.reward)[i] = sl.last_rew[s];
                reinterpret_cast<typename Slot::act_bits*>(ea.action)[i] = sl.last_act[s];
            }
            more(sl, i);
        }
    }
}

// the action the env receives for the head's raw action bits: the 1-based index, or the continuous action clamped to the action space
// (a Float64 env: Float64 of the clamped Float32 action; the bounds are exact in Float32, so this is the clamp in Float64)
template <class Env> __device__ __forceinline__ typename Env::act_t env_action(uint32_t a_bits) {
    using act_t = typename Env::act_t;
    if (std::is_floating_point<act_t>::value) return (act_t)fminf(fmaxf(__uint_as_float(a_bits), -Env::kActionBound), Env::kActionBound);
    return (act_t)(int32_t)a_bits;
}
// act!(env, a) of owner thread s's env in its slot: the act! step of env_step_kernel<Env, false, true>, the fused auto-reset drawing
// from the slot's env stream, a finished episode added to the thread's tally (and to env i's episode log when the caller passes
// one).  The reward it returns is Float32(reward), what a rollout or the replay ring stores; the slot keeps the env's own.
template <class Env, bool LOG = false>
__device__ __forceinline__ ActStep<float> slot_act(EnvSlot<Env>& sl, int s, const typename Env::P& p, int max_timeout, typename Env::act_t act,
                                                   int& fin_cnt, float& fin_ret, int& fin_len, EpisodeLog log = EpisodeLog{}, int64_t i = 0) {
    typename Env::S st = sl.st[s];
    int t = sl.t[s], f = sl.flags[s];
    float ret = sl.ep_ret[s];
    const ActStep<typename Env::real> r = act_step<Env, true, LOG>(p, max_timeout, st, t, f, ret, act, fin_cnt, fin_ret, fin_len, [&](auto&& reset) {
        unsigned long long w[4];
        get_stream(sl.erng, s, w);
        Xo e{w[0], w[1], w[2], w[3]};
        reset(e);
        const unsigned long long o[4] = {e.s0, e.s1, e.s2, e.s3};
        put_stream(sl.erng, s, o);
    }, log, i);
    sl.st[s] = st; sl.t[s] = t; sl.flags[s] = f; sl.ep_ret[s] = ret;
    sl.last_rew[s] = r.rew;
    typename EnvSlot<Env>::act_bits bits;
    memcpy(&bits, &act, sizeof bits);
    sl.last_act[s] = bits;
    return ActStep<float>{(float)r.rew, r.done, r.ret, r.len};
}

// b200rl_explorer without its trailing beta, which the kernels that plan with it take separately: the parameters the ϵ-greedy
// instantiations read keep the offsets they had before the explorer struct grew
struct QExplorer {
    double eps_stable, eps_init;
    int64_t warmup_steps, decay_steps, step;
    int32_t kind, is_break_tie;
};
// plan!(QBasedPolicy) of owner thread s's column on its Q-values z, 1-based: GreedyExplorer (greedy: the first maximum under `>`,
// q_act_kernel with epsilon = 0, no draw) or the BatchExplorer column of explore.cuh at explorer step `step` on the column's stream,
// kept in the slot's transposed array w.  XEXT: the explorer kinds 2-4 (speedy, weighted / Gumbel softmax; explore::select<true>),
// which read beta; without it only the ϵ-greedy kinds 0 / 1 are compiled.  The fused collect and the fused evaluation plan with it.
template <bool XEXT>
__device__ __forceinline__ int plan_q_column(bool greedy, const QExplorer& ex, double beta, long long step, const float* z, int na,
                                             unsigned long long* w, int s) {
    if (greedy) {
        int best = 0;
        for (int o = 1; o < na; ++o) if (z[o] > z[best]) best = o;
        return best + 1;
    }
    unsigned long long xr[4];
    get_stream(w, s, xr);
    int a1;
    if constexpr (XEXT) {
        const b200rl_explorer e{ex.eps_stable, ex.eps_init, ex.warmup_steps, ex.decay_steps, ex.step, ex.kind, ex.is_break_tie, beta};
        a1 = explore::select<true>(e, step, z, na, xr);
    } else {
        a1 = explore::select<false>(ex, step, z, na, xr);
    }
    put_stream(w, s, xr);
    return a1;
}

// ---------------------------------------------------------------------------------------------------------------------
// fused rollout
template <class Env> struct RollSlot : EnvSlot<Env> {
    unsigned long long prng[4 * TM];       // policy stream
};
template <class Env> struct SmemRoll {
    alignas(128) uint8_t T[TILE_BYTES];    // A operand / accumulator image of the tile being evaluated (tc_fwd.cuh)
    NetSm net[2];                          // actor, critic
    float X[kInMax * TM];
    float Zp[2][2 * kOutMax * TM];         // [net][half][o][s]
    RollSlot<Env> slot[kSlots];
    StatsScratch<NT / 32> red;
};

struct RollArgs {
    MlpDesc actor, critic;
    const float* params;
    AcHyper hp;
    int64_t N;
    int t0, nsteps, T;          // rollout columns t0 .. t0 + nsteps - 1 of T
    int final_bootstrap;        // also write states[:, :, t0 + nsteps] and V of it (only when t0 + nsteps == T)
    unsigned long long* policy_rng;   // (4, N)
    float* states;              // (NOBS, N, T + 1)
    void* actions;              // (N, T) int32 | f32: continuous actions as sampled (the env receives them clamped, env_action)
    float* logp;                // (N, T)
    float* values;              // (N, T + 1)
    float* rewards;             // (N, T)
    uint8_t* terminals;         // (N, T)
};

// A CTA owns one group of up to kSlots tiles for the whole launch (the caller bounds N by it).  LOG: finished episodes are also
// written to the env's episode log.
template <class Env, int ACT, bool LOG>
__global__ void __launch_bounds__(NT, 2) rollout_tc_kernel(RollArgs g, typename Env::P p, EnvArgs<LOG> ea) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    SmemRoll<Env>& sm = *reinterpret_cast<SmemRoll<Env>*>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q = warp & 3, c = warp >> 2;
    const int s = 32 * q + lane;
    const bool owner = c == 0;              // warps 0..3: thread s also owns env s of the tile
    const int cta = blockIdx.x, nctas = gridDim.x;
    const int64_t N = g.N;
    load_net<false>(sm.net[0], g.actor, g.params, ACT == B200RL_ACT_RELU ? kScale : 1.0f);
    load_net<false>(sm.net[1], g.critic, g.params + g.actor.nparams(), ACT == B200RL_ACT_RELU ? kScale : 1.0f);
    const int nslots = group_slots(cta, nctas, (N + TM - 1) / TM);
    if (owner)
        load_group(sm.slot, nslots, cta, nctas, ea, N, s, [&](RollSlot<Env>& sl, int64_t i) {
            unsigned long long pr[4];
            explore::xo_load(g.policy_rng, i, pr);
            put_stream(sl.prng, s, pr);
        });
    wg::fence_proxy_async();
    __syncthreads();
    // episode statistics of this thread's envs
    int fin_cnt = 0, fin_len = 0;
    float fin_ret = 0.f;
    const int ns = Env::NOBS;
    const int nst = g.final_bootstrap ? g.nsteps + 1 : g.nsteps;
#pragma unroll 1
    for (int step = 0; step < nst; ++step) {
        const int t = g.t0 + step;
        const bool boot = step == g.nsteps;      // extra pass: V(s_T) only
#pragma unroll 1
        for (int k = 0; k < nslots; ++k) {
            RollSlot<Env>& sl = sm.slot[k];
            const int64_t i = ((int64_t)cta + (int64_t)k * nctas) * TM + s;
            const bool live = i < N;
            // ---- observation of this step -> X (shared) and column t of the rollout states ------------------------
            if (owner) {
                float o[kInMax] = {0.f, 0.f, 0.f, 0.f};
                if (live) {
                    Env::observe(sl.st[s], o);
                    float* dst = g.states + ((size_t)N * ns) * (size_t)t + (size_t)ns * i;
                    if (ns == 4) *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
                    else {
#pragma unroll
                        for (int j = 0; j < kInMax; ++j) if (j < ns) dst[j] = o[j];
                    }
                }
#pragma unroll
                for (int j = 0; j < kInMax; ++j) sm.X[j * TM + s] = o[j];
            }
            __syncthreads();
            if (!boot) tile_forward<ACT>(sm.net[0], g.actor.act, c, s, sm.T, sm.X, sm.Zp[0]);   // actor
            // ---- critic GEMM (warpgroup 1, both blocks) while the owner threads (warpgroup 0) sample the action and step the env
            {
                float x[kInMax];
#pragma unroll
                for (int j = 0; j < kInMax; ++j) x[j] = sm.X[j * TM + s];
                layer1_to_smem<ACT>(sm.net[1], g.critic.act, x, c, s, sm.T);
            }
            wg::fence_proxy_async();
            __syncthreads();
            if (!owner) {
                gemm_block(sm.T, sm.net[1], 1);
                gemm_block(sm.T + BLK, sm.net[1], 1);
            }
            if (owner && live && !boot) {
                float z[kOutMax];
                tile_heads(sm.net[0], sm.Zp[0], s, z);
                unsigned long long pr[4];
                get_stream(sl.prng, s, pr);
                float lp;
                const uint32_t a_bits = policy::sample_head(g.actor.heads2, g.actor.nout, g.hp, z, pr, lp);
                put_stream(sl.prng, s, pr);
                reinterpret_cast<uint32_t*>(g.actions)[(size_t)N * t + i] = a_bits;
                g.logp[(size_t)N * t + i] = lp;
                const ActStep<float> r = slot_act<Env, LOG>(sl, s, p, ea.max_timeout, env_action<Env>(a_bits), fin_cnt, fin_ret, fin_len, episode_log_of(ea), i);
                g.rewards[(size_t)N * t + i] = r.rew;
                g.terminals[(size_t)N * t + i] = r.done ? 1 : 0;
            }
            __syncthreads();
            {
                float zp[kOutMax];
                head_partials<ACT>(sm.net[1], g.critic.act, c, s, sm.T, zp);
                sm.Zp[1][(c * kOutMax) * TM + s] = zp[0];
            }
            __syncthreads();
            if (owner && live) g.values[(size_t)N * t + i] = sm.net[1].b3[0] + sm.Zp[1][s] + sm.Zp[1][kOutMax * TM + s];
            // (the next pass's X / Zp writes are ordered behind this read by its first __syncthreads)
        }
    }
    if (owner)
        store_group(sm.slot, nslots, cta, nctas, ea, N, s, g.nsteps > 0, [&](const RollSlot<Env>& sl, int64_t i) {
            unsigned long long pr[4];
            get_stream(sl.prng, s, pr);
            explore::xo_store(g.policy_rng, i, pr);
        });
    cta_episode_stats(ea.stats, fin_cnt, fin_ret, fin_len, sm.red);
}

// ---------------------------------------------------------------------------------------------------------------------
// fused evaluation (b200rl_evaluate): n_steps x { obs -> actor -> greedy | sampled action -> env step (+ fused auto-reset) ->
// record of the episodes that end }.  The weights are fixed, so nothing couples the tiles: a CTA runs the whole window on one
// group of up to kSlots resident tiles, writes the group back and takes the next one (no limit on N).  The head outputs come
// from the device functions, template activation and operand scale of forward_tc_kernel's mode 1, so the staged greedy
// policy (b200rl_net_act_greedy -> nn_mlp_forward) and this kernel pick the same actions bit for bit.
template <class Env> struct EvalSlot : EnvSlot<Env> {
    int cnt[TM];                           // episodes finished in the window
    unsigned long long prng[4 * TM];       // policy stream (MODE 1) | explorer stream (MODE 2)
};
template <class Env> struct SmemEval {
    alignas(128) uint8_t T[TILE_BYTES];
    NetSm net;                             // actor (or Q-network)
    float X[kInMax * TM];
    float Zp[2 * kOutMax * TM];            // [half][o][s]
    EvalSlot<Env> slot[kSlots];
    int fin_cnt[TM], fin_len[TM];          // episode statistics of owner thread s (shared memory: no registers held across the window)
    float fin_ret[TM];
    StatsScratch<NT / 32> red;
};

struct EvalArgs {
    MlpDesc actor;
    const float* params;
    AcHyper hp;
    int64_t N;
    int nsteps, K;
    unsigned long long* policy_rng;     // (4, N): policy streams (MODE 1) | explorer streams (MODE 2, not greedy)
    float* returns;                     // (K, N), may be null
    int32_t* lengths;                   // (K, N), may be null
    int32_t* counts;                    // (N), may be null
};
// MODE 2: EvalArgs and the explorer of QBasedPolicy; column i at window step k plans at explorer step
// explore::column_step(step0, col0, stride, k, i) = step0 + k N + i on one GPU.  (A struct of its own: the MODE 0 / 1
// instantiations keep the kernel parameters, and the code, they had before MODE 2 existed.)
struct EvalExploreArgs : EvalArgs {
    int greedy;                         // 1: GreedyExplorer (the first maximum under `>`, no draw)
    QExplorer ex;
    double beta;
    long long step0;
    long long col0, stride;             // rank · N and world · N (0 and N on one GPU)
};
template <int MODE> using EvalArgsOf = typename std::conditional<MODE == 2, EvalExploreArgs, EvalArgs>::type;
// RUN: the arguments of MODE and the per-step terminal counts of a stretch of run() (b200rl_eval_run_episodes)
template <int MODE> struct EvalRunArgs : EvalArgsOf<MODE> {
    unsigned long long* step_counts;    // (nsteps): += lanes terminal after step j + 1 of the window; may be null
};
template <int MODE, bool RUN> using EvalKernelArgs = typename std::conditional<RUN, EvalRunArgs<MODE>, EvalArgsOf<MODE>>::type;
// the window reads and writes back a (4, N) stream per env: the policy streams (MODE 1) or the explorer streams (MODE 2, not greedy)
template <int MODE> __device__ __forceinline__ bool eval_streams(const EvalArgsOf<MODE>& g) {
    if constexpr (MODE == 2) return !g.greedy;
    else return MODE == 1;
}

// MODE 0: greedy (greedy.cuh, no draw), 1: sample_head on the policy streams, 2: a Q-network planned by its explorer
// (plan_q_column, b200rl_evaluate_explore).  DUEL (MODE 0 / 2): a dueling Q-network, its head rows combined into Q (duel.cuh) before
// the selection; the instantiations without it are the code of the other kinds.  XEXT (MODE 2): the explorer kinds 2-4 compiled.
// RUN: a stretch of run(policy, env, stop) rather than an evaluation of its own — no records (K = 0); each step's terminal lanes are
// added to g.step_counts[step] (one __syncthreads_count per resident tile, one atomic per CTA and step), and with LOG the finished episodes
// go to the env's episode log as the rollout and collect kernels write it.  The instantiations without RUN are the code of b200rl_evaluate.
// (layer 1 and the head epilogue not unrolled: the relu variants would exceed 128 registers and spill)
template <class Env, int ACT, int MODE, bool DUEL = false, bool XEXT = false, bool RUN = false, bool LOG = false>
__global__ void __launch_bounds__(NT, 2) evaluate_tc_kernel(EvalKernelArgs<MODE, RUN> g, typename Env::P p, EnvArgs<LOG> ea) {
    static_assert(RUN || !LOG, "b200rl_evaluate writes no episode log");
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    SmemEval<Env>& sm = *reinterpret_cast<SmemEval<Env>*>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q = warp & 3, c = warp >> 2;
    const int s = 32 * q + lane;
    const bool owner = c == 0;              // warps 0..3: thread s also owns env s of each resident tile
    const int64_t N = g.N;
    const int nctas = gridDim.x;
    const int64_t ntiles = (N + TM - 1) / TM;
    load_net<DUEL>(sm.net, g.actor, g.params, ACT == B200RL_ACT_RELU ? kScale : 1.0f);
    if (owner) { sm.fin_cnt[s] = 0; sm.fin_len[s] = 0; sm.fin_ret[s] = 0.f; }
#pragma unroll 1
    for (int64_t base = blockIdx.x; base < ntiles; base += (int64_t)nctas * kSlots) {
        const int nslots = group_slots(base, nctas, ntiles);
        if (owner)
            load_group(sm.slot, nslots, base, nctas, ea, N, s, [&](EvalSlot<Env>& sl, int64_t i) {
                sl.cnt[s] = 0;
                if (eval_streams<MODE>(g)) {
                    unsigned long long pr[4];
                    explore::xo_load(g.policy_rng, i, pr);
                    put_stream(sl.prng, s, pr);
                }
            });
        wg::fence_proxy_async();            // (the first pass: the weight image written by load_net, read by wgmma)
        __syncthreads();
#pragma unroll 1
        for (int step = 0; step < g.nsteps; ++step) {
            int ended = 0;                  // RUN: lanes of the group terminal after this step (the same in every thread)
#pragma unroll 1
            for (int k = 0; k < nslots; ++k) {
                // (env index and slot are recomputed after the GEMM rather than held in registers across it)
                if (owner) {
                    float o[kInMax] = {0.f, 0.f, 0.f, 0.f};
                    if ((base + (int64_t)k * nctas) * TM + s < N) Env::observe(sm.slot[k].st[s], o);
#pragma unroll
                    for (int j = 0; j < kInMax; ++j) sm.X[j * TM + s] = o[j];
                }
                __syncthreads();
                tile_forward<ACT, 1>(sm.net, g.actor.act, c, s, sm.T, sm.X, sm.Zp);
                const int64_t i = (base + (int64_t)k * nctas) * TM + s;
                bool done = false;
                if (owner && i < N) {
                    EvalSlot<Env>& sl = sm.slot[k];
                    float z[kOutMax];
                    tile_heads(sm.net, sm.Zp, s, z);
                    if (DUEL) duel::combine(z, g.actor.nout);
                    uint32_t a_bits;
                    if constexpr (MODE == 0) {
                        a_bits = greedy::greedy_action(g.actor, z);
                    } else if constexpr (MODE == 2) {
                        a_bits = (uint32_t)plan_q_column<XEXT>(g.greedy, g.ex, g.beta, explore::column_step(g.step0, g.col0, g.stride, step, i), z, g.actor.nout,
                                                                sl.prng, s);
                    } else {
                        unsigned long long pr[4];
                        get_stream(sl.prng, s, pr);
                        float lp;
                        a_bits = policy::sample_head(g.actor.heads2, g.actor.nout, g.hp, z, pr, lp);
                        put_stream(sl.prng, s, pr);
                    }
                    // (no episode log without RUN: an evaluation is a run of its own, whose episodes the training hook does not see)
                    const ActStep<float> r = slot_act<Env, LOG>(sl, s, p, ea.max_timeout, env_action<Env>(a_bits), sm.fin_cnt[s], sm.fin_ret[s],
                                                                sm.fin_len[s], episode_log_of(ea), i);
                    if constexpr (RUN) {
                        done = r.done;
                    } else if (r.done) {
                        const int e = sl.cnt[s];   // record of the episode that ends: its return and env.t
                        if (e < g.K) {
                            if (g.returns) g.returns[(size_t)g.K * i + e] = r.ret;
                            if (g.lengths) g.lengths[(size_t)g.K * i + e] = r.len;
                        }
                        sl.cnt[s] = e + 1;
                    }
                }
                if constexpr (RUN) ended += __syncthreads_count(done);
            }
            if constexpr (RUN) {
                if (tid == 0 && ended && g.step_counts) atomicAdd(g.step_counts + step, (unsigned long long)ended);
            }
        }
        // (each owner thread touches only its own entries: no barrier before the next group's loads)
        if (owner)
            store_group(sm.slot, nslots, base, nctas, ea, N, s, g.nsteps > 0, [&](const EvalSlot<Env>& sl, int64_t i) {
                if (eval_streams<MODE>(g)) {
                    unsigned long long pr[4];
                    get_stream(sl.prng, s, pr);
                    explore::xo_store(g.policy_rng, i, pr);
                }
                if (g.counts) g.counts[i] = sl.cnt[s];
            });
    }
    cta_episode_stats(ea.stats, owner ? sm.fin_cnt[s] : 0, owner ? sm.fin_ret[s] : 0.f, owner ? sm.fin_len[s] : 0, sm.red);
}

// ---------------------------------------------------------------------------------------------------------------------
// fused DQN collect (b200rl_replay_run): nsteps x { obs -> Q -> BatchExplorer column (explore.cuh) | findmax (GreedyExplorer) ->
// env step (+ fused auto-reset) -> push!(trajectory) of the lane (ring.cuh) }.  The Q-network is fixed during a window, so a CTA
// runs the whole window on one group of up to kSlots resident tiles (env state, env stream and explorer stream in shared
// memory), writes it back and takes the next group (no limit on N).  Sum-tree leaves are written as the pushes happen (a lane
// owns its leaves, so the last write is the final value); after the window each lane emits the keys of its touched slots — a
// contiguous run mod cap + 1, at most cap + 1 of them, no duplicates — and the caller rebuilds the tree once from the children,
// which gives the tree the per-step rebuilds give.  The head outputs are those of nn_mlp_forward's tensor-core path (see
// evaluate_tc_kernel), so the actions equal the staged q_explore / q_act selection bit for bit.
template <class Env> struct ReplaySlot : EnvSlot<Env> {
    int p0[TM];                            // slot of the first touched leaf of the lane (head - 1 at the start)
    int adv[TM];                           // frames written in the window
    unsigned long long xrng[4 * TM];       // explorer stream
};
template <class Env> struct SmemReplay {
    alignas(128) uint8_t T[TILE_BYTES];
    NetSm net;
    float X[kInMax * TM];
    float Zp[2 * kOutMax * TM];
    ReplaySlot<Env> slot[kSlots];
    int fin_cnt[TM], fin_len[TM];
    float fin_ret[TM];
    long long dv[TM];                      // change of the sampleable count, per owner thread
    StatsScratch<NT / 32> red;
    long long red_dv[NT / 32];
};
struct ReplayArgs {
    MlpDesc q;
    const float* params;
    int64_t N;
    int nsteps;
    int greedy;                            // 1: GreedyExplorer (findmax with `>`, no draw)
    QExplorer ex;                          // (beta: the kernel's last parameter)
    const long long* step_dev;             // explorer step before the window (device)
    long long col0, xstride;               // explore::column_step: rank · N and world · N (0 and N on one GPU)
    unsigned long long* xrng;              // (4, N) explorer streams
    Ring ring;
    float default_priority;
    int prioritized;
    int64_t* keys;                         // (stride, lanes): touched leaves of each lane, -1 padded
    float* vals;
    int stride;                            // min(2 nsteps + 1, cap + 1)
};

// DUEL: a dueling Q-network, its head rows combined into Q (duel.cuh) before the selection (the instantiations without it are the
// code of a plain Q-network).  XEXT: the explorer kinds 2-4 (speedy, weighted / Gumbel softmax; explore::select<true>) — the
// instantiations without it compile the ϵ-greedy kinds 0 / 1 only.  LOG: finished episodes are also written to the env's episode log.
template <class Env, int ACT, bool DUEL, bool XEXT, bool LOG>
__global__ void __launch_bounds__(NT, 2) replay_collect_tc_kernel(ReplayArgs g, typename Env::P p, EnvArgs<LOG> ea, double beta) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    SmemReplay<Env>& sm = *reinterpret_cast<SmemReplay<Env>*>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q = warp & 3, c = warp >> 2;
    const int s = 32 * q + lane;
    const bool owner = c == 0;
    const int64_t N = g.N;
    const int nctas = gridDim.x;
    const int64_t ntiles = (N + TM - 1) / TM;
    const long long step0 = g.greedy ? 0 : *g.step_dev;
    const Ring& r = g.ring;
    const int64_t F = r.frames();
    load_net<DUEL>(sm.net, g.q, g.params, ACT == B200RL_ACT_RELU ? kScale : 1.0f);
    if (owner) { sm.fin_cnt[s] = 0; sm.fin_len[s] = 0; sm.fin_ret[s] = 0.f; sm.dv[s] = 0; }
#pragma unroll 1
    for (int64_t base = blockIdx.x; base < ntiles; base += (int64_t)nctas * kSlots) {
        const int nslots = group_slots(base, nctas, ntiles);
        // (the load of load_group written out: through load_group, ptxas spills 8 / 20 B in the Pendulum dueling relu instantiation)
        if (owner)
            for (int k = 0; k < nslots; ++k) {
                const int64_t i = (base + (int64_t)k * nctas) * TM + s;
                ReplaySlot<Env>& sl = sm.slot[k];
                if (i < N) {
                    sl.st[s] = Env::load(ea.state, i);
                    sl.t[s] = ea.t[i];
                    sl.flags[s] = ea.flags[i];
                    sl.ep_ret[s] = ea.ep_ret[i];
                    sl.p0[s] = (int)(((int64_t)r.head[i] + F - 1) % F);
                    sl.adv[s] = 0;
                    Xo e = load_rng(ea.rng, i);
                    sl.erng[s] = e.s0; sl.erng[TM + s] = e.s1; sl.erng[2 * TM + s] = e.s2; sl.erng[3 * TM + s] = e.s3;
                    if (!g.greedy) {
                        unsigned long long xr[4];
                        explore::xo_load(g.xrng, i, xr);
                        sl.xrng[s] = xr[0]; sl.xrng[TM + s] = xr[1]; sl.xrng[2 * TM + s] = xr[2]; sl.xrng[3 * TM + s] = xr[3];
                    }
                }
            }
        wg::fence_proxy_async();
        __syncthreads();
#pragma unroll 1
        for (int step = 0; step < g.nsteps; ++step) {
#pragma unroll 1
            for (int k = 0; k < nslots; ++k) {
                if (owner) {
                    float o[kInMax] = {0.f, 0.f, 0.f, 0.f};
                    if ((base + (int64_t)k * nctas) * TM + s < N) Env::observe(sm.slot[k].st[s], o);
#pragma unroll
                    for (int j = 0; j < kInMax; ++j) sm.X[j * TM + s] = o[j];
                }
                __syncthreads();
                tile_forward<ACT, 1>(sm.net, g.q.act, c, s, sm.T, sm.X, sm.Zp);
                const int64_t i = (base + (int64_t)k * nctas) * TM + s;
                if (owner && i < N) {
                    ReplaySlot<Env>& sl = sm.slot[k];
                    float z[kOutMax];
                    tile_heads(sm.net, sm.Zp, s, z);
                    if (DUEL) duel::combine(z, g.q.nout);
                    const int a1 = plan_q_column<XEXT>(g.greedy, g.ex, beta, explore::column_step(step0, g.col0, g.xstride, step, i), z, g.q.nout,
                                                                sl.xrng, s);
                    const ActStep<float> res = slot_act<Env, LOG>(sl, s, p, ea.max_timeout, (typename Env::act_t)a1, sm.fin_cnt[s], sm.fin_ret[s], sm.fin_len[s], episode_log_of(ea), i);
                    // push!(trajectory, (state = s', action = env.action, reward, terminal)) of lane i
                    float nobs[kInMax];
                    Env::observe(sl.st[s], nobs);
                    RingLeaves lv;
                    int adv = 0;
                    sm.dv[s] += ring::push_sart(r, i, (int32_t)sl.last_act[s], res.rew, (uint8_t)sl.flags[s], nobs, g.default_priority, lv, &adv);
                    sl.adv[s] += adv;
                    if (g.prioritized)
                        for (int j = 0; j < 3; ++j) if (lv.key[j] >= 0) r.tree[r.L + lv.key[j]] = lv.val[j];
                }
            }
        }
        if (owner)
            store_group(sm.slot, nslots, base, nctas, ea, N, s, g.nsteps > 0, [&](const ReplaySlot<Env>& sl, int64_t i) {
                if (!g.greedy) {
                    unsigned long long xr[4];
                    get_stream(sl.xrng, s, xr);
                    explore::xo_store(g.xrng, i, xr);
                }
                if (g.prioritized) {   // the lane's touched slots p0, p0 + 1, ... (mod cap + 1), one key each
                    const int n_touched = (int)min((int64_t)sl.adv[s] + 1, F);
                    for (int j = 0; j < g.stride; ++j) {
                        int64_t key = -1;
                        float v = 0.f;
                        if (j < n_touched) { key = (((int64_t)sl.p0[s] + j) % F) * r.lanes + i; v = r.tree[r.L + key]; }
                        g.keys[(int64_t)j * N + i] = key;
                        g.vals[(int64_t)j * N + i] = v;
                    }
                }
            });
    }
    // episode statistics and the sampleable count: one atomic each per CTA
    cta_episode_stats(ea.stats, owner ? sm.fin_cnt[s] : 0, owner ? sm.fin_ret[s] : 0.f, owner ? sm.fin_len[s] : 0, sm.red,
                      owner ? sm.dv[s] : 0, sm.red_dv, (unsigned long long*)r.n_valid);
}

// ---------------------------------------------------------------------------------------------------------------------
// host side of the fused kernels
// Launches `kernel` on min(2 per SM, units) CTAs of NT threads with sizeof(Smem) of dynamic shared memory; the instantiation's
// shared-memory limit is raised on its first launch on a device (the attribute call is not free and may serialise with running kernels).
template <auto kernel, class Smem, class... Args> int launch_fused(b200rl_ctx* ctx, int64_t units, const Args&... args) {
    const size_t smem = sizeof(Smem) + 128;
    static unsigned long long attr_devices = 0;
    if (first_use_on_device(attr_devices, ctx->device))
        CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int grid = 2 * ctx->sm_count;
    if ((int64_t)grid > units) grid = (int)units;
    kernel<<<grid, NT, smem, ctx->stream>>>(args...);
    LAUNCH_CHECK(ctx);
    return B200RL_OK;
}

template <class Env> struct EnvTag { using type = Env; };
// Calls f(EnvTag<Env>{}, params) with the device env type of the handle and its parameters (a continuous variant reads the
// parameter block of its discrete kind, which has the same layout).  The caller has checked that the networks can read the env
// (b200rl_env_internal_obs_f32): a Float32 env, or a Float64 one behind StateTransformedEnv(env, Float32).
template <class F> int with_learner_env(const EnvView& v, F&& f) {
    if (v.dtype == B200RL_F64) {
        switch (v.kind) {
            case B200RL_ENV_CARTPOLE:   // (CartPoleEnv(continuous = true) is Float32 only)
                return f(EnvTag<CartPoleD<double, false>>{}, v.p.cp64);
            case B200RL_ENV_PENDULUM:
                return v.continuous ? f(EnvTag<PendulumD<true, double>>{}, v.p.pend64) : f(EnvTag<PendulumD<false, double>>{}, v.p.pend64);
            case B200RL_ENV_MOUNTAINCAR:
                return v.continuous ? f(EnvTag<MountainCarD<true, double>>{}, v.p.mc64) : f(EnvTag<MountainCarD<false, double>>{}, v.p.mc64);
        }
        return B200RL_ERR_UNSUPPORTED;
    }
    switch (v.kind) {
        case B200RL_ENV_CARTPOLE: {
            if (!v.continuous) return f(EnvTag<CartPoleD<float, false>>{}, v.p.cp32);
            CartPoleD<float, true>::P q;
            static_assert(sizeof q == sizeof v.p.cp32, "same params layout");
            memcpy(&q, &v.p.cp32, sizeof q);
            return f(EnvTag<CartPoleD<float, true>>{}, q);
        }
        case B200RL_ENV_PENDULUM:
            return v.continuous ? f(EnvTag<PendulumD<true>>{}, v.p.pend) : f(EnvTag<PendulumD<false>>{}, v.p.pend);
        case B200RL_ENV_MOUNTAINCAR: {
            if (!v.continuous) return f(EnvTag<MountainCarD<false>>{}, v.p.mc);
            MountainCarD<true>::P q;
            static_assert(sizeof q == sizeof v.p.mc, "same params layout");
            memcpy(&q, &v.p.mc, sizeof q);
            return f(EnvTag<MountainCarD<true>>{}, q);
        }
    }
    return B200RL_ERR_UNSUPPORTED;
}

// the evaluate_tc_kernel instantiation of the network's activation (and, MODE 0 / 2, of a dueling head)
template <class Env, int MODE, bool XEXT = false, bool RUN = false, bool LOG = false>
int launch_evaluate(b200rl_ctx* ctx, int64_t groups, const EvalKernelArgs<MODE, RUN>& g, const typename Env::P& p, const EnvArgs<LOG>& ea) {
    constexpr int RELU = B200RL_ACT_RELU, TANH = B200RL_ACT_TANH;
    const bool relu = g.actor.act == RELU;
    if constexpr (MODE != 1) {
        if (g.actor.duel)
            return relu ? launch_fused<evaluate_tc_kernel<Env, RELU, MODE, true, XEXT, RUN, LOG>, SmemEval<Env>>(ctx, groups, g, p, ea)
                        : launch_fused<evaluate_tc_kernel<Env, TANH, MODE, true, XEXT, RUN, LOG>, SmemEval<Env>>(ctx, groups, g, p, ea);
    }
    return relu ? launch_fused<evaluate_tc_kernel<Env, RELU, MODE, false, XEXT, RUN, LOG>, SmemEval<Env>>(ctx, groups, g, p, ea)
                : launch_fused<evaluate_tc_kernel<Env, TANH, MODE, false, XEXT, RUN, LOG>, SmemEval<Env>>(ctx, groups, g, p, ea);
}
// a stretch of run(): the instantiation with the episode log when the env has one attached, the one without it otherwise
template <class Env, int MODE, bool XEXT = false>
int launch_eval_run(b200rl_ctx* ctx, int64_t groups, const EvalRunArgs<MODE>& g, const typename Env::P& p, const EnvView& v) {
    if (v.log.count) return launch_evaluate<Env, MODE, XEXT, true, true>(ctx, groups, g, p, EnvArraysLog{v.a, v.log});
    return launch_evaluate<Env, MODE, XEXT, true, false>(ctx, groups, g, p, v.a);
}

template <class Env, bool XEXT, bool LOG>
int launch_replay_collect(b200rl_ctx* ctx, int64_t groups, const ReplayArgs& g, const typename Env::P& p, const EnvArgs<LOG>& ea, double beta) {
    constexpr int RELU = B200RL_ACT_RELU, TANH = B200RL_ACT_TANH;
    const bool relu = g.q.act == RELU;
    if (g.q.duel)
        return relu ? launch_fused<replay_collect_tc_kernel<Env, RELU, true, XEXT, LOG>, SmemReplay<Env>>(ctx, groups, g, p, ea, beta)
                    : launch_fused<replay_collect_tc_kernel<Env, TANH, true, XEXT, LOG>, SmemReplay<Env>>(ctx, groups, g, p, ea, beta);
    return relu ? launch_fused<replay_collect_tc_kernel<Env, RELU, false, XEXT, LOG>, SmemReplay<Env>>(ctx, groups, g, p, ea, beta)
                : launch_fused<replay_collect_tc_kernel<Env, TANH, false, XEXT, LOG>, SmemReplay<Env>>(ctx, groups, g, p, ea, beta);
}
// the instantiation with the episode log when the env has one attached, the one without it otherwise
template <class Env, bool XEXT>
int launch_replay_collect(b200rl_ctx* ctx, int64_t groups, const ReplayArgs& g, const typename Env::P& p, const EnvView& v, double beta) {
    if (v.log.count) return launch_replay_collect<Env, XEXT, true>(ctx, groups, g, p, EnvArraysLog{v.a, v.log}, beta);
    return launch_replay_collect<Env, XEXT, false>(ctx, groups, g, p, v.a, beta);
}
template <class Env, int ACT>
int launch_rollout(b200rl_ctx* ctx, int64_t ntiles, const RollArgs& g, const typename Env::P& p, const EnvView& v) {
    if (v.log.count) return launch_fused<rollout_tc_kernel<Env, ACT, true>, SmemRoll<Env>>(ctx, ntiles, g, p, EnvArraysLog{v.a, v.log});
    return launch_fused<rollout_tc_kernel<Env, ACT, false>, SmemRoll<Env>>(ctx, ntiles, g, p, v.a);
}

}  // namespace

bool nn_tc_supported(const MlpDesc& d) { return d.H == 64 && d.in <= kInMax && d.rows() <= kOutMax; }

int nn_tc_forward(b200rl_ctx* ctx, int grid, const MlpDesc& actor, const MlpDesc& critic, const float* params, const AcHyper& hp, int mode,
                  const float* obs, int64_t N, unsigned long long* rng, void* action_out, float* logp_out, float* value_out, float* head_out,
                  float* state_copy) {
    size_t smem = sizeof(SmemFwd) + 128;
    static unsigned long long attr_devices = 0;   // once per device
    if (first_use_on_device(attr_devices, ctx->device)) {
        CUDA_TRY(cudaFuncSetAttribute(forward_tc_kernel<B200RL_ACT_RELU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(forward_tc_kernel<B200RL_ACT_TANH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(forward_tc_kernel<-1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    const bool same = mode != 0 || actor.act == critic.act;   // mode 1 runs `actor` alone
    if (same && actor.act == B200RL_ACT_RELU)
        forward_tc_kernel<B200RL_ACT_RELU><<<grid, NT, smem, ctx->stream>>>(actor, critic, params, hp, mode, obs, N, rng, action_out, logp_out, value_out, head_out, state_copy);
    else if (same && actor.act == B200RL_ACT_TANH)
        forward_tc_kernel<B200RL_ACT_TANH><<<grid, NT, smem, ctx->stream>>>(actor, critic, params, hp, mode, obs, N, rng, action_out, logp_out, value_out, head_out, state_copy);
    else
        forward_tc_kernel<-1><<<grid, NT, smem, ctx->stream>>>(actor, critic, params, hp, mode, obs, N, rng, action_out, logp_out, value_out, head_out, state_copy);
    LAUNCH_CHECK(ctx);
    return B200RL_OK;
}

// Fused rollout of `nsteps` env steps starting at column t0.  Returns B200RL_ERR_UNSUPPORTED (without setting an error
// message the caller would surface) when the configuration is outside the fused kernel's envelope: the caller then steps
// through plan! / act! launches, which computes the same thing.
int nn_tc_rollout(b200rl_ctx* ctx, b200rl_env* env, const MlpDesc& actor, const MlpDesc& critic, const float* params, const AcHyper& hp,
                  unsigned long long* policy_rng, int t0, int nsteps, int T, int final_bootstrap, float* states, void* actions, float* logp,
                  float* values, float* rewards, uint8_t* terminals) {
    EnvView v;
    TRY(b200rl_env_internal_view(env, &v));
    if (!(nn_tc_supported(actor) && nn_tc_supported(critic)) || critic.nout != 1 || !b200rl_env_internal_obs_f32(env)) return B200RL_ERR_UNSUPPORTED;
    if (actor.act != critic.act) return B200RL_ERR_UNSUPPORTED;   // the fused kernel is compiled per activation (staged launches handle a mixed pair)
    const int64_t ntiles = (v.N + TM - 1) / TM;
    if (ntiles > (int64_t)kSlots * 2 * ctx->sm_count) return B200RL_ERR_UNSUPPORTED;
    if ((actor.heads2 != 0) != (v.continuous != 0)) return B200RL_ERR_UNSUPPORTED;   // Gaussian head <-> continuous action space
    if (!v.continuous && actor.nout != b200rl_env_internal_n_actions(env)) return B200RL_ERR_UNSUPPORTED;
    const RollArgs g{actor, critic, params, hp, v.N, t0, nsteps, T, final_bootstrap, policy_rng, states, actions, logp, values, rewards, terminals};
    const int st = with_learner_env(v, [&](auto env_type, const auto& p) {
        using Env = typename decltype(env_type)::type;
        // the activation is a template parameter (both trunks share it, checked above)
        return actor.act == B200RL_ACT_RELU ? launch_rollout<Env, B200RL_ACT_RELU>(ctx, ntiles, g, p, v)
                                            : launch_rollout<Env, B200RL_ACT_TANH>(ctx, ntiles, g, p, v);
    });
    if (st == B200RL_OK) b200rl_env_internal_add_steps(env, (uint64_t)nsteps);
    return st;
}

// Fused evaluation window (after the caller's forced reset).  mode 0 greedy, 1 sampled, 2 a Q-network planned by the explorer `ex`
// (null: GreedyExplorer) from ex->step on the streams policy_rng.  The caller has validated net <-> env <-> explorer;
// B200RL_ERR_UNSUPPORTED (no side effect, no error message) = outside the fused envelope: the caller steps through staged launches.
int nn_tc_evaluate(b200rl_ctx* ctx, b200rl_env* env, const MlpDesc& actor, const float* params, const AcHyper& hp, int mode, int nsteps,
                   int K, unsigned long long* policy_rng, float* returns, int32_t* lengths, int32_t* counts, const b200rl_explorer* ex) {
    EnvView v;
    TRY(b200rl_env_internal_view(env, &v));
    if (!nn_tc_supported(actor) || !b200rl_env_internal_obs_f32(env) || (mode == 2 && v.continuous)) return B200RL_ERR_UNSUPPORTED;
    const b200rl_explorer e = ex ? *ex : b200rl_explorer{};
    const EvalArgs g{actor, params, hp, v.N, nsteps, K, policy_rng, returns, lengths, counts};
    const EvalExploreArgs gx{g, ex ? 0 : 1, QExplorer{e.eps_stable, e.eps_init, e.warmup_steps, e.decay_steps, e.step, e.kind, e.is_break_tie},
                             e.beta, (long long)e.step, (long long)b200rl_comm_rank(ctx) * v.N, (long long)b200rl_comm_world(ctx) * v.N};
    const int64_t groups = ((v.N + TM - 1) / TM + kSlots - 1) / kSlots;
    const int st = with_learner_env(v, [&](auto env_type, const auto& p) {
        using Env = typename decltype(env_type)::type;
        if (mode == 0) return launch_evaluate<Env, 0>(ctx, groups, g, p, v.a);
        if (mode == 1) return launch_evaluate<Env, 1>(ctx, groups, g, p, v.a);
        if constexpr (std::is_floating_point<typename Env::act_t>::value) return (int)B200RL_ERR_UNSUPPORTED;   // (rejected above)
        else if (ex && ex->kind >= 2) return launch_evaluate<Env, 2, true>(ctx, groups, gx, p, v.a);
        else return launch_evaluate<Env, 2>(ctx, groups, gx, p, v.a);
    });
    if (st == B200RL_OK) b200rl_env_internal_add_steps(env, (uint64_t)nsteps);
    return st;
}

// A stretch of nsteps steps of run(policy, env, stop) on the fused evaluation kernel (RUN instantiations): the window of
// nn_tc_evaluate from the env's current state, without records, with the episode log and the per-step counts.  The caller has
// validated net <-> env <-> explorer; B200RL_ERR_UNSUPPORTED (no side effect, no error message) = outside the fused envelope.
int nn_tc_eval_run(b200rl_ctx* ctx, b200rl_env* env, const MlpDesc& actor, const float* params, const AcHyper& hp, int mode, int nsteps,
                   unsigned long long* policy_rng, const b200rl_explorer* ex, unsigned long long* step_counts) {
    EnvView v;
    TRY(b200rl_env_internal_view(env, &v));
    if (!nn_tc_supported(actor) || !b200rl_env_internal_obs_f32(env) || (mode == 2 && v.continuous)) return B200RL_ERR_UNSUPPORTED;
    const b200rl_explorer e = ex ? *ex : b200rl_explorer{};
    const EvalArgs g{actor, params, hp, v.N, nsteps, 0, policy_rng, nullptr, nullptr, nullptr};
    const EvalRunArgs<0> g0{g, step_counts};
    const EvalRunArgs<2> gx{EvalExploreArgs{g, ex ? 0 : 1,
                                            QExplorer{e.eps_stable, e.eps_init, e.warmup_steps, e.decay_steps, e.step, e.kind, e.is_break_tie},
                                            e.beta, (long long)e.step, (long long)b200rl_comm_rank(ctx) * v.N,
                                            (long long)b200rl_comm_world(ctx) * v.N},
                            step_counts};
    const int64_t groups = ((v.N + TM - 1) / TM + kSlots - 1) / kSlots;
    const int st = with_learner_env(v, [&](auto env_type, const auto& p) {
        using Env = typename decltype(env_type)::type;
        if (mode == 0) return launch_eval_run<Env, 0>(ctx, groups, g0, p, v);
        if (mode == 1) return launch_eval_run<Env, 1>(ctx, groups, EvalRunArgs<1>{g, step_counts}, p, v);
        if constexpr (std::is_floating_point<typename Env::act_t>::value) return (int)B200RL_ERR_UNSUPPORTED;   // (rejected above)
        else if (ex && ex->kind >= 2) return launch_eval_run<Env, 2, true>(ctx, groups, gx, p, v);
        else return launch_eval_run<Env, 2>(ctx, groups, gx, p, v);
    });
    if (st == B200RL_OK) b200rl_env_internal_add_steps(env, (uint64_t)nsteps);
    return st;
}

// Fused DQN collect window (see replay_collect_tc_kernel).  The caller has validated net <-> env <-> ring and sized keys / vals to
// (stride, N); B200RL_ERR_UNSUPPORTED (no side effect) = outside the fused envelope: the caller steps through staged launches.
int nn_tc_replay_collect(b200rl_ctx* ctx, b200rl_env* env, const MlpDesc& q, const float* params, const b200rl_explorer* ex,
                         const long long* step_dev, unsigned long long* xrng, const Ring& ring, float default_priority, int prioritized,
                         int nsteps, int64_t* keys, float* vals, int stride) {
    EnvView v;
    TRY(b200rl_env_internal_view(env, &v));
    if (!nn_tc_supported(q) || !b200rl_env_internal_obs_f32(env) || v.continuous || ring.ns > kInMax) return B200RL_ERR_UNSUPPORTED;
    const b200rl_explorer e = ex ? *ex : b200rl_explorer{};
    const ReplayArgs g{q, params, v.N, nsteps, ex ? 0 : 1, QExplorer{e.eps_stable, e.eps_init, e.warmup_steps, e.decay_steps, e.step, e.kind, e.is_break_tie},
                       step_dev, (long long)b200rl_comm_rank(ctx) * v.N, (long long)b200rl_comm_world(ctx) * v.N, xrng, ring,
                       default_priority, prioritized, keys, vals, stride};
    const int64_t groups = ((v.N + TM - 1) / TM + kSlots - 1) / kSlots;
    const int st = with_learner_env(v, [&](auto env_type, const auto& p) {
        using Env = typename decltype(env_type)::type;
        if constexpr (std::is_floating_point<typename Env::act_t>::value) return (int)B200RL_ERR_UNSUPPORTED;   // (rejected above)
        else if (!g.greedy && g.ex.kind >= 2) return launch_replay_collect<Env, true>(ctx, groups, g, p, v, e.beta);
        else return launch_replay_collect<Env, false>(ctx, groups, g, p, v, 0.0);
    });
    if (st == B200RL_OK) b200rl_env_internal_add_steps(env, (uint64_t)nsteps);
    return st;
}
