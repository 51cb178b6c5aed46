// fwd_tc.cu — K6 on tensor cores and the fused rollout kernel (K6 + K1 + K3 over a whole rollout in ONE launch).
//
//   forward_tc_kernel  : policy inference for one env batch (plan!): actor -> action + log-prob, critic -> value.
//   rollout_tc_kernel  : n_steps x { obs -> actor -> sample action -> critic -> value -> env step (+ fused auto-reset) ->
//                        write the transition into column t of the rollout tensors }.  A CTA owns up to two tiles of 128
//                        envs for the whole launch; their env state and both RNG streams stay in shared memory, the weights of
//                        both networks too.  Replaces 2 launches per env step (agent_base.jl:45-66 stage loop, run.jl:52-68).
//   evaluate_tc_kernel : n_steps x { obs -> actor -> greedy | sampled action -> env step (+ fused auto-reset) -> per-env episode
//                        records }: the actor alone, no rollout tensors (b200rl_evaluate).
//
// Both kernels are built from the same device functions (tc_fwd.cuh, env_device.cuh) and compiled with the env flags
// (-fmad=false): stepping through plan!/act! one launch at a time or through the fused rollout gives bit-identical results.
#include "common.cuh"
#include "duel.cuh"
#include "env_device.cuh"
#include "explore.cuh"
#include "greedy.cuh"
#include "ring.cuh"
#include "tc_fwd.cuh"

using namespace tcfwd;
using namespace envdev;

int b200rl_env_internal_view(b200rl_env* e, envdev::EnvView* out);
void b200rl_env_internal_add_steps(b200rl_env* e, uint64_t n);

namespace {

struct SmemFwd {
    alignas(128) uint8_t T[TILE_BYTES];   // A operand / accumulator image of the tile (tc_fwd.cuh)
    NetSm net;
    float X[kInMax * TM];                 // [i][s]
    float Zp[2 * kOutMax * TM];           // head partials [half][o][s]
};

__device__ __forceinline__ void load_rng32(const unsigned long long* rng, int64_t i, unsigned long long (&s)[4]) {
    const ulonglong2* p = reinterpret_cast<const ulonglong2*>(rng + 4 * i);
    ulonglong2 a = p[0], b = p[1];
    s[0] = a.x; s[1] = a.y; s[2] = b.x; s[3] = b.y;
}
__device__ __forceinline__ void store_rng32(unsigned long long* rng, int64_t i, const unsigned long long (&s)[4]) {
    ulonglong2* p = reinterpret_cast<ulonglong2*>(rng + 4 * i);
    p[0] = make_ulonglong2(s[0], s[1]);
    p[1] = make_ulonglong2(s[2], s[3]);
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
        {
            float x[kInMax];
#pragma unroll
            for (int k = 0; k < kInMax; ++k) x[k] = sm.X[k * TM + s];
            layer1_to_smem<ACT>(sm.net, d.act, x, c, s, sm.T);
        }
        wg::fence_proxy_async();
        __syncthreads();
        gemm_block(sm.T + c * BLK, sm.net, c);   // warpgroup c: samples 64c .. 64c+63
        __syncthreads();
        {
            float zp[kOutMax];
            head_partials<ACT>(sm.net, d.act, c, s, sm.T, zp);
#pragma unroll
            for (int o = 0; o < kOutMax; ++o) sm.Zp[(c * kOutMax + o) * TM + s] = zp[o];
        }
        __syncthreads();               // accumulator reads done before the next tile's layer 1 overwrites the image
        if (tid < TM) {
            int64_t i = tile * TM + tid;
            if (i < N) {
                float z[kOutMax];
#pragma unroll
                for (int o = 0; o < kOutMax; ++o) z[o] = sm.net.b3[o] + sm.Zp[o * TM + tid] + sm.Zp[(kOutMax + o) * TM + tid];
                if (mode == 1 && d.duel) duel::combine(z, d.nout);   // dueling Q-network: the combined Q, not the head rows
                if (head_out && (mode == 1 || role == 0))
                    for (int o = 0; o < d.nout; ++o) head_out[(int64_t)d.nout * i + o] = z[o];
                if (mode == 0 && role == 1) {
                    if (value_out) value_out[i] = z[0];
                } else if (mode == 0) {
                    unsigned long long st[4];
                    load_rng32(rng, i, st);
                    float lp;
                    uint32_t a = sample_head(actor, hp, z, st, lp);
                    if (action_out) reinterpret_cast<uint32_t*>(action_out)[i] = a;
                    if (logp_out) logp_out[i] = lp;
                    store_rng32(rng, i, st);
                }
            }
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// fused rollout
constexpr int kSlots = 2;   // tiles of 128 envs a CTA keeps resident

template <class Env> struct SlotState {   // env state of one tile, one entry per env (owner thread = sample s)
    typename Env::S st[TM];
    int t[TM];
    int flags[TM];
    float ep_ret[TM];
    float last_rew[TM];
    uint32_t last_act[TM];                 // env.action after the last act! (a reset may have redrawn it), raw bits
    unsigned long long erng[4 * TM];   // env stream  [word][env]
    unsigned long long prng[4 * TM];   // policy stream
};
template <class Env> struct SmemRoll {
    alignas(128) uint8_t T[TILE_BYTES];    // A operand / accumulator image of the tile being evaluated (tc_fwd.cuh)
    NetSm net[2];                          // actor, critic
    float X[kInMax * TM];
    float Zp[2][2 * kOutMax * TM];         // [net][half][o][s]
    SlotState<Env> slot[kSlots];
    float red_f[8];
    int red_i[8], red_l[8];
};

struct RollArgs {
    MlpDesc actor, critic;
    const float* params;
    AcHyper hp;
    int64_t N;
    int t0, nsteps, T;          // rollout columns t0 .. t0 + nsteps - 1 of T
    int final_bootstrap;        // also write states[:, :, t0 + nsteps] and V of it (only when t0 + nsteps == T)
    float act_lo, act_hi;       // continuous actions: the env receives clamp(a, lo, hi), the rollout keeps a
    unsigned long long* policy_rng;   // (4, N)
    float* states;              // (NOBS, N, T + 1)
    void* actions;              // (N, T) int32 | f32
    float* logp;                // (N, T)
    float* values;              // (N, T + 1)
    float* rewards;             // (N, T)
    uint8_t* terminals;         // (N, T)
};

template <class Env, int ACT>
__global__ void __launch_bounds__(NT, 2) rollout_tc_kernel(RollArgs g, typename Env::P p, EnvArrays ea) {
    using act_t = typename Env::act_t;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    SmemRoll<Env>& sm = *reinterpret_cast<SmemRoll<Env>*>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q = warp & 3, c = warp >> 2;
    const int s = 32 * q + lane;
    const bool owner = c == 0;              // warps 0..3: thread s also owns env s of the tile
    const int cta = blockIdx.x, nctas = gridDim.x;
    const int64_t N = g.N;
    const int64_t ntiles = (N + TM - 1) / TM;
    load_net<false>(sm.net[0], g.actor, g.params, ACT == B200RL_ACT_RELU ? kScale : 1.0f);
    load_net<false>(sm.net[1], g.critic, g.params + g.actor.nparams(), ACT == B200RL_ACT_RELU ? kScale : 1.0f);
    // resident env state
    int nslots = 0;
    for (int k = 0; k < kSlots; ++k)
        if ((int64_t)cta + (int64_t)k * nctas < ntiles) nslots = k + 1;
    if (owner) {
        for (int k = 0; k < nslots; ++k) {
            const int64_t i = ((int64_t)cta + (int64_t)k * nctas) * TM + s;
            SlotState<Env>& sl = sm.slot[k];
            if (i < N) {
                sl.st[s] = Env::load(ea.state, i);
                sl.t[s] = ea.t[i];
                sl.flags[s] = ea.flags[i];
                sl.ep_ret[s] = ea.ep_ret[i];
                Xo e = load_rng(ea.rng, i);
                sl.erng[s] = e.s0; sl.erng[TM + s] = e.s1; sl.erng[2 * TM + s] = e.s2; sl.erng[3 * TM + s] = e.s3;
                unsigned long long pr[4];
                load_rng32(g.policy_rng, i, pr);
                sl.prng[s] = pr[0]; sl.prng[TM + s] = pr[1]; sl.prng[2 * TM + s] = pr[2]; sl.prng[3 * TM + s] = pr[3];
            }
        }
    }
    wg::fence_proxy_async();
    __syncthreads();
    // episode statistics of this thread's envs (device-side TotalRewardPerEpisode / BatchStepsPerEpisode, hooks.jl:146-231)
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
            SlotState<Env>& sl = sm.slot[k];
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
            float x[kInMax];
#pragma unroll
            for (int j = 0; j < kInMax; ++j) x[j] = sm.X[j * TM + s];
            uint32_t a_bits = 0;
            if (!boot) {
                // ---- actor ---------------------------------------------------------------------------------------
                layer1_to_smem<ACT>(sm.net[0], g.actor.act, x, c, s, sm.T);
                wg::fence_proxy_async();
                __syncthreads();
                gemm_block(sm.T + c * BLK, sm.net[0], c);   // warpgroup c: samples 64c .. 64c+63
                __syncthreads();
                {
                    float zp[kOutMax];
                    head_partials<ACT>(sm.net[0], g.actor.act, c, s, sm.T, zp);
#pragma unroll
                    for (int o = 0; o < kOutMax; ++o) sm.Zp[0][(c * kOutMax + o) * TM + s] = zp[o];
                }
                __syncthreads();
            }
            // ---- critic GEMM (warpgroup 1, both blocks) while the owner threads (warpgroup 0) sample the action and step the env
            layer1_to_smem<ACT>(sm.net[1], g.critic.act, x, c, s, sm.T);
            wg::fence_proxy_async();
            __syncthreads();
            if (!owner) {
                gemm_block(sm.T, sm.net[1], 1);
                gemm_block(sm.T + BLK, sm.net[1], 1);
            }
            if (owner && live && !boot) {
                float z[kOutMax];
#pragma unroll
                for (int o = 0; o < kOutMax; ++o) z[o] = sm.net[0].b3[o] + sm.Zp[0][o * TM + s] + sm.Zp[0][(kOutMax + o) * TM + s];
                unsigned long long pr[4] = {sl.prng[s], sl.prng[TM + s], sl.prng[2 * TM + s], sl.prng[3 * TM + s]};
                float lp;
                a_bits = sample_head(g.actor, g.hp, z, pr, lp);
                sl.prng[s] = pr[0]; sl.prng[TM + s] = pr[1]; sl.prng[2 * TM + s] = pr[2]; sl.prng[3 * TM + s] = pr[3];
                reinterpret_cast<uint32_t*>(g.actions)[(size_t)N * t + i] = a_bits;
                g.logp[(size_t)N * t + i] = lp;
                // act!(env, a) + fused soft reset (MultiThreadEnv): same sequence as env_step_kernel<Env, false, true>
                act_t act;
                if (std::is_same<act_t, float>::value) act = (act_t)fminf(fmaxf(__uint_as_float(a_bits), g.act_lo), g.act_hi);
                else act = (act_t)(int32_t)a_bits;
                typename Env::S st = sl.st[s];
                int tt = sl.t[s];
                const int prev = sl.flags[s];
                bool done;
                float rew;
                Env::step(p, st, tt, act, done, rew);
                if (ea.max_timeout > 0 && tt + 1 > ea.max_timeout) done = true;
                float ret = sl.ep_ret[s] + rew;
                int f = done ? 1 : 0;
                if (done && !((prev & 1) && !(prev & 2))) { fin_cnt += 1; fin_ret += ret; fin_len += tt; }
                if (done) {
                    ret = 0.f;
                    Xo e{sl.erng[s], sl.erng[TM + s], sl.erng[2 * TM + s], sl.erng[3 * TM + s]};
                    Env::reset(p, st, e, act);
                    sl.erng[s] = e.s0; sl.erng[TM + s] = e.s1; sl.erng[2 * TM + s] = e.s2; sl.erng[3 * TM + s] = e.s3;
                    tt = 0;
                    f = 3;
                }
                sl.st[s] = st; sl.t[s] = tt; sl.flags[s] = f; sl.ep_ret[s] = ret;
                g.rewards[(size_t)N * t + i] = rew;
                g.terminals[(size_t)N * t + i] = done ? 1 : 0;
                sl.last_rew[s] = rew;
                { act_t tmp = act; uint32_t bits; memcpy(&bits, &tmp, 4); sl.last_act[s] = bits; }
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
    // ---- write the env back ---------------------------------------------------------------------------------------
    if (owner) {
        for (int k = 0; k < nslots; ++k) {
            const int64_t i = ((int64_t)cta + (int64_t)k * nctas) * TM + s;
            SlotState<Env>& sl = sm.slot[k];
            if (i < N) {
                Env::store(ea.state, i, sl.st[s]);
                if (!Env::kObsIsState) Env::write_obs(ea.obs, i, N, sl.st[s]);
                ea.t[i] = sl.t[s];
                ea.flags[i] = (uint8_t)sl.flags[s];
                ea.ep_ret[i] = sl.ep_ret[s];
                store_rng(ea.rng, i, Xo{sl.erng[s], sl.erng[TM + s], sl.erng[2 * TM + s], sl.erng[3 * TM + s]});
                unsigned long long pr[4] = {sl.prng[s], sl.prng[TM + s], sl.prng[2 * TM + s], sl.prng[3 * TM + s]};
                store_rng32(g.policy_rng, i, pr);
                if (g.nsteps > 0) {
                    reinterpret_cast<float*>(ea.reward)[i] = sl.last_rew[s];
                    reinterpret_cast<uint32_t*>(ea.action)[i] = sl.last_act[s];
                }
            }
        }
    }
    // episode statistics: one atomicAdd triple per CTA
    {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            fin_cnt += __shfl_xor_sync(0xffffffffu, fin_cnt, o);
            fin_len += __shfl_xor_sync(0xffffffffu, fin_len, o);
            fin_ret += __shfl_xor_sync(0xffffffffu, fin_ret, o);
        }
        __syncthreads();
        if (lane == 0) { sm.red_i[warp] = fin_cnt; sm.red_f[warp] = fin_ret; sm.red_l[warp] = fin_len; }
        __syncthreads();
        if (tid == 0) {
            double cc = 0, rr = 0, ll = 0;
            for (int w = 0; w < NT / 32; ++w) { cc += sm.red_i[w]; rr += sm.red_f[w]; ll += sm.red_l[w]; }
            if (cc > 0) { atomicAdd(&ea.stats[0], cc); atomicAdd(&ea.stats[1], rr); atomicAdd(&ea.stats[2], ll); }
        }
    }
}

template <class Env> int launch_rollout(b200rl_ctx* ctx, const RollArgs& g, const typename Env::P& p, const EnvArrays& ea) {
    const size_t smem = sizeof(SmemRoll<Env>) + 128;
    static unsigned long long attr_devices = 0;   // once per device: the attribute call is not free and may serialise with running kernels
    if (first_use_on_device(attr_devices, ctx->device)) {
        CUDA_TRY(cudaFuncSetAttribute(rollout_tc_kernel<Env, B200RL_ACT_RELU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(rollout_tc_kernel<Env, B200RL_ACT_TANH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    const int64_t ntiles = (g.N + TM - 1) / TM;
    int grid = 2 * ctx->sm_count;
    if ((int64_t)grid > ntiles) grid = (int)ntiles;
    // the activation is a template parameter (nn_tc_rollout only comes here when both trunks share it)
    if (g.actor.act == B200RL_ACT_RELU) rollout_tc_kernel<Env, B200RL_ACT_RELU><<<grid, NT, smem, ctx->stream>>>(g, p, ea);
    else rollout_tc_kernel<Env, B200RL_ACT_TANH><<<grid, NT, smem, ctx->stream>>>(g, p, ea);
    LAUNCH_CHECK(ctx);
    return B200RL_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// fused evaluation (b200rl_evaluate): n_steps x { obs -> actor -> greedy | sampled action -> env step (+ fused auto-reset) ->
// record of the episodes that end }.  The weights are fixed, so nothing couples the tiles: a CTA runs the whole window on one
// group of up to kSlots resident tiles, writes the group back and takes the next one (no limit on N).  The head outputs come
// from the device functions, template activation and operand scale of forward_tc_kernel's mode 1, so the staged greedy
// policy (b200rl_net_act_greedy -> nn_mlp_forward) and this kernel pick the same actions bit for bit.
template <class Env> struct EvalSlot {     // env state of one tile, one entry per env (owner thread = sample s)
    typename Env::S st[TM];
    int t[TM];
    int flags[TM];
    float ep_ret[TM];
    float last_rew[TM];
    uint32_t last_act[TM];
    int cnt[TM];                           // episodes finished in the window
    unsigned long long erng[4 * TM];       // env stream  [word][env]
    unsigned long long prng[4 * TM];       // policy stream (MODE 1)
};
template <class Env> struct SmemEval {
    alignas(128) uint8_t T[TILE_BYTES];
    NetSm net;                             // actor (or Q-network)
    float X[kInMax * TM];
    float Zp[2 * kOutMax * TM];            // [half][o][s]
    EvalSlot<Env> slot[kSlots];
    int fin_cnt[TM], fin_len[TM];          // episode statistics of owner thread s (shared memory: no registers held across the window)
    float fin_ret[TM];
    float red_f[8];
    int red_i[8], red_l[8];
};

struct EvalArgs {
    MlpDesc actor;
    const float* params;
    AcHyper hp;
    int64_t N;
    int nsteps, K;
    float act_lo, act_hi;               // continuous actions: the env receives clamp(a, lo, hi)
    unsigned long long* policy_rng;     // (4, N), MODE 1
    float* returns;                     // (K, N), may be null
    int32_t* lengths;                   // (K, N), may be null
    int32_t* counts;                    // (N), may be null
};

// MODE 0: greedy (greedy.cuh, no draw), 1: sample_head on the policy streams.  DUEL (MODE 0 only): a dueling Q-network, its head
// rows combined into Q (duel.cuh) before the selection; the instantiations without it are the code of the other kinds.
// (layer 1 and the head epilogue not unrolled: the relu variants would exceed 128 registers and spill)
template <class Env, int ACT, int MODE, bool DUEL = false>
__global__ void __launch_bounds__(NT, 2) evaluate_tc_kernel(EvalArgs g, typename Env::P p, EnvArrays ea) {
    using act_t = typename Env::act_t;
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
    for (int64_t base = blockIdx.x; base < ntiles; base += (int64_t)nctas * kSlots) {   // tiles base + k * nctas, k < kSlots
        int nslots = 0;
        for (int k = 0; k < kSlots; ++k)
            if (base + (int64_t)k * nctas < ntiles) nslots = k + 1;
        if (owner) {
            for (int k = 0; k < nslots; ++k) {
                const int64_t i = (base + (int64_t)k * nctas) * TM + s;
                EvalSlot<Env>& sl = sm.slot[k];
                if (i < N) {
                    sl.st[s] = Env::load(ea.state, i);
                    sl.t[s] = ea.t[i];
                    sl.flags[s] = ea.flags[i];
                    sl.ep_ret[s] = ea.ep_ret[i];
                    sl.cnt[s] = 0;
                    Xo e = load_rng(ea.rng, i);
                    sl.erng[s] = e.s0; sl.erng[TM + s] = e.s1; sl.erng[2 * TM + s] = e.s2; sl.erng[3 * TM + s] = e.s3;
                    if (MODE == 1) {
                        unsigned long long pr[4];
                        load_rng32(g.policy_rng, i, pr);
                        sl.prng[s] = pr[0]; sl.prng[TM + s] = pr[1]; sl.prng[2 * TM + s] = pr[2]; sl.prng[3 * TM + s] = pr[3];
                    }
                }
            }
        }
        wg::fence_proxy_async();            // (the first pass: the weight image written by load_net, read by wgmma)
        __syncthreads();
#pragma unroll 1
        for (int step = 0; step < g.nsteps; ++step) {
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
                {
                    float x[kInMax];
#pragma unroll
                    for (int j = 0; j < kInMax; ++j) x[j] = sm.X[j * TM + s];
                    layer1_to_smem<ACT, 1>(sm.net, g.actor.act, x, c, s, sm.T);
                }
                wg::fence_proxy_async();
                __syncthreads();
                gemm_block(sm.T + c * BLK, sm.net, c);   // warpgroup c: samples 64c .. 64c+63
                __syncthreads();
                {
                    float zp[kOutMax];
                    head_partials<ACT, 1>(sm.net, g.actor.act, c, s, sm.T, zp);
#pragma unroll
                    for (int o = 0; o < kOutMax; ++o) sm.Zp[(c * kOutMax + o) * TM + s] = zp[o];
                }
                __syncthreads();   // (the next pass's X / tile image writes are ordered behind these reads by its first barrier)
                const int64_t i = (base + (int64_t)k * nctas) * TM + s;
                if (owner && i < N) {
                    EvalSlot<Env>& sl = sm.slot[k];
                    float z[kOutMax];
#pragma unroll
                    for (int o = 0; o < kOutMax; ++o) z[o] = sm.net.b3[o] + sm.Zp[o * TM + s] + sm.Zp[(kOutMax + o) * TM + s];
                    if (DUEL) duel::combine(z, g.actor.nout);
                    uint32_t a_bits;
                    if (MODE == 0) {
                        a_bits = greedy::greedy_action(g.actor, z);
                    } else {
                        unsigned long long pr[4] = {sl.prng[s], sl.prng[TM + s], sl.prng[2 * TM + s], sl.prng[3 * TM + s]};
                        float lp;
                        a_bits = sample_head(g.actor, g.hp, z, pr, lp);
                        sl.prng[s] = pr[0]; sl.prng[TM + s] = pr[1]; sl.prng[2 * TM + s] = pr[2]; sl.prng[3 * TM + s] = pr[3];
                    }
                    // act!(env, a) + fused soft reset: the sequence of env_step_kernel<Env, false, true> (and rollout_tc_kernel)
                    act_t act;
                    if (std::is_same<act_t, float>::value) act = (act_t)fminf(fmaxf(__uint_as_float(a_bits), g.act_lo), g.act_hi);
                    else act = (act_t)(int32_t)a_bits;
                    typename Env::S st = sl.st[s];
                    int tt = sl.t[s];
                    const int prev = sl.flags[s];
                    bool done;
                    float rew;
                    Env::step(p, st, tt, act, done, rew);
                    if (ea.max_timeout > 0 && tt + 1 > ea.max_timeout) done = true;
                    float ret = sl.ep_ret[s] + rew;
                    int f = done ? 1 : 0;
                    if (done && !((prev & 1) && !(prev & 2))) { sm.fin_cnt[s] += 1; sm.fin_ret[s] += ret; sm.fin_len[s] += tt; }
                    if (done) {
                        const int e = sl.cnt[s];   // record of the episode that ends: its return and env.t
                        if (e < g.K) {
                            if (g.returns) g.returns[(size_t)g.K * i + e] = ret;
                            if (g.lengths) g.lengths[(size_t)g.K * i + e] = tt;
                        }
                        sl.cnt[s] = e + 1;
                        ret = 0.f;
                        Xo ex{sl.erng[s], sl.erng[TM + s], sl.erng[2 * TM + s], sl.erng[3 * TM + s]};
                        Env::reset(p, st, ex, act);
                        sl.erng[s] = ex.s0; sl.erng[TM + s] = ex.s1; sl.erng[2 * TM + s] = ex.s2; sl.erng[3 * TM + s] = ex.s3;
                        tt = 0;
                        f = 3;
                    }
                    sl.st[s] = st; sl.t[s] = tt; sl.flags[s] = f; sl.ep_ret[s] = ret;
                    sl.last_rew[s] = rew;
                    { act_t tmp = act; uint32_t bits; memcpy(&bits, &tmp, 4); sl.last_act[s] = bits; }
                }
            }
        }
        // ---- write the group back (each owner thread touches only its own entries: no barrier before the next group's loads)
        if (owner) {
            for (int k = 0; k < nslots; ++k) {
                const int64_t i = (base + (int64_t)k * nctas) * TM + s;
                EvalSlot<Env>& sl = sm.slot[k];
                if (i < N) {
                    Env::store(ea.state, i, sl.st[s]);
                    if (!Env::kObsIsState) Env::write_obs(ea.obs, i, N, sl.st[s]);
                    ea.t[i] = sl.t[s];
                    ea.flags[i] = (uint8_t)sl.flags[s];
                    ea.ep_ret[i] = sl.ep_ret[s];
                    store_rng(ea.rng, i, Xo{sl.erng[s], sl.erng[TM + s], sl.erng[2 * TM + s], sl.erng[3 * TM + s]});
                    if (MODE == 1) {
                        unsigned long long pr[4] = {sl.prng[s], sl.prng[TM + s], sl.prng[2 * TM + s], sl.prng[3 * TM + s]};
                        store_rng32(g.policy_rng, i, pr);
                    }
                    reinterpret_cast<float*>(ea.reward)[i] = sl.last_rew[s];
                    reinterpret_cast<uint32_t*>(ea.action)[i] = sl.last_act[s];
                    if (g.counts) g.counts[i] = sl.cnt[s];
                }
            }
        }
    }
    // episode statistics: one atomicAdd triple per CTA
    {
        int fin_cnt = owner ? sm.fin_cnt[s] : 0, fin_len = owner ? sm.fin_len[s] : 0;
        float fin_ret = owner ? sm.fin_ret[s] : 0.f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            fin_cnt += __shfl_xor_sync(0xffffffffu, fin_cnt, o);
            fin_len += __shfl_xor_sync(0xffffffffu, fin_len, o);
            fin_ret += __shfl_xor_sync(0xffffffffu, fin_ret, o);
        }
        __syncthreads();
        if (lane == 0) { sm.red_i[warp] = fin_cnt; sm.red_f[warp] = fin_ret; sm.red_l[warp] = fin_len; }
        __syncthreads();
        if (tid == 0) {
            double cc = 0, rr = 0, ll = 0;
            for (int w = 0; w < NT / 32; ++w) { cc += sm.red_i[w]; rr += sm.red_f[w]; ll += sm.red_l[w]; }
            if (cc > 0) { atomicAdd(&ea.stats[0], cc); atomicAdd(&ea.stats[1], rr); atomicAdd(&ea.stats[2], ll); }
        }
    }
}

template <class Env> int launch_evaluate(b200rl_ctx* ctx, const EvalArgs& g, const typename Env::P& p, const EnvArrays& ea, int mode) {
    const size_t smem = sizeof(SmemEval<Env>) + 128;
    static unsigned long long attr_devices = 0;   // once per device
    if (first_use_on_device(attr_devices, ctx->device)) {
        CUDA_TRY(cudaFuncSetAttribute(evaluate_tc_kernel<Env, B200RL_ACT_RELU, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(evaluate_tc_kernel<Env, B200RL_ACT_TANH, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(evaluate_tc_kernel<Env, B200RL_ACT_RELU, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(evaluate_tc_kernel<Env, B200RL_ACT_TANH, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(evaluate_tc_kernel<Env, B200RL_ACT_RELU, 0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(evaluate_tc_kernel<Env, B200RL_ACT_TANH, 0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    const int64_t groups = ((g.N + TM - 1) / TM + kSlots - 1) / kSlots;
    int grid = 2 * ctx->sm_count;
    if ((int64_t)grid > groups) grid = (int)groups;
    const bool relu = g.actor.act == B200RL_ACT_RELU;
    if (mode == 0 && g.actor.duel) {
        if (relu) evaluate_tc_kernel<Env, B200RL_ACT_RELU, 0, true><<<grid, NT, smem, ctx->stream>>>(g, p, ea);
        else evaluate_tc_kernel<Env, B200RL_ACT_TANH, 0, true><<<grid, NT, smem, ctx->stream>>>(g, p, ea);
    } else if (mode == 0) {
        if (relu) evaluate_tc_kernel<Env, B200RL_ACT_RELU, 0><<<grid, NT, smem, ctx->stream>>>(g, p, ea);
        else evaluate_tc_kernel<Env, B200RL_ACT_TANH, 0><<<grid, NT, smem, ctx->stream>>>(g, p, ea);
    } else {
        if (relu) evaluate_tc_kernel<Env, B200RL_ACT_RELU, 1><<<grid, NT, smem, ctx->stream>>>(g, p, ea);
        else evaluate_tc_kernel<Env, B200RL_ACT_TANH, 1><<<grid, NT, smem, ctx->stream>>>(g, p, ea);
    }
    LAUNCH_CHECK(ctx);
    return B200RL_OK;
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
template <class Env> struct ReplaySlot {
    typename Env::S st[TM];
    int t[TM];
    int flags[TM];
    float ep_ret[TM];
    float last_rew[TM];
    int32_t last_act[TM];
    int p0[TM];                            // slot of the first touched leaf of the lane (head - 1 at the start)
    int adv[TM];                           // frames written in the window
    unsigned long long erng[4 * TM];       // env stream      [word][env]
    unsigned long long xrng[4 * TM];       // explorer stream [word][env]
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
    float red_f[8];
    int red_i[8], red_l[8];
    long long red_v[8];
};
// b200rl_explorer without its trailing beta, which the kernel takes as its last parameter: the parameters the ϵ-greedy
// instantiations read keep the offsets they had before the explorer struct grew
struct ReplayExplorer {
    double eps_stable, eps_init;
    int64_t warmup_steps, decay_steps, step;
    int32_t kind, is_break_tie;
};
struct ReplayArgs {
    MlpDesc q;
    const float* params;
    int64_t N;
    int nsteps;
    int greedy;                            // 1: GreedyExplorer (findmax with `>`, no draw)
    ReplayExplorer ex;
    const long long* step_dev;             // explorer step before the window (device)
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
// instantiations without it compile the ϵ-greedy kinds 0 / 1 only.
template <class Env, int ACT, bool DUEL = false, bool XEXT = false>
__global__ void __launch_bounds__(NT, 2) replay_collect_tc_kernel(ReplayArgs g, typename Env::P p, EnvArrays ea, double beta) {
    using act_t = typename Env::act_t;
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
        int nslots = 0;
        for (int k = 0; k < kSlots; ++k)
            if (base + (int64_t)k * nctas < ntiles) nslots = k + 1;
        if (owner) {
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
                        load_rng32(g.xrng, i, xr);
                        sl.xrng[s] = xr[0]; sl.xrng[TM + s] = xr[1]; sl.xrng[2 * TM + s] = xr[2]; sl.xrng[3 * TM + s] = xr[3];
                    }
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
                {
                    float x[kInMax];
#pragma unroll
                    for (int j = 0; j < kInMax; ++j) x[j] = sm.X[j * TM + s];
                    layer1_to_smem<ACT, 1>(sm.net, g.q.act, x, c, s, sm.T);
                }
                wg::fence_proxy_async();
                __syncthreads();
                gemm_block(sm.T + c * BLK, sm.net, c);
                __syncthreads();
                {
                    float zp[kOutMax];
                    head_partials<ACT, 1>(sm.net, g.q.act, c, s, sm.T, zp);
#pragma unroll
                    for (int o = 0; o < kOutMax; ++o) sm.Zp[(c * kOutMax + o) * TM + s] = zp[o];
                }
                __syncthreads();
                const int64_t i = (base + (int64_t)k * nctas) * TM + s;
                if (owner && i < N) {
                    ReplaySlot<Env>& sl = sm.slot[k];
                    float z[kOutMax];
#pragma unroll
                    for (int o = 0; o < kOutMax; ++o) z[o] = sm.net.b3[o] + sm.Zp[o * TM + s] + sm.Zp[(kOutMax + o) * TM + s];
                    if (DUEL) duel::combine(z, g.q.nout);
                    int a1;
                    if (g.greedy) {
                        int best = 0;      // q_act_kernel with epsilon = 0: the first maximum under `>`
                        for (int o = 1; o < g.q.nout; ++o) if (z[o] > z[best]) best = o;
                        a1 = best + 1;
                    } else {
                        unsigned long long xr[4] = {sl.xrng[s], sl.xrng[TM + s], sl.xrng[2 * TM + s], sl.xrng[3 * TM + s]};
                        if constexpr (XEXT) {
                            const b200rl_explorer ex{g.ex.eps_stable, g.ex.eps_init, g.ex.warmup_steps, g.ex.decay_steps, g.ex.step, g.ex.kind,
                                                     g.ex.is_break_tie, beta};
                            a1 = explore::select<true>(ex, step0 + (long long)step * N + i, z, g.q.nout, xr);
                        } else {
                            a1 = explore::select<false>(g.ex, step0 + (long long)step * N + i, z, g.q.nout, xr);
                        }
                        sl.xrng[s] = xr[0]; sl.xrng[TM + s] = xr[1]; sl.xrng[2 * TM + s] = xr[2]; sl.xrng[3 * TM + s] = xr[3];
                    }
                    // act!(env, a) + fused auto-reset: the sequence of env_step_kernel<Env, false, true>
                    act_t act = (act_t)a1;
                    typename Env::S st = sl.st[s];
                    int tt = sl.t[s];
                    const int prev = sl.flags[s];
                    bool done;
                    float rew;
                    Env::step(p, st, tt, act, done, rew);
                    if (ea.max_timeout > 0 && tt + 1 > ea.max_timeout) done = true;
                    float ret = sl.ep_ret[s] + rew;
                    int f = done ? 1 : 0;
                    if (done && !((prev & 1) && !(prev & 2))) { sm.fin_cnt[s] += 1; sm.fin_ret[s] += ret; sm.fin_len[s] += tt; }
                    if (done) {
                        ret = 0.f;
                        Xo ex{sl.erng[s], sl.erng[TM + s], sl.erng[2 * TM + s], sl.erng[3 * TM + s]};
                        Env::reset(p, st, ex, act);
                        sl.erng[s] = ex.s0; sl.erng[TM + s] = ex.s1; sl.erng[2 * TM + s] = ex.s2; sl.erng[3 * TM + s] = ex.s3;
                        tt = 0;
                        f = 3;
                    }
                    sl.st[s] = st; sl.t[s] = tt; sl.flags[s] = f; sl.ep_ret[s] = ret;
                    sl.last_rew[s] = rew;
                    sl.last_act[s] = (int32_t)act;
                    // push!(trajectory, (state = s', action, reward, terminal)) of lane i
                    float nobs[kInMax];
                    Env::observe(st, nobs);
                    RingLeaves lv;
                    int adv = 0;
                    sm.dv[s] += ring::push_sart(r, i, (int32_t)act, rew, (uint8_t)f, nobs, g.default_priority, lv, &adv);
                    sl.adv[s] += adv;
                    if (g.prioritized)
                        for (int j = 0; j < 3; ++j) if (lv.key[j] >= 0) r.tree[r.L + lv.key[j]] = lv.val[j];
                }
            }
        }
        if (owner) {
            for (int k = 0; k < nslots; ++k) {
                const int64_t i = (base + (int64_t)k * nctas) * TM + s;
                ReplaySlot<Env>& sl = sm.slot[k];
                if (i < N) {
                    Env::store(ea.state, i, sl.st[s]);
                    if (!Env::kObsIsState) Env::write_obs(ea.obs, i, N, sl.st[s]);
                    ea.t[i] = sl.t[s];
                    ea.flags[i] = (uint8_t)sl.flags[s];
                    ea.ep_ret[i] = sl.ep_ret[s];
                    store_rng(ea.rng, i, Xo{sl.erng[s], sl.erng[TM + s], sl.erng[2 * TM + s], sl.erng[3 * TM + s]});
                    if (!g.greedy) {
                        unsigned long long xr[4] = {sl.xrng[s], sl.xrng[TM + s], sl.xrng[2 * TM + s], sl.xrng[3 * TM + s]};
                        store_rng32(g.xrng, i, xr);
                    }
                    if (g.nsteps > 0) {
                        reinterpret_cast<float*>(ea.reward)[i] = sl.last_rew[s];
                        reinterpret_cast<int32_t*>(ea.action)[i] = sl.last_act[s];
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
                }
            }
        }
    }
    // episode statistics and the sampleable count: one atomic each per CTA
    {
        int fin_cnt = owner ? sm.fin_cnt[s] : 0, fin_len = owner ? sm.fin_len[s] : 0;
        float fin_ret = owner ? sm.fin_ret[s] : 0.f;
        long long dv = owner ? sm.dv[s] : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            fin_cnt += __shfl_xor_sync(0xffffffffu, fin_cnt, o);
            fin_len += __shfl_xor_sync(0xffffffffu, fin_len, o);
            fin_ret += __shfl_xor_sync(0xffffffffu, fin_ret, o);
            dv += __shfl_xor_sync(0xffffffffu, dv, o);
        }
        __syncthreads();
        if (lane == 0) { sm.red_i[warp] = fin_cnt; sm.red_f[warp] = fin_ret; sm.red_l[warp] = fin_len; sm.red_v[warp] = dv; }
        __syncthreads();
        if (tid == 0) {
            double cc = 0, rr = 0, ll = 0;
            long long vv = 0;
            for (int w = 0; w < NT / 32; ++w) { cc += sm.red_i[w]; rr += sm.red_f[w]; ll += sm.red_l[w]; vv += sm.red_v[w]; }
            if (cc > 0) { atomicAdd(&ea.stats[0], cc); atomicAdd(&ea.stats[1], rr); atomicAdd(&ea.stats[2], ll); }
            if (vv != 0) atomicAdd((unsigned long long*)r.n_valid, (unsigned long long)vv);
        }
    }
}

template <class Env, bool XEXT> int launch_replay_collect_x(b200rl_ctx* ctx, const ReplayArgs& g, const typename Env::P& p, const EnvArrays& ea,
                                                           double beta) {
    const size_t smem = sizeof(SmemReplay<Env>) + 128;
    static unsigned long long attr_devices = 0;   // once per device (and per XEXT)
    if (first_use_on_device(attr_devices, ctx->device)) {
        CUDA_TRY(cudaFuncSetAttribute(replay_collect_tc_kernel<Env, B200RL_ACT_RELU, false, XEXT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(replay_collect_tc_kernel<Env, B200RL_ACT_TANH, false, XEXT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(replay_collect_tc_kernel<Env, B200RL_ACT_RELU, true, XEXT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(replay_collect_tc_kernel<Env, B200RL_ACT_TANH, true, XEXT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    const int64_t groups = ((g.N + TM - 1) / TM + kSlots - 1) / kSlots;
    int grid = 2 * ctx->sm_count;
    if ((int64_t)grid > groups) grid = (int)groups;
    if (g.q.duel) {
        if (g.q.act == B200RL_ACT_RELU) replay_collect_tc_kernel<Env, B200RL_ACT_RELU, true, XEXT><<<grid, NT, smem, ctx->stream>>>(g, p, ea, beta);
        else replay_collect_tc_kernel<Env, B200RL_ACT_TANH, true, XEXT><<<grid, NT, smem, ctx->stream>>>(g, p, ea, beta);
    } else if (g.q.act == B200RL_ACT_RELU) replay_collect_tc_kernel<Env, B200RL_ACT_RELU, false, XEXT><<<grid, NT, smem, ctx->stream>>>(g, p, ea, beta);
    else replay_collect_tc_kernel<Env, B200RL_ACT_TANH, false, XEXT><<<grid, NT, smem, ctx->stream>>>(g, p, ea, beta);
    LAUNCH_CHECK(ctx);
    return B200RL_OK;
}
template <class Env> int launch_replay_collect(b200rl_ctx* ctx, const ReplayArgs& g, const typename Env::P& p, const EnvArrays& ea, double beta) {
    if (!g.greedy && g.ex.kind >= 2) return launch_replay_collect_x<Env, true>(ctx, g, p, ea, beta);
    return launch_replay_collect_x<Env, false>(ctx, g, p, ea, 0.0);
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
    if (!(nn_tc_supported(actor) && nn_tc_supported(critic)) || critic.nout != 1 || v.dtype != B200RL_F32) return B200RL_ERR_UNSUPPORTED;
    if (actor.act != critic.act) return B200RL_ERR_UNSUPPORTED;   // the fused kernel is compiled per activation (staged launches handle a mixed pair)
    const int64_t ntiles = (v.N + TM - 1) / TM;
    if (ntiles > (int64_t)kSlots * 2 * ctx->sm_count) return B200RL_ERR_UNSUPPORTED;
    if ((actor.heads2 != 0) != (v.continuous != 0)) return B200RL_ERR_UNSUPPORTED;   // Gaussian head <-> continuous action space
    RollArgs g{actor, critic, params, hp, v.N, t0, nsteps, T, final_bootstrap, -1.0f, 1.0f, policy_rng, states, actions, logp, values, rewards, terminals};
    int st = B200RL_ERR_UNSUPPORTED;
    switch (v.kind) {
        case B200RL_ENV_CARTPOLE:
            if (v.continuous) {
                CartPoleD<float, true>::P q;
                memcpy(&q, &v.p.cp32, sizeof q);
                st = launch_rollout<CartPoleD<float, true>>(ctx, g, q, v.a);
            } else {
                if (actor.nout != 2) return B200RL_ERR_UNSUPPORTED;
                st = launch_rollout<CartPoleD<float, false>>(ctx, g, v.p.cp32, v.a);
            }
            break;
        case B200RL_ENV_PENDULUM:
            if (v.continuous) {
                g.act_lo = -2.0f; g.act_hi = 2.0f;      // PendulumEnv.jl:73: action_space -2.0..2.0
                st = launch_rollout<PendulumD<true>>(ctx, g, v.p.pend, v.a);
            } else {
                if (actor.nout != v.p.pend.n_actions) return B200RL_ERR_UNSUPPORTED;
                st = launch_rollout<PendulumD<false>>(ctx, g, v.p.pend, v.a);
            }
            break;
        case B200RL_ENV_MOUNTAINCAR:
            if (v.continuous) {
                MountainCarD<true>::P q;
                memcpy(&q, &v.p.mc, sizeof q);
                st = launch_rollout<MountainCarD<true>>(ctx, g, q, v.a);
            } else {
                if (actor.nout != 3) return B200RL_ERR_UNSUPPORTED;
                st = launch_rollout<MountainCarD<false>>(ctx, g, v.p.mc, v.a);
            }
            break;
    }
    if (st == B200RL_OK) b200rl_env_internal_add_steps(env, (uint64_t)nsteps);
    return st;
}

// Fused evaluation window (after the caller's forced reset).  The caller has validated net <-> env; B200RL_ERR_UNSUPPORTED
// (no side effect, no error message) = outside the fused envelope: the caller steps through staged launches instead.
int nn_tc_evaluate(b200rl_ctx* ctx, b200rl_env* env, const MlpDesc& actor, const float* params, const AcHyper& hp, int mode, int nsteps,
                   int K, unsigned long long* policy_rng, float* returns, int32_t* lengths, int32_t* counts) {
    EnvView v;
    TRY(b200rl_env_internal_view(env, &v));
    if (!nn_tc_supported(actor) || v.dtype != B200RL_F32) return B200RL_ERR_UNSUPPORTED;
    EvalArgs g{actor, params, hp, v.N, nsteps, K, -1.0f, 1.0f, policy_rng, returns, lengths, counts};
    int st = B200RL_ERR_UNSUPPORTED;
    switch (v.kind) {
        case B200RL_ENV_CARTPOLE:
            if (v.continuous) {
                CartPoleD<float, true>::P q;
                memcpy(&q, &v.p.cp32, sizeof q);
                st = launch_evaluate<CartPoleD<float, true>>(ctx, g, q, v.a, mode);
            } else {
                st = launch_evaluate<CartPoleD<float, false>>(ctx, g, v.p.cp32, v.a, mode);
            }
            break;
        case B200RL_ENV_PENDULUM:
            if (v.continuous) {
                g.act_lo = -2.0f; g.act_hi = 2.0f;      // PendulumEnv.jl:73: action_space -2.0..2.0
                st = launch_evaluate<PendulumD<true>>(ctx, g, v.p.pend, v.a, mode);
            } else {
                st = launch_evaluate<PendulumD<false>>(ctx, g, v.p.pend, v.a, mode);
            }
            break;
        case B200RL_ENV_MOUNTAINCAR:
            if (v.continuous) {
                MountainCarD<true>::P q;
                memcpy(&q, &v.p.mc, sizeof q);
                st = launch_evaluate<MountainCarD<true>>(ctx, g, q, v.a, mode);
            } else {
                st = launch_evaluate<MountainCarD<false>>(ctx, g, v.p.mc, v.a, mode);
            }
            break;
    }
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
    if (!nn_tc_supported(q) || v.dtype != B200RL_F32 || v.continuous || ring.ns > kInMax) return B200RL_ERR_UNSUPPORTED;
    const b200rl_explorer e = ex ? *ex : b200rl_explorer{};
    ReplayArgs g{q, params, v.N, nsteps, ex ? 0 : 1, ReplayExplorer{e.eps_stable, e.eps_init, e.warmup_steps, e.decay_steps, e.step, e.kind, e.is_break_tie},
                 step_dev, xrng, ring, default_priority, prioritized, keys, vals, stride};
    int st = B200RL_ERR_UNSUPPORTED;
    switch (v.kind) {
        case B200RL_ENV_CARTPOLE: st = launch_replay_collect<CartPoleD<float, false>>(ctx, g, v.p.cp32, v.a, e.beta); break;
        case B200RL_ENV_PENDULUM: st = launch_replay_collect<PendulumD<false>>(ctx, g, v.p.pend, v.a, e.beta); break;
        case B200RL_ENV_MOUNTAINCAR: st = launch_replay_collect<MountainCarD<false>>(ctx, g, v.p.mc, v.a, e.beta); break;
    }
    if (st == B200RL_OK) b200rl_env_internal_add_steps(env, (uint64_t)nsteps);
    return st;
}
