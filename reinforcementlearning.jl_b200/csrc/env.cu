// env.cu — K1/K2: batched classic-control env step, reset and fused random policy.
//
// One thread per env, 256 threads per CTA.  State is (NS, N) column-major so one env's state
// is one 16-byte (Float32 CartPole: float4) or 8-byte vector; reward/flags/t are SoA vectors;
// the per-env Xoshiro256++ state is 32 B AoS and is only touched by threads that draw.
// Arithmetic follows the reference line by line with Julia's promotion rules (which
// sub-expressions are Float64 for T = Float32) — see DESIGN.md §K1 and
//   RLEnvs/src/environments/examples/CartPoleEnv.jl:98-140
//   RLEnvs/src/environments/examples/PendulumEnv.jl:84-122
//   RLEnvs/src/environments/examples/MountainCarEnv.jl:99-135
// Compiled with -fmad=false (no contraction; Julia never contracts) and IEEE div.
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "env_device.cuh"
#include "internal.h"

using jld::Xo;
using namespace envdev;

namespace {

constexpr int kBlock = 256;

// ------------------------------------------------------------------ kernels -----------
// LOG: a finished episode is also written to the env's episode log (EnvArraysLog)
template <class Env, bool RANDOM, bool AUTO, bool LOG>
__global__ void __launch_bounds__(kBlock) env_step_kernel(typename Env::P p, EnvArgs<LOG> a, int64_t N, const void* actions_v) {
    using T = typename Env::real;
    using act_t = typename Env::act_t;
    __shared__ StatsScratch<kBlock / 32> red;
    int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
    bool active = i < N;
    int fin_cnt = 0, fin_len = 0;
    float fin_ret = 0.f;
    if (active) {
        typename Env::S s = Env::load(a.state, i);
        int t = a.t[i];
        int f = a.flags[i];
        Xo g;
        bool have_rng = false;
        act_t act;
        bool ok = true;
        if (RANDOM) {  // plan!(RandomPolicy): rand(rng, Base.OneTo(n)) on the env's own stream
            g = load_rng(a.rng, i);
            have_rng = true;
            act = Env::from_index(p, jld::rand_oneto(g, Env::n_random(p)));
        } else {
            act = reinterpret_cast<const act_t*>(actions_v)[i];
            ok = Env::valid(p, act);
            if (!ok) *a.err = 1;  // `@assert a in action_space(env)` -> flag, env left untouched
        }
        if (ok) {
            float ret = a.ep_ret[i];
            const ActStep<T> r = act_step<Env, AUTO, LOG>(p, a.max_timeout, s, t, f, ret, act, fin_cnt, fin_ret, fin_len, [&](auto&& reset) {
                if (!have_rng) { g = load_rng(a.rng, i); have_rng = true; }
                reset(g);
            }, episode_log_of(a), i);
            Env::store(a.state, i, s);
            if (!Env::kObsIsState) Env::write_obs(a.obs, i, N, s);
            store_obs_f32<Env>(a, i, N, s);
            a.t[i] = t;
            a.flags[i] = (uint8_t)f;
            reinterpret_cast<T*>(a.reward)[i] = r.rew;
            reinterpret_cast<act_t*>(a.action)[i] = act;
            a.ep_ret[i] = ret;
            if (a.traj_reward) reinterpret_cast<float*>(a.traj_reward)[i] = (float)r.rew;   // the rollout's Float32 reward
            if (a.traj_terminal) a.traj_terminal[i] = r.done ? 1 : 0;
        }
        if (have_rng) store_rng(a.rng, i, g);
    }
    cta_episode_stats(a.stats, fin_cnt, fin_ret, fin_len, red);
}

// envs whose reset! also sets the reward field (AcrobotEnv.jl:105: env.reward = -1); the others derive reward(env) from `done`
template <class Env> struct ResetReward { static constexpr bool set = false; static __device__ double value() { return 0.0; } };
template <> struct ResetReward<AcrobotD> { static constexpr bool set = true; static __device__ double value() { return -1.0; } };

template <class Env>
__global__ void __launch_bounds__(kBlock) env_reset_kernel(typename Env::P p, EnvArrays a, int64_t N, int force) {
    using act_t = typename Env::act_t;
    int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
    if (i >= N) return;
    uint8_t f = a.flags[i];
    if (force || ((f & 1) && !(f & 2))) {
        typename Env::S s = Env::load(a.state, i);
        Xo g = load_rng(a.rng, i);
        act_t act = reinterpret_cast<act_t*>(a.action)[i];
        Env::reset(p, s, g, act);
        store_rng(a.rng, i, g);
        Env::store(a.state, i, s);
        if (!Env::kObsIsState) Env::write_obs(a.obs, i, N, s);
        store_obs_f32<Env>(a, i, N, s);
        a.t[i] = 0;
        reinterpret_cast<act_t*>(a.action)[i] = act;
        a.ep_ret[i] = 0.f;
        if (ResetReward<Env>::set) reinterpret_cast<typename Env::real*>(a.reward)[i] = (typename Env::real)ResetReward<Env>::value();
    }
    a.flags[i] = 0;
}

// Float32(x) of n doubles: the observation mirror after env_set, the Float32 reward a trajectory push reads
__global__ void narrow_f64_kernel(float* __restrict__ dst, const double* __restrict__ src, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
    if (i < n) dst[i] = (float)src[i];
}

// ------------------------------------------------------------------ episode log flush --
// One flush turns the records every env logged since the previous flush into one list ordered by (env, episode): the pending
// counts of each CTA (log_count_kernel), an exclusive scan of the CTA totals (log_offsets_kernel), and each env's records written at
// its offset (log_scatter_kernel), which recomputes the in-CTA prefix.  The list goes straight to the caller's pinned host buffer.

// pending records of env i (0 past N); an env with more than K counts as overflowing (overflow != null) and contributes K
__device__ __forceinline__ uint32_t flush_pending(const EpisodeLog& log, const uint32_t* cursor, int64_t i, int64_t N,
                                                  unsigned long long* overflow) {
    if (i >= N) return 0;
    uint32_t n = log_pending(log, cursor, i);
    if (n > (uint32_t)log.K) {
        if (overflow) atomicAdd(overflow, 1ull);
        n = (uint32_t)log.K;
    }
    return n;
}
// exclusive prefix of v over the CTA: a warp-shuffle scan, then the warp totals; *total is the CTA's sum.  Every thread calls it.
__device__ __forceinline__ long long cta_exclusive_scan(long long v, long long (&warp_tot)[kBlock / 32], long long* total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_tot[w] = x;
    __syncthreads();
    long long before = 0, all = 0;
#pragma unroll
    for (int k = 0; k < kBlock / 32; ++k) {
        if (k < w) before += warp_tot[k];
        all += warp_tot[k];
    }
    __syncthreads();   // (warp_tot may be rewritten by the caller's next scan)
    *total = all;
    return before + x - v;
}

__global__ void __launch_bounds__(kBlock) log_count_kernel(EpisodeLog log, const uint32_t* __restrict__ cursor, int64_t N,
                                                           long long* __restrict__ cta_tot, unsigned long long* overflow) {
    __shared__ long long warp_tot[kBlock / 32];
    const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
    long long total;
    cta_exclusive_scan(flush_pending(log, cursor, i, N, overflow), warp_tot, &total);
    if (threadIdx.x == 0) cta_tot[blockIdx.x] = total;
}

// one CTA: cta_tot[0 .. nb) -> exclusive offsets in place; hdr = {list length, overflowing envs}; the overflow counter is cleared
__global__ void __launch_bounds__(kBlock) log_offsets_kernel(long long* __restrict__ cta_tot, int64_t nb, unsigned long long* overflow,
                                                             long long* hdr) {
    __shared__ long long warp_tot[kBlock / 32];
    long long carry = 0;
    for (int64_t b0 = 0; b0 < nb; b0 += kBlock) {
        const int64_t b = b0 + threadIdx.x;
        long long total;
        const long long ex = cta_exclusive_scan(b < nb ? cta_tot[b] : 0, warp_tot, &total);
        if (b < nb) cta_tot[b] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) {
        hdr[0] = carry;
        hdr[1] = (long long)*overflow;
        *overflow = 0;
    }
}

__global__ void __launch_bounds__(kBlock) log_scatter_kernel(EpisodeLog log, uint32_t* __restrict__ cursor, int64_t N,
                                                             const long long* __restrict__ cta_off, int64_t global0, EpisodeRecord* out,
                                                             int64_t capacity) {
    __shared__ long long warp_tot[kBlock / 32];
    const int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
    const uint32_t n = flush_pending(log, cursor, i, N, nullptr);
    long long total;
    const long long off = cta_off[blockIdx.x] + cta_exclusive_scan(n, warp_tot, &total);
    if (i < N) {
        if (n) log_emit(log, cursor, i, n, global0 + i, out + off, capacity - off);
        cursor[i] = log.count[i];
    }
}

}  // namespace

// ------------------------------------------------------------------ handle ------------
struct b200rl_env {
    b200rl_ctx* ctx;
    int kind, dtype;
    int64_t N;
    int ns, nobs;
    bool continuous;
    size_t tsize;
    union {
        CartPoleD<float>::P cp32;
        CartPoleD<double>::P cp64;
        PendP pend;
        MountainCarD<false>::P mc;
        PendPT<double> pend64;
        MountainCarPT<double> mc64;
        AcrobotP acro;
    } p;
    size_t asize;   // bytes per stored action (8 for a Float64 continuous action space, else 4)
    bool state_f32;   // StateTransformedEnv(env; state_mapping = s -> Float32.(s)): the learners read the Float32 mirror
    float* rew_f32;   // (N) Float32(reward) for the trajectory pushes of a Float64 env (null for the others)
    EnvArrays a;
    uint64_t steps_launched;
    // episode log (b200rl_env_episode_log): the device ring (written by the env's steps unless a staged evaluation holds it off);
    // the flush keeps each env's read position, its scan scratch (CTA totals, then the overflow counter) and the last flush into
    // each buffer
    EpisodeLog log_ring;
    bool log_held;
    uint32_t* log_cursor;
    long long* log_scratch;
    struct LogFlush { const void* buf; int64_t capacity; cudaEvent_t done; };
    std::vector<LogFlush> log_flushes;
};

static void log_free(b200rl_env* e) {
    if (e->log_ring.count) cudaStreamSynchronize(e->ctx->stream);
    cudaFree(e->log_ring.ret); cudaFree(e->log_ring.len); cudaFree(e->log_ring.count);
    cudaFree(e->log_cursor); cudaFree(e->log_scratch);
    for (auto& f : e->log_flushes) cudaEventDestroy(f.done);
    e->log_flushes.clear();
    e->log_ring = EpisodeLog{};
    e->log_cursor = nullptr;
    e->log_scratch = nullptr;
}

// the episode log the env's steps write: none while a staged evaluation holds it off
static EpisodeLog active_log(const b200rl_env* e) { return e->log_held ? EpisodeLog{} : e->log_ring; }

template <class Env, bool RANDOM, bool AUTO> static void launch_step_as(b200rl_env* e, const typename Env::P& p, const void* actions) {
    const unsigned grid = grid_for(e->N, kBlock);
    cudaStream_t st = e->ctx->stream;
    const EpisodeLog log = active_log(e);
    if (log.count) env_step_kernel<Env, RANDOM, AUTO, true><<<grid, kBlock, 0, st>>>(p, EnvArraysLog{e->a, log}, e->N, actions);
    else env_step_kernel<Env, RANDOM, AUTO, false><<<grid, kBlock, 0, st>>>(p, e->a, e->N, actions);
}
template <class Env> static int launch_step(b200rl_env* e, const typename Env::P& p, const void* actions, bool random, bool auto_reset) {
    if (random) {
        if (auto_reset) launch_step_as<Env, true, true>(e, p, nullptr);
        else launch_step_as<Env, true, false>(e, p, nullptr);
    } else {
        if (auto_reset) launch_step_as<Env, false, true>(e, p, actions);
        else launch_step_as<Env, false, false>(e, p, actions);
    }
    LAUNCH_CHECK(e->ctx);
    return B200RL_OK;
}
template <class Env> static int launch_reset(b200rl_env* e, const typename Env::P& p, int force) {
    env_reset_kernel<Env><<<grid_for(e->N, kBlock), kBlock, 0, e->ctx->stream>>>(p, e->a, e->N, force);
    LAUNCH_CHECK(e->ctx);
    return B200RL_OK;
}

static int dispatch_step(b200rl_env* e, const void* actions, bool random, bool auto_reset) {
    switch (e->kind) {
        case B200RL_ENV_CARTPOLE:
            if (e->dtype == B200RL_F64) return launch_step<CartPoleD<double>>(e, e->p.cp64, actions, random, auto_reset);
            if (e->continuous && !random) {
                CartPoleD<float, true>::P q;
                static_assert(sizeof(q) == sizeof(e->p.cp32), "same params layout");
                memcpy(&q, &e->p.cp32, sizeof q);
                return launch_step<CartPoleD<float, true>>(e, q, actions, random, auto_reset);
            }
            return launch_step<CartPoleD<float>>(e, e->p.cp32, actions, random, auto_reset);
        case B200RL_ENV_PENDULUM:
            if (e->dtype == B200RL_F64) {
                if (e->continuous && !random) return launch_step<PendulumD<true, double>>(e, e->p.pend64, actions, random, auto_reset);
                return launch_step<PendulumD<false, double>>(e, e->p.pend64, actions, random, auto_reset);
            }
            if (e->continuous && !random) return launch_step<PendulumD<true>>(e, e->p.pend, actions, random, auto_reset);
            return launch_step<PendulumD<false>>(e, e->p.pend, actions, random, auto_reset);
        case B200RL_ENV_MOUNTAINCAR:
            if (e->dtype == B200RL_F64) {
                if (e->continuous && !random) return launch_step<MountainCarD<true, double>>(e, e->p.mc64, actions, random, auto_reset);
                return launch_step<MountainCarD<false, double>>(e, e->p.mc64, actions, random, auto_reset);
            }
            if (e->continuous && !random) {
                MountainCarD<true>::P q;
                static_assert(sizeof(q) == sizeof(e->p.mc), "same params layout");
                memcpy(&q, &e->p.mc, sizeof q);
                return launch_step<MountainCarD<true>>(e, q, actions, random, auto_reset);
            }
            return launch_step<MountainCarD<false>>(e, e->p.mc, actions, random, auto_reset);
        case B200RL_ENV_ACROBOT:
            return launch_step<AcrobotD>(e, e->p.acro, actions, random, auto_reset);
    }
    return B200RL_ERR_INVALID;
}
static int dispatch_reset(b200rl_env* e, int force) {
    switch (e->kind) {
        case B200RL_ENV_CARTPOLE:
            if (e->dtype == B200RL_F64) return launch_reset<CartPoleD<double>>(e, e->p.cp64, force);
            if (e->continuous) {
                CartPoleD<float, true>::P q;
                memcpy(&q, &e->p.cp32, sizeof q);
                return launch_reset<CartPoleD<float, true>>(e, q, force);
            }
            return launch_reset<CartPoleD<float>>(e, e->p.cp32, force);
        case B200RL_ENV_PENDULUM:
            if (e->dtype == B200RL_F64)
                return e->continuous ? launch_reset<PendulumD<true, double>>(e, e->p.pend64, force) : launch_reset<PendulumD<false, double>>(e, e->p.pend64, force);
            return launch_reset<PendulumD<true>>(e, e->p.pend, force);
        case B200RL_ENV_MOUNTAINCAR:
            if (e->dtype == B200RL_F64)
                return e->continuous ? launch_reset<MountainCarD<true, double>>(e, e->p.mc64, force) : launch_reset<MountainCarD<false, double>>(e, e->p.mc64, force);
            return launch_reset<MountainCarD<false>>(e, e->p.mc, force);
        case B200RL_ENV_ACROBOT:
            return launch_reset<AcrobotD>(e, e->p.acro, force);
    }
    return B200RL_ERR_INVALID;
}

// a Float64 env other than Acrobot keeps the (NOBS, N) float mirror of its observation behind the observation (env_device.cuh)
static bool has_obs_f32(const b200rl_env* e) { return e->dtype == B200RL_F64 && e->kind != B200RL_ENV_ACROBOT; }
static float* obs_f32_ptr(const b200rl_env* e) {
    return has_obs_f32(e) ? reinterpret_cast<float*>(reinterpret_cast<double*>(e->a.obs) + (size_t)e->N * e->nobs) : (float*)e->a.obs;
}

static size_t field_bytes(const b200rl_env* e, int field) {
    size_t N = (size_t)e->N;
    switch (field) {
        case B200RL_FIELD_OBS_F32: return b200rl_env_internal_obs_f32(e) ? N * e->nobs * 4 : 0;
        case B200RL_FIELD_STATE: return N * e->ns * e->tsize;
        case B200RL_FIELD_OBS: return N * e->nobs * e->tsize;
        case B200RL_FIELD_REWARD: return N * e->tsize;
        case B200RL_FIELD_TERMINAL: case B200RL_FIELD_FLAGS: return N;
        case B200RL_FIELD_T: return N * 4;
        case B200RL_FIELD_RNG: return N * 32;
        case B200RL_FIELD_ACTION: return N * e->asize;
        case B200RL_FIELD_EPISODE_RETURN: return N * 4;
        case B200RL_FIELD_EPISODE_STATS: return 4 * sizeof(double);
    }
    return 0;
}
static void* field_ptr(const b200rl_env* e, int field) {
    switch (field) {
        case B200RL_FIELD_STATE: return e->a.state;
        case B200RL_FIELD_OBS: return e->a.obs;
        case B200RL_FIELD_REWARD: return e->a.reward;
        case B200RL_FIELD_TERMINAL: case B200RL_FIELD_FLAGS: return e->a.flags;
        case B200RL_FIELD_T: return e->a.t;
        case B200RL_FIELD_RNG: return e->a.rng;
        case B200RL_FIELD_ACTION: return e->a.action;
        case B200RL_FIELD_EPISODE_RETURN: return e->a.ep_ret;
        case B200RL_FIELD_EPISODE_STATS: return e->a.stats;
        case B200RL_FIELD_OBS_F32: return (void*)b200rl_env_internal_obs_f32(e);
    }
    return nullptr;
}

static int env_alloc(b200rl_env* e) {
    size_t N = (size_t)e->N;
    const size_t mirror = has_obs_f32(e) ? N * e->nobs * 4 : 0;   // the Float32 mirror behind the observation
    const bool own_obs = e->kind == B200RL_ENV_PENDULUM || e->kind == B200RL_ENV_ACROBOT;
    CUDA_TRY(cudaMalloc(&e->a.state, N * e->ns * e->tsize + (own_obs ? 0 : mirror)));
    if (own_obs) CUDA_TRY(cudaMalloc(&e->a.obs, N * e->nobs * e->tsize + mirror));
    else e->a.obs = e->a.state;
    if (mirror) {
        CUDA_TRY(cudaMalloc(&e->rew_f32, N * 4));
        CUDA_TRY(cudaMemsetAsync(obs_f32_ptr(e), 0, mirror, e->ctx->stream));
    }
    CUDA_TRY(cudaMalloc(&e->a.reward, N * e->tsize));
    CUDA_TRY(cudaMalloc(&e->a.flags, N));
    CUDA_TRY(cudaMalloc(&e->a.t, N * 4));
    CUDA_TRY(cudaMalloc(&e->a.rng, N * 32));
    CUDA_TRY(cudaMalloc(&e->a.action, N * 8));
    CUDA_TRY(cudaMalloc(&e->a.ep_ret, N * 4));
    CUDA_TRY(cudaMalloc(&e->a.stats, 4 * sizeof(double)));
    CUDA_TRY(cudaMalloc(&e->a.err, sizeof(int)));
    cudaStream_t st = e->ctx->stream;
    CUDA_TRY(cudaMemsetAsync(e->a.state, 0, N * e->ns * e->tsize, st));
    if (e->a.obs != e->a.state) CUDA_TRY(cudaMemsetAsync(e->a.obs, 0, N * e->nobs * e->tsize, st));
    CUDA_TRY(cudaMemsetAsync(e->a.reward, 0, N * e->tsize, st));
    CUDA_TRY(cudaMemsetAsync(e->a.flags, 0, N, st));
    CUDA_TRY(cudaMemsetAsync(e->a.t, 0, N * 4, st));
    CUDA_TRY(cudaMemsetAsync(e->a.action, 0, N * 8, st));
    CUDA_TRY(cudaMemsetAsync(e->a.ep_ret, 0, N * 4, st));
    CUDA_TRY(cudaMemsetAsync(e->a.stats, 0, 4 * sizeof(double), st));
    CUDA_TRY(cudaMemsetAsync(e->a.err, 0, sizeof(int), st));
    e->a.traj_reward = nullptr;
    e->a.traj_terminal = nullptr;
    return B200RL_OK;
}

extern "C" {

int b200rl_env_create(b200rl_ctx* ctx, int kind, int dtype, int64_t n_envs, const void* params,
                      const uint64_t* rng_state, b200rl_env** out) {
    TRY(ctx_bind(ctx));
    REQUIRE(out && rng_state, B200RL_ERR_INVALID, "null out / rng_state");
    REQUIRE(n_envs > 0, B200RL_ERR_INVALID, "n_envs must be positive");
    REQUIRE(dtype == B200RL_F32 || dtype == B200RL_F64, B200RL_ERR_INVALID, "dtype must be B200RL_F32 or B200RL_F64");
    b200rl_env* e = new b200rl_env();
    memset(&e->a, 0, sizeof e->a);
    bool cont_kind = kind == B200RL_ENV_CARTPOLE_CONTINUOUS || kind == B200RL_ENV_MOUNTAINCAR_CONTINUOUS;
    if (kind == B200RL_ENV_CARTPOLE_CONTINUOUS && dtype != B200RL_F32) { delete e; REQUIRE(false, B200RL_ERR_UNSUPPORTED, "CartPoleEnv(continuous = true) is Float32 only"); }
    if (kind == B200RL_ENV_CARTPOLE_CONTINUOUS) kind = B200RL_ENV_CARTPOLE;
    if (kind == B200RL_ENV_MOUNTAINCAR_CONTINUOUS) kind = B200RL_ENV_MOUNTAINCAR;
    e->ctx = ctx; e->kind = kind; e->dtype = dtype; e->N = n_envs; e->continuous = cont_kind;
    e->state_f32 = false; e->rew_f32 = nullptr;
    e->tsize = dtype == B200RL_F64 ? 8 : 4;
    e->steps_launched = 0;
    if (kind == B200RL_ENV_CARTPOLE) {
        b200rl_cartpole_params d;
        if (params) d = *(const b200rl_cartpole_params*)params;
        else if (dtype == B200RL_F64)
            d = b200rl_cartpole_params{9.8, 1.0, 0.1, 1.0 + 0.1, 0.5, 0.1 * 0.5, 10.0, 0.02, 12.0 * JLD_PI / 180, 2.4, 200};
        else
            d = b200rl_cartpole_params{(float)9.8, 1.0, (float)0.1, (float)(1.0 + 0.1), 0.5, (float)(0.1 * 0.5), 10.0, (float)0.02,
                                       (float)(12.0 * JLD_PI / 180), (float)2.4, 200};
        e->ns = 4; e->nobs = 4;
        if (dtype == B200RL_F64)
            e->p.cp64 = CartPoleD<double>::P{d.gravity, d.totalmass, d.masspole, d.halflength, d.polemasslength, d.forcemag, d.dt,
                                              d.thetathreshold, d.xthreshold, (int)d.max_steps};
        else
            e->p.cp32 = CartPoleD<float>::P{(float)d.gravity, (float)d.totalmass, (float)d.masspole, (float)d.halflength,
                                             (float)d.polemasslength, (float)d.forcemag, (float)d.dt, (float)d.thetathreshold,
                                             (float)d.xthreshold, (int)d.max_steps};
    } else if (kind == B200RL_ENV_PENDULUM) {
        b200rl_pendulum_params d = params ? *(const b200rl_pendulum_params*)params
                                          : b200rl_pendulum_params{8, 2, 10, 1, 1, (float)0.05, 200, 3, 1};
        REQUIRE(d.continuous || d.n_actions >= 2, B200RL_ERR_INVALID, "n_actions must be >= 2");
        e->ns = 2; e->nobs = 3; e->continuous = d.continuous != 0;
        if (dtype == B200RL_F64) {   // PendulumEnv() default T = Float64 (PendulumEnv.jl:42): dt = Float64(0.05) unless the caller says otherwise
            if (!params) d.dt = 0.05;
            e->p.pend64 = PendPT<double>{d.max_speed, d.max_torque, d.g, d.m, d.l, d.dt, (int)d.max_steps, (int)d.n_actions};
        } else {
            e->p.pend = PendP{(float)d.max_speed, (float)d.max_torque, (float)d.g, (float)d.m, (float)d.l, (float)d.dt,
                              (int)d.max_steps, (int)d.n_actions};
        }
    } else if (kind == B200RL_ENV_MOUNTAINCAR) {
        // ContinuousMountainCarEnv defaults: goal_pos = 0.45, power = 0.0015 (MountainCarEnv.jl:73-74)
        b200rl_mountaincar_params d = params ? *(const b200rl_mountaincar_params*)params
                                      : cont_kind ? b200rl_mountaincar_params{(float)-1.2, (float)0.6, (float)0.07, (float)0.45, 0.0,
                                                                              (float)0.0015, (float)0.0025, 200}
                                                  : b200rl_mountaincar_params{(float)-1.2, (float)0.6, (float)0.07, (float)0.5, 0.0,
                                                                              (float)0.001, (float)0.0025, 200};
        e->ns = 2; e->nobs = 2;
        if (dtype == B200RL_F64) {   // MountainCarEnv() default T = Float64 (MountainCarEnv.jl:67): the Float64 literals of :19-29
            if (!params) d = cont_kind ? b200rl_mountaincar_params{-1.2, 0.6, 0.07, 0.45, 0.0, 0.0015, 0.0025, 200}
                                       : b200rl_mountaincar_params{-1.2, 0.6, 0.07, 0.5, 0.0, 0.001, 0.0025, 200};
            e->p.mc64 = MountainCarPT<double>{d.min_pos, d.max_pos, d.max_speed, d.goal_pos, d.goal_velocity, d.power, d.gravity, (int)d.max_steps};
        } else {
            e->p.mc = MountainCarD<false>::P{(float)d.min_pos, (float)d.max_pos, (float)d.max_speed, (float)d.goal_pos, (float)d.goal_velocity,
                                             (float)d.power, (float)d.gravity, (int)d.max_steps};
        }
    } else if (kind == B200RL_ENV_ACROBOT) {
        if (dtype != B200RL_F64) { delete e; REQUIRE(false, B200RL_ERR_UNSUPPORTED, "AcrobotEnv is Float64 only (the reference constructor's default T)"); }
        b200rl_acrobot_params d = params ? *(const b200rl_acrobot_params*)params
                                         : b200rl_acrobot_params{1.0, 1.0, 1.0, 1.0, 0.5, 0.5, 1.0, 0.0, 4 * JLD_PI, 9 * JLD_PI, 9.8, 0.2, 200, 1};
        if (d.max_torque_noise != 0.0) { delete e; REQUIRE(false, B200RL_ERR_UNSUPPORTED, "AcrobotEnv: max_torque_noise > 0 is not supported"); }
        e->ns = 4; e->nobs = 6;
        e->p.acro = AcrobotP{d.link_length_a, d.link_length_b, d.link_mass_a, d.link_mass_b, d.link_com_pos_a, d.link_com_pos_b, d.link_moi,
                             d.max_torque_noise, d.max_vel_a, d.max_vel_b, d.g, d.dt, (int)d.max_steps, (int)d.book};
    } else {
        delete e;
        REQUIRE(false, B200RL_ERR_INVALID, "unknown env kind");
    }
    e->asize = (e->continuous && dtype == B200RL_F64) ? 8 : 4;
    int s = env_alloc(e);
    if (s != B200RL_OK) { b200rl_env_destroy(e); return s; }
    CUDA_TRY(cudaMemcpyAsync(e->a.rng, rng_state, (size_t)n_envs * 32, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));  // rng_state is borrowed only for this call
    s = dispatch_reset(e, 1);  // the reference constructors call reset!(env) once
    if (s != B200RL_OK) { b200rl_env_destroy(e); return s; }
    *out = e;
    return B200RL_OK;
}

int b200rl_env_destroy(b200rl_env* e) {
    if (!e) return B200RL_OK;
    cudaSetDevice(e->ctx->device);
    cudaStreamSynchronize(e->ctx->stream);
    cudaFree(e->a.state);
    if (e->a.obs != e->a.state) cudaFree(e->a.obs);
    cudaFree(e->a.reward); cudaFree(e->a.flags); cudaFree(e->a.t); cudaFree(e->a.rng); cudaFree(e->a.action);
    cudaFree(e->a.ep_ret); cudaFree(e->a.stats); cudaFree(e->a.err); cudaFree(e->rew_f32);
    log_free(e);
    delete e;
    return B200RL_OK;
}

int b200rl_env_copy(b200rl_env* src, b200rl_env** out) {
    REQUIRE(src && out, B200RL_ERR_INVALID, "null handle");
    TRY(ctx_bind(src->ctx));
    b200rl_env* e = new b200rl_env(*src);
    memset(&e->a, 0, sizeof e->a);
    e->rew_f32 = nullptr;
    e->log_ring = EpisodeLog{}; e->log_held = false; e->log_cursor = nullptr; e->log_scratch = nullptr;   // (hook data, not env state)
    e->log_flushes.clear();
    e->a.max_timeout = src->a.max_timeout;
    int s = env_alloc(e);
    if (s != B200RL_OK) { b200rl_env_destroy(e); return s; }
    cudaStream_t st = src->ctx->stream;
    for (int f : {B200RL_FIELD_STATE, B200RL_FIELD_REWARD, B200RL_FIELD_FLAGS, B200RL_FIELD_T, B200RL_FIELD_RNG, B200RL_FIELD_ACTION})
        CUDA_TRY(cudaMemcpyAsync(field_ptr(e, f), field_ptr(src, f), field_bytes(src, f), cudaMemcpyDeviceToDevice, st));
    if (e->a.obs != e->a.state)
        CUDA_TRY(cudaMemcpyAsync(e->a.obs, src->a.obs, field_bytes(src, B200RL_FIELD_OBS), cudaMemcpyDeviceToDevice, st));
    if (has_obs_f32(e))
        CUDA_TRY(cudaMemcpyAsync(obs_f32_ptr(e), obs_f32_ptr(src), (size_t)e->N * e->nobs * 4, cudaMemcpyDeviceToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(e->a.ep_ret, src->a.ep_ret, (size_t)src->N * 4, cudaMemcpyDeviceToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(e->a.stats, src->a.stats, 4 * sizeof(double), cudaMemcpyDeviceToDevice, st));
    *out = e;
    return B200RL_OK;
}

int b200rl_env_seed(b200rl_env* e, const uint64_t* rng_state) {
    REQUIRE(e && rng_state, B200RL_ERR_INVALID, "null argument");
    TRY(ctx_bind(e->ctx));
    CUDA_TRY(cudaMemcpyAsync(e->a.rng, rng_state, (size_t)e->N * 32, cudaMemcpyHostToDevice, e->ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(e->ctx->stream));
    return B200RL_OK;
}

int b200rl_env_reset(b200rl_env* e, int force_all) {
    REQUIRE(e, B200RL_ERR_INVALID, "null env");
    TRY(ctx_bind(e->ctx));
    return dispatch_reset(e, force_all);
}

int b200rl_env_step(b200rl_env* e, const void* actions, int actions_on_device, int auto_reset) {
    REQUIRE(e && actions, B200RL_ERR_INVALID, "null argument");
    TRY(ctx_bind(e->ctx));
    const void* dact = actions;
    if (actions_on_device != 1) {   // 0: pageable / borrowed host buffer, 2: pinned host buffer that stays untouched until the next sync
        void* stage;
        TRY(ctx_scratch(e->ctx, (size_t)e->N * e->asize, &stage));
        CUDA_TRY(cudaMemcpyAsync(stage, actions, (size_t)e->N * e->asize, cudaMemcpyHostToDevice, e->ctx->stream));
        dact = stage;
    }
    e->steps_launched += 1;
    TRY(dispatch_step(e, dact, false, auto_reset != 0));
    if (actions_on_device == 0) CUDA_TRY(cudaStreamSynchronize(e->ctx->stream));  // host buffer is borrowed for this call only
    return B200RL_OK;
}

int b200rl_env_set_max_timeout(b200rl_env* e, int64_t max_t) {
    REQUIRE(e, B200RL_ERR_INVALID, "null env");
    REQUIRE(max_t >= 0 && max_t < (1ll << 31), B200RL_ERR_INVALID, "max_t out of range");
    e->a.max_timeout = (int)max_t;
    return B200RL_OK;
}

int b200rl_env_set_state_f32(b200rl_env* e, int on) {
    REQUIRE(e, B200RL_ERR_INVALID, "null env");
    REQUIRE(e->kind != B200RL_ENV_ACROBOT, B200RL_ERR_UNSUPPORTED, "AcrobotEnv has 6 observations: no learner reads them");
    e->state_f32 = on != 0;   // (the env kernels keep a Float64 env's mirror current: turning the wrapper on needs no fill)
    return B200RL_OK;
}

int b200rl_env_step_random(b200rl_env* e, int auto_reset) {
    REQUIRE(e, B200RL_ERR_INVALID, "null env");
    REQUIRE(!e->continuous, B200RL_ERR_UNSUPPORTED,
            "RandomPolicy on a continuous interval (DomainSets sampler) is not restated; use a discrete-action env");
    TRY(ctx_bind(e->ctx));
    e->steps_launched += 1;
    return dispatch_step(e, nullptr, true, auto_reset != 0);
}

int b200rl_env_get(b200rl_env* e, int field, void* host_dst, size_t bytes) {
    REQUIRE(e && host_dst, B200RL_ERR_INVALID, "null argument");
    TRY(ctx_bind(e->ctx));
    size_t need = field_bytes(e, field);
    REQUIRE(need != 0, B200RL_ERR_INVALID, "unknown field");
    REQUIRE(bytes >= need, B200RL_ERR_INVALID, "destination too small");
    CUDA_TRY(cudaMemcpyAsync(host_dst, field_ptr(e, field), need, cudaMemcpyDeviceToHost, e->ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(e->ctx->stream));
    if (field == B200RL_FIELD_TERMINAL) {
        uint8_t* p = (uint8_t*)host_dst;
        for (size_t i = 0; i < need; ++i) p[i] &= 1;
    }
    if (field == B200RL_FIELD_EPISODE_STATS) ((double*)host_dst)[3] = (double)e->steps_launched * (double)e->N;   // host-side counter
    return B200RL_OK;
}

int b200rl_env_set(b200rl_env* e, int field, const void* host_src, size_t bytes) {
    REQUIRE(e && host_src, B200RL_ERR_INVALID, "null argument");
    TRY(ctx_bind(e->ctx));
    size_t need = field_bytes(e, field);
    REQUIRE(need != 0 && field != B200RL_FIELD_TERMINAL, B200RL_ERR_INVALID, "field not settable (TERMINAL is bit 0 of FLAGS)");
    REQUIRE(field != B200RL_FIELD_OBS_F32, B200RL_ERR_INVALID, "OBS_F32 follows the observation: set STATE / OBS");
    REQUIRE(bytes >= need, B200RL_ERR_INVALID, "source too small");
    CUDA_TRY(cudaMemcpyAsync(field_ptr(e, field), host_src, need, cudaMemcpyHostToDevice, e->ctx->stream));
    if (has_obs_f32(e) && (field == B200RL_FIELD_STATE || field == B200RL_FIELD_OBS)) {   // the mirror follows the observation
        const int64_t n = e->N * e->nobs;
        narrow_f64_kernel<<<grid_for(n, kBlock), kBlock, 0, e->ctx->stream>>>(obs_f32_ptr(e), (const double*)e->a.obs, n);
        LAUNCH_CHECK(e->ctx);
    }
    CUDA_TRY(cudaStreamSynchronize(e->ctx->stream));
    if (field == B200RL_FIELD_EPISODE_STATS) e->steps_launched = (uint64_t)(((const double*)host_src)[3] / (double)e->N + 0.5);
    return B200RL_OK;
}

int b200rl_env_ptr(b200rl_env* e, int field, void** dptr_out) {
    REQUIRE(e && dptr_out, B200RL_ERR_INVALID, "null argument");
    void* p = field_ptr(e, field);
    REQUIRE(p, B200RL_ERR_INVALID, "unknown field");
    *dptr_out = p;
    return B200RL_OK;
}

int b200rl_env_check(b200rl_env* e) {
    REQUIRE(e, B200RL_ERR_INVALID, "null env");
    TRY(ctx_bind(e->ctx));
    int flag = 0;
    CUDA_TRY(cudaMemcpyAsync(&flag, e->a.err, sizeof flag, cudaMemcpyDeviceToHost, e->ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(e->ctx->stream));
    if (flag) {
        CUDA_TRY(cudaMemsetAsync(e->a.err, 0, sizeof(int), e->ctx->stream));
        b200rl_set_error("b200rl_env_step: an action outside action_space(env) was passed (the reference asserts `a in action_space(env)`)");
        return B200RL_ERR_ACTION;
    }
    return B200RL_OK;
}

int b200rl_env_episode_stats(b200rl_env* e, double* out4, int reset_after) {
    REQUIRE(e && out4, B200RL_ERR_INVALID, "null argument");
    TRY(ctx_bind(e->ctx));
    CUDA_TRY(cudaMemcpyAsync(out4, e->a.stats, 4 * sizeof(double), cudaMemcpyDeviceToHost, e->ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(e->ctx->stream));
    out4[3] = (double)e->steps_launched * (double)e->N;
    if (reset_after) {
        CUDA_TRY(cudaMemsetAsync(e->a.stats, 0, 4 * sizeof(double), e->ctx->stream));
        e->steps_launched = 0;
    }
    return B200RL_OK;
}

int b200rl_env_episode_log(b200rl_env* e, int32_t K) {
    REQUIRE(e, B200RL_ERR_INVALID, "null env");
    REQUIRE(K >= 0 && K <= (1 << 20), B200RL_ERR_INVALID, "K must be in 0 .. 2^20");
    TRY(ctx_bind(e->ctx));
    const size_t N = (size_t)e->N, nb = grid_for(e->N, kBlock);
    cudaStream_t st = e->ctx->stream;
    if (K > 0 && K == e->log_ring.K) {   // the same ring, emptied: the captured launches that write it stay valid
        CUDA_TRY(cudaMemsetAsync(e->log_ring.count, 0, N * 4, st));
        CUDA_TRY(cudaMemsetAsync(e->log_cursor, 0, N * 4, st));
        CUDA_TRY(cudaMemsetAsync(e->log_scratch, 0, (nb + 1) * sizeof(long long), st));
        for (auto& f : e->log_flushes) f.buf = nullptr;   // (every buffer starts without a flush)
        CUDA_TRY(cudaStreamSynchronize(st));
        return B200RL_OK;
    }
    log_free(e);
    if (K == 0) return B200RL_OK;
    EpisodeLog& l = e->log_ring;
    CUDA_TRY_OR(cudaMalloc(&l.ret, N * K * 4), log_free(e));
    CUDA_TRY_OR(cudaMalloc(&l.len, N * K * 4), log_free(e));
    CUDA_TRY_OR(cudaMalloc(&l.count, N * 4), log_free(e));
    CUDA_TRY_OR(cudaMalloc(&e->log_cursor, N * 4), log_free(e));
    CUDA_TRY_OR(cudaMalloc(&e->log_scratch, (nb + 1) * sizeof(long long)), log_free(e));
    CUDA_TRY_OR(cudaMemsetAsync(l.count, 0, N * 4, st), log_free(e));
    CUDA_TRY_OR(cudaMemsetAsync(e->log_cursor, 0, N * 4, st), log_free(e));
    CUDA_TRY_OR(cudaMemsetAsync(e->log_scratch, 0, (nb + 1) * sizeof(long long), st), log_free(e));
    // the events of the flushes into two host buffers (what DeviceEpisodeLog uses) are created now: creating one may wait for the
    // device, and ranks sharing a device must not do that while a peer's kernel waits for them inside an exchange
    for (int j = 0; j < 2; ++j) {
        cudaEvent_t ev;
        CUDA_TRY_OR(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming), log_free(e));
        e->log_flushes.push_back(b200rl_env::LogFlush{nullptr, 0, ev});
    }
    CUDA_TRY_OR(cudaStreamSynchronize(st), log_free(e));
    l.K = K;
    return B200RL_OK;
}

int b200rl_env_episode_log_flush(b200rl_env* e, void* host_buf, int64_t capacity) {
    REQUIRE(e && host_buf, B200RL_ERR_INVALID, "null argument");
    REQUIRE(e->log_ring.count, B200RL_ERR_INVALID, "no episode log attached (b200rl_env_episode_log)");
    REQUIRE(capacity >= 0, B200RL_ERR_INVALID, "capacity must be >= 0");
    TRY(ctx_bind(e->ctx));
    cudaPointerAttributes at;
    CUDA_TRY(cudaPointerGetAttributes(&at, host_buf));
    REQUIRE(at.type == cudaMemoryTypeHost && at.devicePointer, B200RL_ERR_INVALID, "host_buf must be pinned host memory (b200rl_host_alloc)");
    b200rl_env::LogFlush* f = nullptr;
    for (auto& x : e->log_flushes) if (x.buf == host_buf) f = &x;
    for (auto& x : e->log_flushes) if (!f && !x.buf) { f = &x; f->buf = host_buf; }   // a spare event
    if (!f) {
        cudaEvent_t ev;
        CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        e->log_flushes.push_back(b200rl_env::LogFlush{host_buf, 0, ev});
        f = &e->log_flushes.back();
    }
    f->capacity = capacity;
    const unsigned nb = grid_for(e->N, kBlock);
    long long* hdr = (long long*)at.devicePointer;
    unsigned long long* overflow = (unsigned long long*)(e->log_scratch + nb);
    cudaStream_t st = e->ctx->stream;
    log_count_kernel<<<nb, kBlock, 0, st>>>(e->log_ring, e->log_cursor, e->N, e->log_scratch, overflow);
    LAUNCH_CHECK(e->ctx);
    log_offsets_kernel<<<1, kBlock, 0, st>>>(e->log_scratch, nb, overflow, hdr);
    LAUNCH_CHECK(e->ctx);
    log_scatter_kernel<<<nb, kBlock, 0, st>>>(e->log_ring, e->log_cursor, e->N, e->log_scratch, (int64_t)b200rl_comm_rank(e->ctx) * e->N,
                                              reinterpret_cast<EpisodeRecord*>(hdr + 2), capacity);
    LAUNCH_CHECK(e->ctx);
    CUDA_TRY(cudaEventRecord(f->done, st));
    return B200RL_OK;
}

int b200rl_env_episode_log_read(b200rl_env* e, const void* host_buf, int64_t* n_out) {
    REQUIRE(e && host_buf && n_out, B200RL_ERR_INVALID, "null argument");
    const b200rl_env::LogFlush* f = nullptr;
    for (const auto& x : e->log_flushes) if (host_buf && x.buf == host_buf) f = &x;
    REQUIRE(f, B200RL_ERR_INVALID, "no flush into this buffer since the log was attached");
    TRY(ctx_bind(e->ctx));
    CUDA_TRY(cudaEventSynchronize(f->done));
    const long long* hdr = (const long long*)host_buf;
    *n_out = hdr[0];
    if (hdr[1]) {
        b200rl_set_error("b200rl_env_episode_log_read: %lld of the %lld envs finished more than K = %d episodes between two flushes "
                         "(records were overwritten before they were read): flush at least every K env steps",
                         (long long)hdr[1], (long long)e->N, e->log_ring.K);
        return B200RL_ERR_OVERFLOW;
    }
    if (hdr[0] > f->capacity) {
        b200rl_set_error("b200rl_env_episode_log_read: the flush found %lld records, the buffer holds %lld", (long long)hdr[0],
                         (long long)f->capacity);
        return B200RL_ERR_OVERFLOW;
    }
    return B200RL_OK;
}

}  // extern "C"

// internal hooks for other translation units (fused consumers; internal.h)
void b200rl_env_internal_log_hold(b200rl_env* e, bool hold) { e->log_held = hold; }
void b200rl_env_internal_log_key(const b200rl_env* e, uint64_t key[4]) {
    const EpisodeLog l = active_log(e);
    key[0] = (uint64_t)(uintptr_t)l.ret; key[1] = (uint64_t)(uintptr_t)l.len;
    key[2] = (uint64_t)(uintptr_t)l.count; key[3] = (uint64_t)l.K;
}
int b200rl_env_internal_set_traj_targets(b200rl_env* e, void* reward_col, uint8_t* terminal_col) {
    e->a.traj_reward = reward_col;
    e->a.traj_terminal = terminal_col;
    return B200RL_OK;
}
int b200rl_env_internal_view(b200rl_env* e, envdev::EnvView* out) {
    REQUIRE(e && out, B200RL_ERR_INVALID, "null argument");
    out->kind = e->kind; out->dtype = e->dtype; out->continuous = e->continuous ? 1 : 0; out->N = e->N; out->a = e->a;
    out->log = active_log(e);
    static_assert(sizeof(out->p) == sizeof(e->p), "params union");
    memcpy(&out->p, &e->p, sizeof out->p);
    return B200RL_OK;
}
int b200rl_env_internal_step_regions(const b200rl_env* e, DevRegion* out) {
    const size_t N = (size_t)e->N, mirror = has_obs_f32(e) ? N * e->nobs * 4 : 0;
    int n = 0;
    if (e->a.obs == e->a.state) {
        out[n++] = {e->a.state, N * e->ns * e->tsize + mirror};
    } else {
        out[n++] = {e->a.state, N * e->ns * e->tsize};
        out[n++] = {e->a.obs, N * e->nobs * e->tsize + mirror};
    }
    out[n++] = {e->a.reward, N * e->tsize};
    if (e->rew_f32) out[n++] = {e->rew_f32, N * 4};
    out[n++] = {e->a.flags, N};
    out[n++] = {e->a.t, N * 4};
    out[n++] = {e->a.rng, N * 32};
    out[n++] = {e->a.action, N * e->asize};
    out[n++] = {e->a.ep_ret, N * 4};
    out[n++] = {e->a.stats, 4 * sizeof(double)};
    if (e->log_ring.count) out[n++] = {e->log_ring.count, N * 4};
    return n;
}
size_t b200rl_env_internal_step_bytes_max(const b200rl_env* e) {
    DevRegion r[kEnvStepRegionsMax];
    const int n = b200rl_env_internal_step_regions(e, r);
    size_t total = e->log_ring.count ? 0 : (size_t)e->N * 4 + 256;   // (room for the write counts of an episode log attached later)
    for (int k = 0; k < n; ++k) total += (r[k].bytes + 255) / 256 * 256;
    return total;
}
void b200rl_env_internal_add_steps(b200rl_env* e, uint64_t n) { e->steps_launched += n; }
uint64_t b200rl_env_internal_steps(const b200rl_env* e) { return e->steps_launched; }
int b200rl_env_internal_max_timeout(const b200rl_env* e) { return e->a.max_timeout; }
bool b200rl_env_internal_state_f32(const b200rl_env* e) { return e->dtype == B200RL_F64 && e->state_f32; }   // (the identity on Float32)
const float* b200rl_env_internal_obs_f32(const b200rl_env* e) {
    if (e->dtype == B200RL_F32) return (const float*)e->a.obs;
    return e->state_f32 ? obs_f32_ptr(e) : nullptr;
}
int b200rl_env_internal_reward_f32(b200rl_env* e, const float** out) {   // (a launch on the ctx stream for a Float64 env)
    if (e->dtype == B200RL_F32) { *out = (const float*)e->a.reward; return B200RL_OK; }
    REQUIRE(e->rew_f32, B200RL_ERR_UNSUPPORTED, "AcrobotEnv has no Float32 view");
    narrow_f64_kernel<<<grid_for(e->N, kBlock), kBlock, 0, e->ctx->stream>>>(e->rew_f32, (const double*)e->a.reward, e->N);
    LAUNCH_CHECK(e->ctx);
    *out = e->rew_f32;
    return B200RL_OK;
}
int b200rl_env_internal_dtype(const b200rl_env* e) { return e->dtype; }
int64_t b200rl_env_internal_n(const b200rl_env* e) { return e->N; }
int b200rl_env_internal_kind(const b200rl_env* e) { return e->kind; }
int b200rl_env_internal_nobs(const b200rl_env* e) { return e->nobs; }
int b200rl_env_internal_n_actions(const b200rl_env* e) {   // size of a discrete action space (0: continuous)
    if (e->continuous) return 0;
    if (e->kind == B200RL_ENV_PENDULUM) return e->dtype == B200RL_F64 ? e->p.pend64.n_actions : e->p.pend.n_actions;
    return e->kind == B200RL_ENV_CARTPOLE ? 2 : 3;
}
float b200rl_env_internal_action_bound(const b200rl_env* e) {   // continuous action space -bound..bound
    switch (e->kind) {
        case B200RL_ENV_PENDULUM: return PendulumD<true>::kActionBound;
        case B200RL_ENV_MOUNTAINCAR: return MountainCarD<true>::kActionBound;
    }
    return CartPoleD<float, true>::kActionBound;
}
b200rl_ctx* b200rl_env_internal_ctx(const b200rl_env* e) { return e->ctx; }
bool b200rl_env_internal_continuous(const b200rl_env* e) { return e->continuous; }
