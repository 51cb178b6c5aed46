// tests/hostdev/episode_log.cpp — TEST INFRASTRUCTURE.  The episode-log write of act_step and the flush helpers of env_device.cuh,
// compiled for the host (see cuda_runtime.h), behind a flat C interface for tests/test_episode_log_host.py.
#include <cuda_runtime.h>

#include "env_device.cuh"

using namespace envdev;

namespace {
CartPoleD<float>::P cartpole_params() {
    // g, total mass, pole mass, half length, pole mass * length, force, dt, angle and position thresholds, max steps
    return CartPoleD<float>::P{(float)9.8, (float)(1.0 + 0.1), (float)0.1, 0.5f, (float)(0.1 * 0.5), 10.0f, (float)0.02,
                               (float)(12.0 * JLD_PI / 180), (float)2.4, 200};
}
}  // namespace

extern "C" {

// Steps env i of a CartPole batch n_steps times with the given 1-based actions (rng: its Xoshiro state, updated).  reset_mode 0:
// the fused auto-reset (act_step<AUTO = true>), 1: MultiThreadEnv's soft reset before each step of an env that terminated, 2: no
// reset (a terminal env is stepped again).  The log (K, N) ret / len and count (N) are written by act_step; rew / done / fin receive
// each step's Float32 reward, done and the finished-episode tally increment.
int el_cartpole_run(int64_t i, int K, int max_timeout, int reset_mode, const int32_t* actions, int n_steps, uint64_t* rng,
                    float* log_ret, int32_t* log_len, uint32_t* log_count, float* rew, uint8_t* done, int32_t* fin) {
    using Env = CartPoleD<float>;
    const Env::P p = cartpole_params();
    Xo g{rng[0], rng[1], rng[2], rng[3]};
    Env::S s;
    int32_t act = 0;
    Env::reset(p, s, g, act);
    int t = 0, flags = 0;
    float ep_ret = 0.f;
    const EpisodeLog log{log_ret, log_len, log_count, K};
    for (int k = 0; k < n_steps; ++k) {
        if (reset_mode == 1 && (flags & 1) && !(flags & 2)) {   // b200rl_env_reset(force = 0)
            Env::reset(p, s, g, act);
            t = 0; flags = 0; ep_ret = 0.f;
        }
        act = actions[k];
        int fin_cnt = 0, fin_len = 0;
        float fin_ret = 0.f;
        ActStep<float> r;
        auto with_rng = [&](auto&& reset) { reset(g); };
        if (reset_mode == 0) r = act_step<Env, true, true>(p, max_timeout, s, t, flags, ep_ret, act, fin_cnt, fin_ret, fin_len, with_rng, log, i);
        else r = act_step<Env, false, true>(p, max_timeout, s, t, flags, ep_ret, act, fin_cnt, fin_ret, fin_len, with_rng, log, i);
        rew[k] = r.rew;
        done[k] = r.done ? 1 : 0;
        fin[k] = fin_cnt;
    }
    rng[0] = g.s0; rng[1] = g.s1; rng[2] = g.s2; rng[3] = g.s3;
    return 0;
}

// The flush of env.cu restated serially with the same helpers: each env's pending records (count - cursor, an env above K counts as
// overflowing and gives K) at the running offset, cursors advanced.  Returns the list length; *overflow = overflowing envs.
int64_t el_flush(int K, int64_t N, float* log_ret, int32_t* log_len, uint32_t* log_count, uint32_t* cursor, int64_t global0,
                 EpisodeRecord* out, int64_t capacity, int64_t* overflow) {
    const EpisodeLog log{log_ret, log_len, log_count, K};
    int64_t off = 0;
    *overflow = 0;
    for (int64_t i = 0; i < N; ++i) {
        uint32_t n = log_pending(log, cursor, i);
        if (n > (uint32_t)K) { *overflow += 1; n = (uint32_t)K; }
        if (n) log_emit(log, cursor, i, n, global0 + i, out + off, capacity - off);
        cursor[i] = log_count[i];
        off += n;
    }
    return off;
}

}  // extern "C"
