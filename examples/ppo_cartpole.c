/* examples/ppo_cartpole.c — a pure-C client of libb200rl.so: what any host language's FFI does.
 *
 * The reference's loop (RLCore/src/core/run.jl:36-78) for N batched CartPole envs and a PPO agent:
 *     run(agent, env, StopAfterNSteps(n_iter * T), hook)
 * driven through the C ABI only (include/b200rl.h) — no Python, no torch, no Julia.
 *
 *   gcc -O2 -Iinclude examples/ppo_cartpole.c -Lreinforcementlearning.jl_b200 -lb200rl \
 *       -Wl,-rpath,$PWD/reinforcementlearning.jl_b200 -lm -o /tmp/ppo_cartpole && /tmp/ppo_cartpole [n_envs] [iterations]
 *
 * Needs an H100 to run (there is no CPU fallback: b200rl_init fails loudly otherwise); building needs none.
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "b200rl.h"

#define CHECK(expr)                                                                  \
    do {                                                                             \
        int s_ = (expr);                                                             \
        if (s_ != B200RL_OK) {                                                       \
            fprintf(stderr, "%s -> %d: %s\n", #expr, s_, b200rl_last_error());       \
            return 1;                                                                \
        }                                                                            \
    } while (0)

/* test-harness seeding (SURVEY §8d): four splitmix64 outputs of seed ^ i per stream; Julia passes Xoshiro(seed_i) states */
static uint64_t splitmix64(uint64_t* x) {
    uint64_t z = (*x += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
static uint64_t* make_streams(int64_t n, uint64_t seed) {
    uint64_t* s = (uint64_t*)malloc((size_t)n * 4 * sizeof(uint64_t));
    for (int64_t i = 0; s && i < n; ++i) {
        uint64_t x = seed ^ (uint64_t)i;
        for (int k = 0; k < 4; ++k) s[4 * i + k] = splitmix64(&x);
    }
    return s;
}
/* Flux glorot_uniform Dense init in Flux.destructure order: W (out, in) column-major, then the bias (zeros) */
static float* dense(float* p, int out, int in, uint64_t* x) {
    const double lim = sqrt(6.0 / (in + out));
    for (int k = 0; k < out * in; ++k) *p++ = (float)((2.0 * ((double)(splitmix64(x) >> 11) * 0x1p-53) - 1.0) * lim);
    for (int k = 0; k < out; ++k) *p++ = 0.0f;
    return p;
}

int main(int argc, char** argv) {
    const int64_t n_envs = argc > 1 ? atoll(argv[1]) : 65536;
    const int iterations = argc > 2 ? atoi(argv[2]) : 10;
    const int T = 32, hidden = 64;

    b200rl_ctx* ctx = NULL;
    CHECK(b200rl_init(0, &ctx));

    /* MultiThreadEnv([CartPoleEnv(T = Float32, rng = ...) for i in 1:N]) */
    uint64_t* env_seeds = make_streams(n_envs, 1);
    uint64_t* policy_seeds = make_streams(n_envs, 2);
    if (!env_seeds || !policy_seeds) return 1;
    b200rl_env* env = NULL;
    CHECK(b200rl_env_create(ctx, B200RL_ENV_CARTPOLE, B200RL_F32, n_envs, NULL, env_seeds, &env));

    /* ActorCritic(actor 4-64-64-2, critic 4-64-64-1) as one flat parameter vector */
    b200rl_net_desc desc = {4, hidden, 0 /* relu */, 2, 0 /* categorical actor-critic */};
    int64_t np = 0;
    CHECK(b200rl_net_nparams(&desc, &np));
    float* params = (float*)malloc((size_t)np * sizeof(float));
    if (!params) return 1;
    uint64_t x = 123;
    float* p = params;
    p = dense(p, hidden, 4, &x); p = dense(p, hidden, hidden, &x); p = dense(p, 2, hidden, &x);      /* actor  */
    p = dense(p, hidden, 4, &x); p = dense(p, hidden, hidden, &x); p = dense(p, 1, hidden, &x);      /* critic */
    if (p - params != np) { fprintf(stderr, "parameter count mismatch\n"); return 1; }
    b200rl_net* net = NULL;
    CHECK(b200rl_net_create(ctx, &desc, params, &net));

    /* Agent(PPOPolicy(...), PPOTrajectory(capacity = T)): the in-tree example's hyper-parameters */
    b200rl_onpolicy_config cfg = {0.99f, 0.95f, 0.1f, 0.5f, 1.0f, 0.5f, 0.001f, 1e-3f, 0.9f, 0.999f, 1e-8f, 0.0f, INFINITY,
                                  1 /* normalize advantages */, 4 /* epochs */, 4 /* minibatches */, T, 0 /* PPO */};
    b200rl_onpolicy* agent = NULL;
    CHECK(b200rl_onpolicy_create(ctx, net, env, &cfg, policy_seeds, &agent));

    CHECK(b200rl_env_reset(env, 1));                       /* run.jl:46 */
    float stats[16 * 6];
    for (int it = 0; it < iterations; ++it) {
        CHECK(b200rl_timer_start(ctx));
        CHECK(b200rl_onpolicy_collect(agent, T));          /* T x {plan!, act!, push!} in one launch */
        CHECK(b200rl_onpolicy_update(agent, NULL, stats)); /* optimise!: GAE + 4 x 4 optimiser steps */
        float ms = 0.f;
        CHECK(b200rl_timer_stop_ms(ctx, &ms));
        double ep[4];
        CHECK(b200rl_env_episode_stats(env, ep, 0));
        printf("iteration %2d  %.3f ms  %.1f M env-steps/s  loss %.4f  grad-norm %.4f  mean episode length %.1f\n", it, ms,
               (double)n_envs * T / ms / 1e3, stats[15 * 6 + 3], stats[15 * 6 + 4], ep[0] > 0 ? ep[2] / ep[0] : 0.0);
    }
    CHECK(b200rl_env_check(env));                          /* the reference's `@assert a in action_space(env)` */

    b200rl_onpolicy_destroy(agent);
    b200rl_net_destroy(net);
    b200rl_env_destroy(env);
    b200rl_destroy(ctx);
    free(params); free(env_seeds); free(policy_seeds);
    return 0;
}
