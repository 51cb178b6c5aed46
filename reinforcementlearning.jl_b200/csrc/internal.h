// internal.h — what the translation units of libb200rl.so export to each other outside the C ABI: the accessors of the env,
// trajectory, returns and communicator handles.  Included by the units that define them too, so that the compiler checks every
// declaration against its definition.
#pragma once
#include "common.cuh"

struct Ring;                              // ring.cuh
namespace envdev { struct EnvView; }     // env_device.cuh

// a device array {pointer, bytes}: the state a stretch of the fused loops changes (b200rl_*_run_episodes shadow it)
struct DevRegion { void* p; size_t bytes; };

// ---- env.cu
// the device arrays an env step writes (state, observation and its Float32 mirror, reward, flags, t, streams, action, episode
// return and statistics, the episode log's write counts) -> out[0 .. n), n <= kEnvStepRegionsMax
constexpr int kEnvStepRegionsMax = 11;
int b200rl_env_internal_step_regions(const b200rl_env* e, DevRegion* out);
// their bytes, each rounded up to 256, with room for the write counts of an episode log attached later
size_t b200rl_env_internal_step_bytes_max(const b200rl_env* e);
int b200rl_env_internal_set_traj_targets(b200rl_env* e, void* reward_col, uint8_t* terminal_col);
int b200rl_env_internal_view(b200rl_env* e, envdev::EnvView* out);
void b200rl_env_internal_add_steps(b200rl_env* e, uint64_t n);
uint64_t b200rl_env_internal_steps(const b200rl_env* e);
int b200rl_env_internal_max_timeout(const b200rl_env* e);
// hold = true: the env's kernels stop writing its episode log (a staged evaluation is not logged); false: they write it again
void b200rl_env_internal_log_hold(b200rl_env* e, bool hold);
// the episode log the env's kernels write (all zero: none) as {ret, len, count, K} — captured launches bake it in
void b200rl_env_internal_log_key(const b200rl_env* e, uint64_t key[4]);
// StateTransformedEnv(env, Float32) in effect: a Float64 env with the wrapper (on a Float32 env the wrapper changes nothing)
bool b200rl_env_internal_state_f32(const b200rl_env* e);
// the Float32 observation (NOBS, N) the networks read: FIELD_OBS of a Float32 env, the mirror of a Float64 env wrapped by
// b200rl_env_set_state_f32; null for a Float64 env without the wrapper
const float* b200rl_env_internal_obs_f32(const b200rl_env* e);
// Float32(reward(env)) (N): FIELD_REWARD of a Float32 env, a converted copy (launched on the ctx stream) of a Float64 env's
int b200rl_env_internal_reward_f32(b200rl_env* e, const float** out);
int b200rl_env_internal_dtype(const b200rl_env* e);
int64_t b200rl_env_internal_n(const b200rl_env* e);
int b200rl_env_internal_kind(const b200rl_env* e);
int b200rl_env_internal_nobs(const b200rl_env* e);
int b200rl_env_internal_n_actions(const b200rl_env* e);
float b200rl_env_internal_action_bound(const b200rl_env* e);
b200rl_ctx* b200rl_env_internal_ctx(const b200rl_env* e);
bool b200rl_env_internal_continuous(const b200rl_env* e);

// ---- traj.cu
struct TrajBatchView { const float* s; const int32_t* a; const float* r; const uint8_t* t; const float* s2; const float* w; int64_t B; int ns; };
TrajBatchView b200rl_traj_internal_batch(b200rl_traj* t);
bool b200rl_traj_internal_prioritized(b200rl_traj* t);
b200rl_ctx* b200rl_traj_internal_ctx(b200rl_traj* t);
int64_t b200rl_traj_internal_lanes(b200rl_traj* t);
void b200rl_traj_internal_add_pushed(b200rl_traj* t, int64_t n);
// the ring's checkpoint fields (b200rl_traj_get 0 .. 9: frames, head, count, pending, n_sampleable, sum tree, sampler streams)
// -> out[0 .. n), n <= kTrajStateRegionsMax
constexpr int kTrajStateRegionsMax = 10;
int b200rl_traj_internal_state_regions(b200rl_traj* t, DevRegion* out);
int64_t b200rl_traj_internal_pushed(b200rl_traj* t);
Ring b200rl_traj_internal_ring(b200rl_traj* t);
float b200rl_traj_internal_default_priority(b200rl_traj* t);
void b200rl_traj_internal_nstep(b200rl_traj* t, int* n, float* gamma);
const float* b200rl_traj_internal_discount(b200rl_traj* t);
int b200rl_traj_internal_tree_rebuild(b200rl_traj* t, const int64_t* keys, const float* vals, int64_t n);
int b200rl_traj_internal_priority_from_td(b200rl_traj* t, const float* td_dev, float eps, float alpha);

// ---- returns.cu
int b200rl_gae_fused_internal(b200rl_ctx* ctx, float* adv, float* ret, const float* r, const float* v, const uint8_t* term, float gamma,
                              float lambda, int64_t S, int64_t n_time, double* partials);
int b200rl_gae_fused_partials_count(int64_t S);

// ---- comm.cu
int b200rl_comm_allreduce_internal(b200rl_ctx* ctx, void* buf, int64_t n, int is_double);
void b200rl_comm_destroy_internal(b200rl_ctx* ctx);
