/* b200rl.h — C ABI of libb200rl.so: the H100 (sm_90a) vectorised RL inner loop that
 * sits behind ReinforcementLearning.jl's `Base.run(policy, env, stop, hook)` surface.
 *
 * The reference has no FFI: its extension mechanism is Julia multiple dispatch on
 * `AbstractEnv` / `AbstractPolicy` (src/ReinforcementLearningBase/src/interface.jl:27,67).
 * "Drop-in" therefore means new Julia subtypes whose methods `ccall` the entry points below
 * (see INTEGRATION.md and reinforcementlearning.jl_b200/julia/B200RL.jl).  Each entry point
 * cites the reference method(s) it stands in for; paths are relative to /root/reference/src.
 *
 * Conventions
 *  - every function returns 0 (B200RL_OK) or a negative b200rl_status; nothing throws across
 *    the ABI; b200rl_last_error() returns a thread-local message for the last failure.
 *  - plain pointers and sizes only.  Host arrays are borrowed for the duration of the call.
 *    Arrays use Julia's column-major convention: env state is (NS, N), rollout tensors are
 *    (N, T) env-fastest.
 *  - the library owns all device memory behind the opaque handles.  Each ctx owns one CUDA
 *    stream; calls are asynchronous on it except *_get / *_sync and calls taking host arrays.
 *  - handles are not thread-safe (one driver task per ctx, like the reference's
 *    single-threaded _run, RLCore/src/core/run.jl:36-78).
 *  - there is NO CPU fallback: every entry point fails with B200RL_ERR_CUDA when no sm_90
 *    device is usable.
 */
#ifndef B200RL_H
#define B200RL_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    B200RL_OK = 0,
    B200RL_ERR_INVALID = -1,        /* bad argument / handle */
    B200RL_ERR_CUDA = -2,           /* CUDA runtime / launch failure */
    B200RL_ERR_UNSUPPORTED = -3,    /* configuration outside the hot-path scope */
    B200RL_ERR_ACTION = -4,         /* an action outside action_space(env) was seen (replaces `@assert a in action_space(env)`) */
    B200RL_ERR_NCCL = -5,
    B200RL_ERR_OOM = -6,
    B200RL_ERR_OVERFLOW = -7        /* an episode log lost records: more than K episodes of one env between two flushes */
} b200rl_status;

typedef struct b200rl_ctx b200rl_ctx;
typedef struct b200rl_env b200rl_env;
typedef struct b200rl_traj b200rl_traj;
typedef struct b200rl_net b200rl_net;

/* ---------------------------------------------------------------- context ---------- */
int b200rl_init(int device, b200rl_ctx** out);
void b200rl_destroy(b200rl_ctx* ctx);
const char* b200rl_last_error(void);
int b200rl_sync(b200rl_ctx* ctx);                   /* cudaStreamSynchronize(ctx stream) */
int b200rl_abi_version(void);
/* raw CUDA stream of the ctx (cudaStream_t as void*) so a host can order its own work */
int b200rl_stream(b200rl_ctx* ctx, void** stream_out);
/* device timing on the ctx stream (CUDA events) for hosts without a CUDA binding */
int b200rl_timer_start(b200rl_ctx* ctx);
int b200rl_timer_stop_ms(b200rl_ctx* ctx, float* ms_out);   /* synchronises */
/* event slots (0..511): record points on the ctx stream without synchronising the host, read the intervals afterwards
 * (elapsed_ms waits for slot_to's event only).  A benchmark loop records 2 slots per step and syncs once at the end, so the
 * host can run ahead of the device. */
int b200rl_timer_record(b200rl_ctx* ctx, int slot);
int b200rl_timer_elapsed_ms(b200rl_ctx* ctx, int slot_from, int slot_to, float* ms_out);
/* measurement aid: base_slot >= 0 makes b200rl_onpolicy_update (eager launches only) record its phases into the slots
 * base_slot + {0 entry, 1 after bootstrap/GAE/normalisation/record packing, 2+2i after loss+backward i, 3+2i after optimiser step i};
 * -1 switches it off */
int b200rl_debug_phase_slots(b200rl_ctx* ctx, int base_slot);
/* device / pinned-host buffers for hosts without a CUDA binding (Julia without CUDA.jl) */
int b200rl_malloc(b200rl_ctx* ctx, size_t bytes, void** dptr_out);
int b200rl_free(b200rl_ctx* ctx, void* dptr);
int b200rl_host_alloc(b200rl_ctx* ctx, size_t bytes, void** hptr_out);   /* pinned */
int b200rl_host_free(b200rl_ctx* ctx, void* hptr);
int b200rl_memcpy_h2d(b200rl_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes, int async);
int b200rl_memcpy_d2h(b200rl_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes, int async);
int b200rl_memset(b200rl_ctx* ctx, void* dst_dev, int value, size_t bytes);
/* number of kernels this ctx has launched so far (bench `gpu_launches`) */
int b200rl_launch_count(b200rl_ctx* ctx, uint64_t* count_out);
/* write > L2-capacity bytes so the next kernel starts from a cold L2 (bench hygiene) */
int b200rl_flush_l2(b200rl_ctx* ctx);

/* ---------------------------------------------------------------- vector env ------- */
typedef enum {
    B200RL_ENV_CARTPOLE = 0, B200RL_ENV_PENDULUM = 1, B200RL_ENV_MOUNTAINCAR = 2,
    B200RL_ENV_CARTPOLE_CONTINUOUS = 3,     /* CartPoleEnv(continuous = true): Float32 action in -1.0..1.0 (CartPoleEnv.jl:74-79,106-110) */
    B200RL_ENV_MOUNTAINCAR_CONTINUOUS = 4,  /* ContinuousMountainCarEnv (MountainCarEnv.jl:73-74,83,107-111); params as mountaincar */
    B200RL_ENV_ACROBOT = 5                  /* AcrobotEnv{Float64} (3rd_party/AcrobotEnv.jl:19-225): B200RL_F64 only, 6 observations, 3 actions;
                                               one classical RK4 step per act! (the reference's adaptive OrdinaryDiffEq controller is external) */
} b200rl_env_kind;
typedef enum { B200RL_F32 = 0, B200RL_F64 = 1 } b200rl_dtype;
typedef enum {
    B200RL_FIELD_STATE = 0,     /* (NS, N) T      env.state                                      */
    B200RL_FIELD_OBS = 1,       /* (NOBS, N) T    state(env)  (Pendulum: [sin th, cos th, thdot]) */
    B200RL_FIELD_REWARD = 2,    /* (N,) T         reward(env)                                    */
    B200RL_FIELD_TERMINAL = 3,  /* (N,) uint8     is_terminated(env)                             */
    B200RL_FIELD_T = 4,         /* (N,) int32     env.t                                          */
    B200RL_FIELD_RNG = 5,       /* (4, N) uint64  raw Xoshiro256++ state s0..s3 per env          */
    B200RL_FIELD_FLAGS = 6,     /* (N,) uint8     bit0 terminal, bit1 already auto-reset         */
    B200RL_FIELD_ACTION = 7,    /* (N,) int32 | T last action                                    */
    B200RL_FIELD_EPISODE_RETURN = 8,  /* (N,) float32  running return of the episode in progress (device-side hooks)  */
    B200RL_FIELD_EPISODE_STATS = 9,   /* (4,) float64  the counters b200rl_env_episode_stats reads (checkpoints)      */
    B200RL_FIELD_OBS_F32 = 10         /* (NOBS, N) float32  Float32.(state(env)), round to nearest (what the learners read):
                                         FIELD_OBS itself for a Float32 env, a mirror kept by every env kernel for a Float64
                                         one wrapped by b200rl_env_set_state_f32 (unknown field without the wrapper);
                                         read-only, it follows env_set of STATE / OBS */
} b200rl_field;

/* Final field values of the reference's params structs (already rounded to T by the
 * reference constructor; double embeds Float32 exactly).  Pass NULL for the defaults. */
typedef struct {   /* CartPoleEnvParams{T}: RLEnvs/src/environments/examples/CartPoleEnv.jl:3-46 */
    double gravity, masscart, masspole, totalmass, halflength, polemasslength, forcemag, dt,
        thetathreshold, xthreshold;
    int64_t max_steps;
} b200rl_cartpole_params;
typedef struct {   /* PendulumEnvParams{T} + n_actions + continuous: PendulumEnv.jl:3-66 */
    double max_speed, max_torque, g, m, l, dt;
    int64_t max_steps, n_actions;
    int32_t continuous;
} b200rl_pendulum_params;
typedef struct {   /* MountainCarEnvParams{T}: MountainCarEnv.jl:3-40 */
    double min_pos, max_pos, max_speed, goal_pos, goal_velocity, power, gravity;
    int64_t max_steps;
} b200rl_mountaincar_params;
typedef struct {   /* AcrobotEnvParams{T} + book_or_nips: 3rd_party/AcrobotEnv.jl:19-60 (max_torque_noise must be 0) */
    double link_length_a, link_length_b, link_mass_a, link_mass_b, link_com_pos_a, link_com_pos_b, link_moi, max_torque_noise,
        max_vel_a, max_vel_b, g, dt;
    int64_t max_steps;
    int32_t book;   /* 1: book_or_nips = "book" (default), 0: "nips" */
} b200rl_acrobot_params;

/* Replaces N x `CartPoleEnv(; T, rng)` / `PendulumEnv` / `MountainCarEnv` constructors
 * (CartPoleEnv.jl:74-79, PendulumEnv.jl:41-66, MountainCarEnv.jl:67-81) and the absent
 * `MultiThreadEnv([...])`.  `rng_state` = (4, N) uint64 host array: raw Xoshiro state per
 * env (Julia side: `Xoshiro(seed_i)` fields s0..s3).  Like the reference constructors it
 * performs one reset!() per env.  Supported: CartPole f32|f64 discrete, f32 continuous; Pendulum f32|f64
 * continuous|discrete; MountainCar f32|f64 discrete|continuous (T = Float64 is the reference constructors' default,
 * PendulumEnv.jl:42, MountainCarEnv.jl:67; the learners / trajectory take Float32 envs and Float64 envs wrapped by
 * b200rl_env_set_state_f32). */
int b200rl_env_create(b200rl_ctx* ctx, int kind, int dtype, int64_t n_envs, const void* params,
                      const uint64_t* rng_state, b200rl_env** out);
int b200rl_env_destroy(b200rl_env* env);
/* MaxTimeoutEnv(env, max_t) (RLEnvs/src/environments/wrappers/MaxTimeoutEnv.jl:17-28): is_terminated(env)
 * also when the wrapper's current_t (= env.t + 1) exceeds max_t; reward(env) still forwards to the wrapped
 * env.  max_t = 0 removes the wrapper. */
int b200rl_env_set_max_timeout(b200rl_env* env, int64_t max_t);
/* StateTransformedEnv(env; state_mapping = s -> Float32.(s)) (RLEnvs/src/environments/wrappers/StateTransformedEnv.jl:15-19):
 * on != 0 lets the learners, the trajectory push and the evaluation take a Float64 env.  The dynamics are untouched (state, RNG
 * streams, t, flags, rewards, episode statistics and FIELD_OBS stay bit for bit the unwrapped env's); the networks read
 * FIELD_OBS_F32, rewards enter a rollout or replay ring as Float32(reward), and a continuous Float32 action reaches the env as
 * Float64(clamp(a, lo, hi)).  On a Float32 env it is the identity (accepted, changes nothing); on Acrobot B200RL_ERR_UNSUPPORTED.
 * on = 0 removes the wrapper. */
int b200rl_env_set_state_f32(b200rl_env* env, int on);
/* Base.copy(env) (RLBase/src/interface.jl:443): deep copy incl. RNG streams */
int b200rl_env_copy(b200rl_env* env, b200rl_env** out);
/* Random.seed!(env, seed) (CartPoleEnv.jl:83): replace the raw RNG states */
int b200rl_env_seed(b200rl_env* env, const uint64_t* rng_state);
/* RLBase.reset!(env) (CartPoleEnv.jl:98-104, PendulumEnv.jl:84-92, MountainCarEnv.jl:99-105).
 * force_all != 0: every env; 0: only envs that are terminated and not yet re-initialised
 * (MultiThreadEnv's soft reset). */
int b200rl_env_reset(b200rl_env* env, int force_all);
/* RLBase.act!(env, a) for all N envs in one kernel (CartPoleEnv.jl:112-140,
 * PendulumEnv.jl:94-118, MountainCarEnv.jl:113-135).  actions: int32 (N,) 1-based for
 * discrete spaces, T (N,) for a continuous action space (Float64 actions for a Float64 env).  auto_reset != 0 fuses the soft reset of
 * envs that just terminated into the same launch (reward/terminal keep the terminating
 * step's values; state/obs become the fresh episode's).
 * actions_on_device: 0 = host buffer borrowed for the call (synchronises before returning), 1 = device pointer,
 * 2 = PINNED host buffer (b200rl_host_alloc) the caller leaves untouched until its next synchronising call on this
 *     ctx — the copy is only stream-ordered, the call does not wait (the per-step action hand-off of the stage protocol). */
int b200rl_env_step(b200rl_env* env, const void* actions, int actions_on_device, int auto_reset);
/* plan!(RandomPolicy(), env) + act!(env, a) fused (RLCore/src/policies/random_policy.jl:29-32):
 * the action is drawn from each env's own Xoshiro stream with rand(rng, Base.OneTo(n)),
 * i.e. the reference default where policy and env share Random.default_rng(). */
int b200rl_env_step_random(b200rl_env* env, int auto_reset);
/* state(env) / reward(env) / is_terminated(env) ...: synchronous copy-out to host */
int b200rl_env_get(b200rl_env* env, int field, void* host_dst, size_t bytes);
/* every field but TERMINAL (bit 0 of FLAGS) is settable, so an env can be restored from a checkpoint:
 * STATE, OBS (a separate buffer only for Pendulum), REWARD, FLAGS, T, RNG, ACTION, EPISODE_RETURN, EPISODE_STATS */
int b200rl_env_set(b200rl_env* env, int field, const void* host_src, size_t bytes);
/* zero-copy device pointer of a field for fused consumers */
int b200rl_env_ptr(b200rl_env* env, int field, void** dptr_out);
/* raises B200RL_ERR_ACTION if any launch since the last check saw an out-of-space action */
int b200rl_env_check(b200rl_env* env);
/* device-side hooks: per-env episode statistics accumulated by the step kernel, the batched
 * form of TotalRewardPerEpisode / BatchStepsPerEpisode (RLCore/src/core/hooks.jl:146-231).
 * out[0] = finished episodes, out[1] = sum of their returns, out[2] = sum of their lengths,
 * out[3] = total env-steps taken.  reset_after != 0 zeroes the counters. */
int b200rl_env_episode_stats(b200rl_env* env, double* out4, int reset_after);
/* device episode log: the per-env lists of TotalRewardPerEpisode / BatchStepsPerEpisode (RLCore/src/core/hooks.jl:146-231)
 * without a host copy per step.  b200rl_env_episode_log attaches a ring of K records per env (K = 0 detaches it, and
 * attaching again starts empty; with the same K it keeps the same ring, so captured agent loops are not re-captured).  The
 * kernels that write it run as instantiations of their own; an env without a log runs the code it ran before the log existed.
 * Every act! that ends an episode (the finished-episode rule of b200rl_env_episode_stats:
 * the MaxTimeoutEnv cut counts, a terminal env stepped again without a reset does not) writes {return, length} to the env's
 * next slot: the return is the Float32 step-order sum of the episode's rewards (FIELD_EPISODE_RETURN), the length env.t.
 * b200rl_env_step / _step_random, the fused rollout, b200rl_onpolicy_iterate, b200rl_replay_run and b200rl_eval_run_episodes write
 * it; b200rl_evaluate / b200rl_evaluate_explore do not (an evaluation is a run of its own).  b200rl_env_copy does not copy it. */
int b200rl_env_episode_log(b200rl_env* env, int32_t K);
/* one record of a flushed list: env = rank * N + i on a sharded ctx (rank of b200rl_comm_rank_world), else i */
typedef struct {
    int64_t env;
    float ret;
    int32_t len;
} b200rl_episode_record;
/* Starts (asynchronously, on the ctx stream) the hand-over of every record logged since the previous flush: host_buf is
 * PINNED host memory (b200rl_host_alloc) of 16 + 16 * capacity bytes, which receives int64 n, int64 overflowing envs, then n
 * b200rl_episode_record ordered by (env, episode).  The caller leaves host_buf alone until b200rl_env_episode_log_read of it
 * returns; a flush every K env steps or less cannot overflow (an episode lasts at least one step). */
int b200rl_env_episode_log_flush(b200rl_env* env, void* host_buf, int64_t capacity);
/* waits for the last flush into host_buf and sets *n_out to its list length.  B200RL_ERR_OVERFLOW when an env finished more
 * than K episodes between the two flushes (its oldest records were overwritten; the message names how many envs) or the list
 * is longer than capacity. */
int b200rl_env_episode_log_read(b200rl_env* env, const void* host_buf, int64_t* n_out);

/* ---------------------------------------------------------------- returns ---------- */
/* generalized_advantage_estimation / discount_rewards / discount_rewards_reduced
 * (RLCore/src/utils/basic.jl:334-417, :138-235, :237-319).  rewards is an (R, C)
 * column-major matrix; dims = 1: each column is a series (time along dim 1), dims = 2: each
 * row is a series (time along dim 2, the PPO (N, T) layout).  values has one extra entry
 * along the time dim.  terminal (uint8, same shape) and init (one per series) may be NULL.
 * on_device = 0: pointers are host arrays (copied in/out, synchronous); 1: device pointers
 * (asynchronous on the ctx stream).  Results are bit-identical to the reference's serial
 * loop (same operation order, no FMA contraction). */
int b200rl_gae_f32(b200rl_ctx* ctx, float* adv, const float* rewards, const float* values,
                   const uint8_t* terminal, float gamma, float lambda, int64_t R, int64_t C,
                   int dims, int on_device);
int b200rl_gae_f64(b200rl_ctx* ctx, double* adv, const double* rewards, const double* values,
                   const uint8_t* terminal, double gamma, double lambda, int64_t R, int64_t C,
                   int dims, int on_device);
int b200rl_discount_rewards_f32(b200rl_ctx* ctx, float* out, const float* rewards,
                                const uint8_t* terminal, const float* init, float gamma,
                                int64_t R, int64_t C, int dims, int on_device);
int b200rl_discount_rewards_f64(b200rl_ctx* ctx, double* out, const double* rewards,
                                const uint8_t* terminal, const double* init, double gamma,
                                int64_t R, int64_t C, int dims, int on_device);
int b200rl_discount_rewards_reduced_f32(b200rl_ctx* ctx, float* out, const float* rewards,
                                        const uint8_t* terminal, const float* init, float gamma,
                                        int64_t R, int64_t C, int dims, int on_device);
int b200rl_discount_rewards_reduced_f64(b200rl_ctx* ctx, double* out, const double* rewards,
                                        const uint8_t* terminal, const double* init, double gamma,
                                        int64_t R, int64_t C, int dims, int on_device);

/* ---------------------------------------------------------------- trajectory ------- */
/* Device-resident CircularArraySARTSTraces (+ CircularPrioritizedTraces) wrapped in an EpisodesBuffer, with a BatchSampler
 * (ReinforcementLearningTrajectories 0.4, external to the reference tree; call sites
 * RLCore/src/policies/agent/agent_base.jl:45-59, agent_srt_cache.jl:30-50; layout
 * docs/src/How_to_implement_a_new_algorithm.md:84-112; length semantics RLCore/test/core/base.jl:20,
 * test/policies/agent.jl:27-34).  `lanes` independent rings of capacity+1 slots, one per sub-env (lanes = 1 is the
 * reference's single stream): every lane keeps its own position, the first state of each of its episodes is a frame of its
 * own, and the entry straddling two episodes counts towards the length but is never sampled.  sampler_rng:
 * (4, batch_size) uint64 host array, one Xoshiro stream per batch slot.  capacity >= 2. */
int b200rl_traj_create(b200rl_ctx* ctx, int ns, int64_t lanes, int64_t capacity, int prioritized, float default_priority,
                       const uint64_t* sampler_rng, int64_t batch_size, b200rl_traj** out);
int b200rl_traj_destroy(b200rl_traj* traj);
/* length(trajectory.container) of lane 0: 0 after the first state, 1 after the first transition
 * (RLCore/test/policies/agent.jl:27-34); lane_lengths: all lanes (== steps + episodes - 1 per lane, test/core/base.jl:20);
 * n_sampleable: entries a sampler may return, summed over the lanes.  All three synchronise. */
int b200rl_traj_length(b200rl_traj* traj, int64_t* frames_out);
int b200rl_traj_lane_lengths(b200rl_traj* traj, int64_t* lengths_out);
int b200rl_traj_n_sampleable(b200rl_traj* traj, int64_t* out);
/* push!(trajectory, (state = s0,))  — the PreEpisodeStage push, agent_base.jl:45-47.  obs: (ns, lanes).
 * push_state = every lane starts an episode; push_episode_start(mode 1) = only the lanes whose last transition was terminal
 * (after a soft reset of the finished sub-envs). */
int b200rl_traj_push_state(b200rl_traj* traj, const float* obs, int on_device);
int b200rl_traj_push_episode_start(b200rl_traj* traj, const float* obs, int on_device, int mode);
/* push!(trajectory, (state = s', action, reward, terminal)) — agent_base.jl:56-59.  terminal: bit0 = is_terminated; bit1 = "the
 * env has already auto-reset, next_obs is the next episode's first state" (the env's FLAGS byte): the episode-start frame is then
 * written by the same call. */
int b200rl_traj_push(b200rl_traj* traj, const int32_t* action, const float* reward, const uint8_t* terminal, const float* next_obs,
                     int on_device);
/* the same, reading the env's device fields directly (no host round trip).  A Float64 env wrapped by b200rl_env_set_state_f32 is
 * accepted: FIELD_OBS_F32 and Float32(reward) are pushed. */
int b200rl_traj_push_env(b200rl_traj* traj, b200rl_env* env, int first_state_only);
/* checkpoint of the ring: field 0 state (ns, lanes, cap+1) f32 | 1 action i32 | 2 reward f32 | 3 flag u8 (bit0 terminal, bit1
 * sampleable) | 4 head (lanes) i32 | 5 count (lanes) i32 | 6 pending (lanes) u8 | 7 n_sampleable i64 | 8 sum tree (2L) f32 |
 * 9 sampler streams (4, B) u64 */
int b200rl_traj_field_bytes(b200rl_traj* traj, int field, size_t* bytes_out);
int b200rl_traj_get(b200rl_traj* traj, int field, void* host_dst, size_t bytes);
int b200rl_traj_set(b200rl_traj* traj, int field, const void* host_src, size_t bytes);
/* sample(trajectory): with replacement, uniform over the sampleable entries (rejection) or proportional to priority (sum-tree
 * descent that never enters an empty subtree); the batch (state, action, reward, terminal, next_state, key, priority, weight) stays
 * on device.  beta: importance-weight exponent, w = (n p / total)^-beta / max w, n = n_sampleable */
int b200rl_traj_sample(b200rl_traj* traj, float beta);
/* NStepBatchSampler(n, gamma) (ReinforcementLearningTrajectories 0.4; DESIGN.md §3): from the next sample on, the drawn entry q
 * (drawn exactly as by the 1-step sampler) opens a window of m <= n entries of its lane that ends early at a terminal entry or
 * before an entry that is not sampleable; the batch then holds reward = the Float32 discounted sum of the window (in
 * discount_rewards' order), terminal = that of entry q+m-1, next_state = state frame q+m, discount = gamma^m, horizon = m.
 * n = 1 is the BatchSampler (the default, with gamma 0.99).  Refused, before any side effect, unless 1 <= n <= min(32, capacity)
 * and gamma is finite in [0, 1].  Configuration, not state: b200rl_traj_get / set do not carry it. */
int b200rl_traj_set_nstep(b200rl_traj* traj, int32_t n, float gamma);
/* field: 0 state (ns,B) | 1 action (B) i32 | 2 reward | 3 terminal u8 | 4 next_state | 5 key i64 |
 * 6 priority | 7 weight | 8 sampler rng (4,B) u64 | 9 discount (B) f32 | 10 horizon (B) i32 (n = 1: gamma and 1) */
int b200rl_traj_batch_get(b200rl_traj* traj, int field, void* host_dst, size_t bytes);
/* priority write-back for the keys of the last sampled batch (trajectory[:priority, keys] = p) */
int b200rl_traj_update_priority(b200rl_traj* traj, const float* priority, int on_device);
int b200rl_traj_total_priority(b200rl_traj* traj, float* out);

/* ---------------------------------------------------------------- networks --------- */
/* kind 0: ActorCritic(actor -> n_out logits, critic -> 1)   (RLCore/src/utils/networks.jl:15-20, 405-432)
 * kind 1: ActorCritic(GaussianNetwork mu/sigma heads, 1-d action; sigma = clamp(softplus(raw)))  (networks.jl:44-116)
 * kind 2: Q-network n_in -> hidden -> hidden -> n_out with a TargetNetwork copy (target_network.jl:27-88)
 * kind 3: dueling Q-network, DuelingNetwork(base = trunk, val = Dense(hidden,1), adv = Dense(hidden,n_out)) (networks.jl:500-522)
 *         with a TargetNetwork copy: Q = (val + adv) - mean(adv), n_out = number of actions (1..3; 4 -> B200RL_ERR_UNSUPPORTED).
 *         Flat vector: trunk, Wv (1 x hidden), bv, Wa (n_out x hidden), ba — Flux.destructure(DuelingNetwork(...)) as it is.
 * Trunks are Dense(n_in,hidden,act) -> Dense(hidden,hidden,act); act 0 relu, 1 tanh; hidden 64|128.
 * Parameters are one flat fp32 vector in Flux.destructure order (weights (out,in) column-major).
 * Q-network entry points (kinds 2 and 3): net_values, net_q_act, net_q_explore, net_act_greedy, evaluate mode 0, evaluate_explore,
 * dqn_update, dqn_last_td, replay_create.  Actor-critic entry points (kinds 0 and 1): net_act, net_ac_step, onpolicy_create, evaluate
 * mode 1; they refuse kinds 2 and 3 before any side effect. */
typedef struct { int32_t n_in, hidden, act, n_out, kind; } b200rl_net_desc;
int b200rl_net_nparams(const b200rl_net_desc* desc, int64_t* out);
/* FluxApproximator(model, Adam) (RLCore/src/policies/learners/flux_approximator.jl:11-46) */
int b200rl_net_create(b200rl_ctx* ctx, const b200rl_net_desc* desc, const float* params_host, b200rl_net** out);
int b200rl_net_destroy(b200rl_net* net);
int b200rl_net_configure_optimizer(b200rl_net* net, float lr, float beta1, float beta2, float eps, float max_grad_norm);
/* actor-critic kinds (0, 1): the critic trunk's activation (0 relu, 1 tanh) when it differs from the actor's (desc->act), e.g.
 * ActorCritic(Chain(Dense(.., relu), ..), Chain(Dense(.., tanh), ..)).  A mixed pair runs the staged launches and the
 * runtime-activation learner kernel (the fused rollout returns B200RL_ERR_UNSUPPORTED for it). */
int b200rl_net_set_critic_act(b200rl_net* net, int act);
/* export / import (checkpoint hooks, docs/src/How_to_use_hooks.md:124-167).
 * which: 0 params | 1 last gradient | 2 Adam m | 3 Adam v | 4 beta^t (2) | 5 target params */
int b200rl_net_get(b200rl_net* net, int which, float* host_dst, int64_t count);
int b200rl_net_set(b200rl_net* net, int which, const float* host_src, int64_t count);
int b200rl_net_ptr(b200rl_net* net, int which, void** dptr_out);
/* optimiser steps taken so far: the TargetNetwork's sync phase (n_optimise, target_network.jl:70-88) — checkpoint / resume */
int b200rl_net_get_step(b200rl_net* net, int64_t* out);
int b200rl_net_set_step(b200rl_net* net, int64_t step);
/* optimise!(::TargetNetwork): target = rho*target + (1-rho)*model (target_network.jl:70-88) */
int b200rl_net_target_sync(b200rl_net* net, float rho);
/* plan!(policy, obs batch): obs (n_in, N); rng_dev (4, N) uint64 DEVICE streams (advanced);
 * action int32 1-based (kind 0) or float (kind 1), log-prob, V(s), raw head outputs (n_head, N).
 * Outputs may be NULL; on_device applies to obs and outputs. */
int b200rl_net_act(b200rl_net* net, const float* obs, int64_t n, uint64_t* rng_dev, void* action_out, float* logp_out, float* value_out,
                   float* heads_out, int on_device);
/* critic V(s) -> (N) for kinds 0/1, Q(s, .) -> (n_out, N) for kinds 2/3 (kind 3: the combined Q) */
int b200rl_net_values(b200rl_net* net, const float* obs, int64_t n, float* out, int use_target, int on_device);
/* QBasedPolicy + EpsilonGreedyExplorer (q_based_policy.jl:13-49, explorers/epsilon_greedy_explorer.jl:69-131); DEVICE pointers */
int b200rl_net_q_act(b200rl_net* net, const float* obs_dev, int64_t n, uint64_t* rng_dev, float epsilon, int32_t* action_out_dev);
/* A value-based explorer applied to a batch the way BatchExplorer does (explorers/batch_explorer.jl:15-21): the inner explorer
 * is called once per column, column i draws from its own stream rng_dev[:, i] (the reference draws all columns from one
 * stream — not parallel; DESIGN.md §3), and for the kinds with a step column i is planned at step + i and the caller advances
 * `step` by n afterwards.  On a sharded ctx (rank r of a communicator of `world` ranks, b200rl_comm_rank_world) the n columns are
 * columns r n .. r n + n - 1 of one BatchExplorer over the world n columns of all ranks: column i is planned at step + r n + i,
 * and the caller advances `step` by world n (the same on every rank).  Per column, on Q = the column's Q-values (n_actions of them):
 *   kind 0 / 1  EpsilonGreedyExplorer{:linear | :exp, is_break_tie} (explorers/epsilon_greedy_explorer.jl:47-112): eps =
 *               get_eps(step + i) (Float64 schedule); u = rand(rng) is always drawn; u >= eps ? findmax(Q)[2] (or, is_break_tie,
 *               rand(rng, find_all_max(Q)[2])) : rand(rng, 1:n_actions)
 *   kind 2      EpsilonSpeedyExplorer(beta) (ReinforcementLearningFarm): the same selection without break-tie, with
 *               eps = exp((beta * -1) * (step + i)) (Float64)
 *   kind 3      WeightedSoftmaxExplorer(): sample(rng, Weights(softmax(Q), 1f0)) — one Float64 draw, Float32 softmax
 *   kind 4      GumbelSoftmaxExplorer(): argmax(logsoftmax(Q) .- log.(-log.(rand(rng, Float32, n_actions)))) — n_actions draws
 * Kinds 3 and 4 have no step (it is advanced but never read).  The fields a kind 2-4 explorer does not read (the epsilon schedule,
 * is_break_tie, and beta for kinds 3 / 4) must be 0.  Refused: an unknown kind, a bad schedule (kinds 0 / 1), a non-finite beta
 * (kind 2), a nonzero field the kind does not read. */
typedef struct {
    double eps_stable, eps_init;
    int64_t warmup_steps, decay_steps;
    int64_t step;            /* explorer.step before this call (the reference starts at 1) */
    int32_t kind;            /* 0 :linear, 1 :exp, 2 speedy, 3 weighted softmax, 4 Gumbel softmax */
    int32_t is_break_tie;
    double beta;             /* kind 2: EpsilonSpeedyExplorer's beta */
} b200rl_explorer;
int b200rl_net_q_explore(b200rl_net* net, const float* obs_dev, int64_t n, uint64_t* rng_dev, const b200rl_explorer* explorer,
                         int32_t* action_out_dev);
/* plan!(greedy policy, obs): findmax of the logits / Q-values (kinds 0, 2, 3; int32 1-based, first maximum wins, NaN ranks
 * highest, -0.0 below 0.0), mu (kind 1; float, unclamped); no RNG.  on_device applies to obs and action_out. */
int b200rl_net_act_greedy(b200rl_net* net, const float* obs, int64_t n, void* action_out, int on_device);

/* ---------------------------------------------------------------- evaluation ------- */
/* run(policy, env, StopAfterNSteps(n_steps)) (RLCore/src/core/run.jl:36-78) with the network's greedy (mode 0, see
 * b200rl_net_act_greedy; a continuous env receives clamp(mu, lo, hi)) or sampling (mode 1, b200rl_net_act's sampler on the
 * (4, N) DEVICE streams policy_rng_dev, advanced; kinds 0 / 1) policy: reset!(env; is_force = true) for every env, then n_steps
 * x {plan!, act!} with the env's in-kernel auto-reset (MaxTimeoutEnv honoured).  Outputs (each may be NULL):
 *   returns (K, N) f32, lengths (K, N) i32 : the first K = max_episodes episodes of each env that end inside the window, the
 *       Float32 sum of their rewards in step order and env.t at termination; slots no episode reaches are left untouched
 *   counts (N) i32                         : episodes each env finished in the window (may exceed K)
 * The env ends where the stage protocol leaves it (every field, its streams and episode statistics); the network and every
 * other handle are only read.  Float32 envs with <= 4 observations, or Float64 ones wrapped by b200rl_env_set_state_f32 (the
 * network reads FIELD_OBS_F32; a record is the Float32 sum of Float32(reward), as the env's EPISODE_RETURN).  on_device = 0: host outputs (synchronises), 1: device
 * outputs (asynchronous on the ctx stream). */
typedef struct { int32_t mode, n_steps, max_episodes; } b200rl_eval_config;   /* mode 0 greedy, 1 sample */
int b200rl_evaluate(b200rl_net* net, b200rl_env* env, const b200rl_eval_config* cfg, uint64_t* policy_rng_dev,
                    float* returns_out, int32_t* lengths_out, int32_t* counts_out, int on_device);
/* run(QBasedPolicy(learner, explorer), env, StopAfterNSteps(n_steps)) for a Q-network (kinds 2 and 3; a dueling head combined into Q
 * first): reset!(env; is_force = true) for every env, then n_steps x {plan!, act!} where plan! is b200rl_net_q_explore's BatchExplorer
 * — column i at window step k is planned at explorer step ex->step + k N + i on its stream explorer_rng_dev[:, i] — or, ex = NULL,
 * GreedyExplorer (the first maximum under `>`, b200rl_net_q_act with epsilon = 0; no draw, no streams needed).  Outputs, env side
 * effects and on_device as b200rl_evaluate; the (4, N) DEVICE explorer streams are advanced in place and, on success, ex->step by
 * N n_steps (as b200rl_replay_run).  The network (its update counter and target too) is only read.  Refused before any side effect:
 * B200RL_ERR_UNSUPPORTED for Float64 envs without b200rl_env_set_state_f32, Acrobot and continuous-action envs; B200RL_ERR_INVALID for a network that is not a Q-network,
 * an input / head width that does not match the env, n_steps < 1, max_episodes < 0, an explorer without streams and a bad explorer
 * (see b200rl_explorer).  One fused launch for hidden = 64 on the tensor-core path.  On a sharded ctx the columns are numbered
 * over the ranks' union as in b200rl_net_q_explore: column i of rank r at window step k plans at ex->step + k world N + r N + i,
 * and ex->step advances by world N n_steps. */
int b200rl_evaluate_explore(b200rl_net* net, b200rl_env* env, int32_t n_steps, int32_t max_episodes, b200rl_explorer* ex,
                            uint64_t* explorer_rng_dev, float* returns_out, int32_t* lengths_out, int32_t* counts_out, int on_device);
/* run(policy, env, StopAfterNSteps | StopAfterNEpisodes(k), hook) for a policy that does not train: the network's greedy (mode 0)
 * or sampling (mode 1, kinds 0 / 1) policy, or QBasedPolicy (mode 2, kinds 2 / 3).  Unlike b200rl_evaluate it continues from the
 * env's current state (run() has force-reset it once), writes no records but the env's episode log when one is attached, and stops
 * on an episode count.  The handle holds the buffers of the episode count across calls; create refuses what b200rl_evaluate[_explore]
 * refuse, with their statuses (a Float64 env without b200rl_env_set_state_f32, Acrobot, mode 1 on a Q-network, a Q-network on a
 * continuous env, an input / head width that does not match).  The net and env must outlive the handle. */
typedef struct b200rl_eval b200rl_eval;
int b200rl_eval_create(b200rl_net* net, b200rl_env* env, int32_t mode, b200rl_eval** out);
int b200rl_eval_destroy(b200rl_eval* h);
/* At most max_steps (>= 1) steps of the stage loop's {plan!, act! with the in-kernel auto-reset, check!}: plan! is mode 0's
 * b200rl_net_act_greedy, mode 1's b200rl_net_act sampler on the (4, N) DEVICE policy streams rng_dev, mode 2's b200rl_net_q_explore
 * (ex; column numbering and ex->step as b200rl_evaluate_explore, on the explorer streams rng_dev) or, ex = NULL, GreedyExplorer.
 * Every env field (streams, statistics and the episode log's records and write counts included) and the streams end bit for bit
 * where the stage loop leaves them; ex->step advances by N · world per step run, only on success; the network is only read.
 * budget < 0 (StopAfterNSteps): exactly max_steps steps, nothing counted (*episodes_done = 0), allocated or synchronised; a sharded
 * ctx is accepted.  budget >= 0 (StopAfterNEpisodes, budget = max(0, k - cur)): stops after s*, *steps_done and *episodes_done as
 * b200rl_onpolicy_run_episodes.  Stretches of at most 1024 steps, one fused evaluation launch each for hidden = 64 on the tensor-core
 * path (staged plan! / act! / count launches otherwise, no host sync per step), and one synchronisation per stretch; a stretch that
 * could reach the budget first copies the env's step arrays and the streams to a shadow (about 100 B per env, allocated by the
 * handle's first call with a budget), and stretches of 64 steps are used once fewer than 64 N episodes remain.  Refused before any
 * side effect: the create checks again, max_steps < 1, an explorer outside mode 2, missing streams, a bad explorer or an explorer
 * step overflow (B200RL_ERR_INVALID; with a budget: when not one more step fits, and a run stops early where the next would not),
 * and a budget on a sharded ctx (B200RL_ERR_UNSUPPORTED). */
int b200rl_eval_run_episodes(b200rl_eval* h, uint64_t* rng_dev, b200rl_explorer* ex, int64_t max_steps, int64_t budget,
                             int64_t* steps_done, int64_t* episodes_done);

/* ---------------------------------------------------------------- on-policy agent -- */
/* PPO (clipped surrogate) / A2C hyper-parameters; defaults of the in-tree example
 * docs/homepage/blog/a_practical_introduction_to_RL.jl/index.html:15238-15286:
 * gamma .99 lambda .95 clip .1 max_grad_norm .5 w 1/.5/.001 Adam(1e-3) update_freq 32 epochs 4 microbatches 4 */
typedef struct {
    float gamma, lambda, clip_range, max_grad_norm, w_actor, w_critic, w_entropy;
    float lr, beta1, beta2, eps;
    float min_sigma, max_sigma;
    int32_t normalize_advantage, n_epochs, n_microbatches, update_freq;
    int32_t algo;   /* 0 PPO, 1 A2C (GAE advantage, discounted-gain critic target) */
} b200rl_onpolicy_config;
typedef struct b200rl_onpolicy b200rl_onpolicy;
/* one optimiser step on explicit HOST minibatch arrays (generic / test entry).
 * losses_out[6] = actor_loss, critic_loss, entropy, loss, grad_norm, 0 */
int b200rl_net_ac_step(b200rl_net* net, const b200rl_onpolicy_config* cfg, const float* states, const void* actions,
                       const float* logp_old, const float* adv, const float* ret, int64_t total, const int32_t* idx, int64_t batch,
                       float adv_mean, float adv_inv_std, int apply_update, float* losses_out);
/* Agent(PPOPolicy | A2CPolicy, PPOTrajectory): rollout tensors (N, T) on the device.  A Float64 env wrapped by
 * b200rl_env_set_state_f32 is accepted: the rollout states are FIELD_OBS_F32, its rewards Float32(reward), and a continuous
 * action reaches the env as Float64(clamp(a, lo, hi)) while the rollout keeps the unclamped Float32 sample. */
int b200rl_onpolicy_create(b200rl_ctx* ctx, b200rl_net* net, b200rl_env* env, const b200rl_onpolicy_config* cfg,
                           const uint64_t* policy_rng, b200rl_onpolicy** out);
int b200rl_onpolicy_destroy(b200rl_onpolicy* agent);
/* plan!(agent, env)  (agent_base.jl:52-54): actions_host (N) may be NULL */
int b200rl_onpolicy_plan(b200rl_onpolicy* agent, void* actions_host);
/* act!(env, planned action) without leaving the device */
int b200rl_onpolicy_act(b200rl_onpolicy* agent);
/* push!(agent, PostActStage, env, action)  (agent_base.jl:56-59) */
int b200rl_onpolicy_push(b200rl_onpolicy* agent);
int b200rl_onpolicy_collect(b200rl_onpolicy* agent, int n_steps);
int b200rl_onpolicy_fill(b200rl_onpolicy* agent, int* t_out, int* T_out);
/* optimise!(agent): GAE + n_epochs x n_microbatches optimiser steps; see algo.cu */
int b200rl_onpolicy_update(b200rl_onpolicy* agent, const int32_t* perm_host, float* stats_host);
/* n_iters x { collect(update_freq); optimise! }: the whole PPO / A2C iteration replayed as ONE CUDA graph launch per iteration
 * (captured on the second iteration; the first one runs eagerly).  Needs an empty rollout.  Same results as collect + update.
 * stats_host: optional (n_epochs * n_microbatches, 6) rows of the last iteration (forces a sync).  This is the path the
 * `_run` specialisation takes between hook calls (RLCore/src/core/run.jl:52-68 — plan!, act!, push!, optimise! for
 * update_freq steps) when no host-side hook needs per-step data. */
int b200rl_onpolicy_iterate(b200rl_onpolicy* agent, int n_iters, float* stats_host);
int b200rl_onpolicy_graph_active(b200rl_onpolicy* agent, int* out);   /* 1: iterate replays a captured graph */
/* run(agent, env, StopAfterNSteps | StopAfterNEpisodes(k)) on the fused path, for at most max_steps env steps; max_steps: the
 * longest window between two flushes of an episode log.  The result equals the stage loop's (plan!, act!, push!, optimise!, check
 * per step) bit for bit: a rollout completed inside the run is updated, a part-filled one stays so (b200rl_onpolicy_fill) and the
 * next call continues it.  Each stretch is the rest of the rollout; whole rollouts that cannot reach a budget run as
 * b200rl_onpolicy_iterate, one graph launch each.  stats_host: as b200rl_onpolicy_iterate, rows of the last update run (untouched
 * when none ran).
 * budget < 0 (StopAfterNSteps): no episodes are counted (*episodes_done = 0), nothing is allocated and nothing synchronises per
 * stretch; the run returns at the last rollout boundary inside max_steps if there is one (*steps_done = the steps up to it), so that
 * a caller's window never splits a whole-rollout graph launch, and otherwise runs max_steps steps.  A sharded ctx is accepted.
 * budget >= 0 (StopAfterNEpisodes(k), budget = max(0, k - cur); RLCore/src/core/stop_conditions.jl:82-118, batched: every lane
 * whose is_terminated is true after a step counts one episode, a MaxTimeoutEnv cut included): the loop runs steps 1 .. s*, s* =
 * the first step after which the episodes counted reach budget (budget 0: exactly one step, as the stage loop checks only after a
 * step), or max_steps steps when the budget is not reached.  *steps_done = steps run, *episodes_done = episodes those steps ended
 * (>= budget when the budget was reached; may overshoot it).  Each stretch that could reach the budget (N · steps >= budget -
 * episodes so far) first copies the env arrays, policy streams and rollout columns to a shadow (allocated by the agent's first call
 * with a budget, then kept: about the rollout's size again); a counting kernel reduces the stretch's terminal columns per step and
 * finds the crossing; a crossing before the stretch's last step restores the shadow and runs collect(s*).  One synchronisation per
 * stretch.  A sharded ctx (world > 1) is refused with B200RL_ERR_UNSUPPORTED before any side effect. */
int b200rl_onpolicy_run_episodes(b200rl_onpolicy* agent, int64_t max_steps, int64_t budget, float* stats_host, int64_t* steps_done,
                                 int64_t* episodes_done);
/* field: 0 state (ns,N,T+1) | 1 action | 2 logp | 3 reward | 4 terminal u8 | 5 value (N,T+1) |
 * 6 advantage | 7 return | 8 policy rng (4,N) u64 | 9 {adv mean, inv std} */
int b200rl_onpolicy_get(b200rl_onpolicy* agent, int field, void* host_dst, size_t bytes);
/* Checkpoint / resume (the JLD2 hook pattern, docs/src/How_to_use_hooks.md:124-167): together with b200rl_net_get/set
 * (parameters, Adam moments, beta^t, target) and b200rl_env_get/set (every env field) these restore a run bit for bit, at a
 * rollout boundary or in the middle of a rollout.  onpolicy_set takes fields 0-5 and 8 of b200rl_onpolicy_get;
 * counters3 = {rollout fill level t, updates done by the agent (keys the minibatch permutation), optimiser steps of the net}. */
int b200rl_onpolicy_set(b200rl_onpolicy* agent, int field, const void* host_src, size_t bytes);
int b200rl_onpolicy_export_state(b200rl_onpolicy* agent, int64_t* counters3_out);
int b200rl_onpolicy_import_state(b200rl_onpolicy* agent, const int64_t* counters3);

/* measurement aid: average device ms of `reps` back-to-back launches of one hot-path kernel on the
 * agent's tensors (0 loss+backward, 1 policy inference, 2 env step, 3 GAE, 4 reduce+clip+Adam) */
int b200rl_onpolicy_time_kernel(b200rl_onpolicy* agent, int which, int reps, float* avg_ms_out);

/* ---------------------------------------------------------------- DQN -------------- */
typedef struct {
    float gamma, lr, beta1, beta2, eps, max_grad_norm, rho;
    float per_alpha, per_beta, per_eps;
    int32_t huber, double_dqn, target_update_freq;
} b200rl_dqn_config;
/* optimise!(DQNLearner / PrioritizedDQNLearner): sample, TD loss + backward, clip + Adam,
 * priority write-back, target sync.  stats_host[4] = loss, grad_norm, mean|td|, n_updates (NULL: async).
 * With an n-step sampler (n > 1) the target is R = reward + discount * (1 - terminal) * q'(next_state), and a trajectory whose
 * n-step gamma differs from cfg->gamma is refused before any side effect. */
int b200rl_dqn_update(b200rl_net* net, b200rl_traj* traj, const b200rl_dqn_config* cfg, float* stats_host);
int b200rl_dqn_last_td(b200rl_net* net, b200rl_traj* traj, float* host_dst, int64_t count);

/* ---------------------------------------------------------------- DQN agent loop --- */
/* InsertSampleRatioController(ratio, threshold) (ReinforcementLearningTrajectories 0.4): one insertion = one pushed frame of
 * every lane; after it, batches are sampled while n_inserted >= threshold and n_sampled <= (n_inserted - threshold) * ratio
 * (Float64 product, as the Julia / Python controller computes it). */
typedef struct { double ratio; int64_t threshold, n_inserted, n_sampled; } b200rl_insert_sample_ratio;
typedef struct b200rl_replay b200rl_replay;
/* run(Agent(QBasedPolicy(DQNLearner, explorer), Trajectory), env, StopAfterNSteps(n)) (RLCore/src/core/run.jl:52-68) on the
 * device, for a hook with nothing to do per step: n_steps x {plan! (BatchExplorer over Q(state(env), .)), act!, push!(trajectory),
 * optimise! (one DQN update per batch the controller allows)}.  act! ALWAYS uses the in-kernel auto-reset (b200rl_env_step(..., 1))
 * and honours MaxTimeoutEnv: drive a soft-reset env through the stage protocol instead.  A stretch of steps without an update is
 * ONE collect launch for H = 64 on the tensor-core path (replay_collect_tc_kernel; the sum tree is rebuilt once per stretch) and
 * staged launches otherwise; each "1 step + m updates" unit is replayed from a CUDA graph keyed by m (captured on its second use).
 * Results equal the stage protocol's bit for bit (the FP64 return sum of the episode statistics may differ in its last bits
 * where rewards are not integers).  The explorer step, the update counter and the controller counters advance on the host by
 * arithmetic.  The trajectory keeps (min(2k + 1, capacity + 1), N) touched-leaf keys for the longest stretch k (prioritised).
 * create refuses, before any side effect: a network that is not a Q-network, a Float64 / continuous-action / Acrobot env,
 * trajectory lanes != N or a state width that does not match, a sharded ctx with neither the peer exchange attached nor an NCCL
 * communicator, an n-step gamma != cfg->gamma (also refused by run).  The trajectory needs a sampler; a change of its n-step
 * setting between runs re-captures the graphs.
 *
 * Sharded (a ctx whose communicator has world G > 1; one process per GPU, DESIGN.md §3): G ranks of N envs each run what
 * run(Agent(QBasedPolicy(DQNLearner, explorer), Trajectory), env, StopAfterNSteps(n)) runs over G N envs, in this sense:
 *   1. Envs, rings, sum trees and sampler streams are per rank: rank r owns global envs [r N, (r + 1) N), its env and explorer
 *      streams are keyed by the global env index, its trajectory holds only its own lanes.
 *   2. Explorer columns are numbered globally: column i of rank r plans at explorer step s + r N + i, and a plan! advances the
 *      step by G N — one BatchExplorer over the G N columns (see b200rl_net_q_explore).
 *   3. Each update draws B per rank: the global batch is G B, the gradient their mean (1 / (B G)), one exchange per update.  PER
 *      weights stay per rank, (N_r P_r(i))^-beta normalised over the rank's own batch — not one prioritised ring over the union.
 *   4. Every rank runs the same InsertSampleRatioController schedule, hence the same updates per step and the target sync at the
 *      same update: parameters, Adam state and target stay bit-identical on all ranks.
 *   5. stats4: loss and grad_norm are global, mean |td| is the rank's own.
 *   6. Each run starts with one small all-reduce in which the ranks compare N, B, n_steps, the controller (ratio, threshold,
 *      counters), the explorer (kind, schedule, step), a digest of the DQN config and the n-step setting; if any differs — or a
 *      rank refuses the run for a reason of its own — every rank returns B200RL_ERR_INVALID with nothing else touched.
 * The update units are replayed as CUDA graphs when the peer exchange is attached and every rank owns its device
 * (b200rl_comm_p2p_set_exclusive); with NCCL only, or ranks sharing a device, they launch eagerly. */
/* A Float64 env wrapped by b200rl_env_set_state_f32 is accepted (the ring stores FIELD_OBS_F32 and Float32(reward)); whether the
 * wrapper is in effect (a wrapped Float64 env; on a Float32 env it changes nothing) takes part in the graph key and, on a sharded
 * ctx, in the agreement of point 6. */
int b200rl_replay_create(b200rl_ctx* ctx, b200rl_net* q, b200rl_env* env, b200rl_traj* traj, const b200rl_dqn_config* cfg,
                         b200rl_replay** out);
/* explorer_rng_dev: (4, N) DEVICE explorer streams (one per env, advanced).  ex: any b200rl_explorer kind (its step is advanced
 * by n_steps * N * world), NULL = GreedyExplorer (findmax, no draw).  ctl: counters advanced.  stats4 (may be NULL; synchronises):
 * loss, grad_norm, mean |td|, n_updates of the last update in the window (untouched when the window ran none).  Refuses a bad
 * explorer schedule or controller values before any side effect.  A CUDA error part-way through returns with the device state
 * advanced and *ex / *ctl NOT advanced: the run cannot be continued from them. */
int b200rl_replay_run(b200rl_replay* r, uint64_t* explorer_rng_dev, b200rl_explorer* ex, b200rl_insert_sample_ratio* ctl,
                      int64_t n_steps, float* stats4);
/* run(Agent(QBasedPolicy(DQNLearner, explorer), Trajectory), env, StopAfterNSteps | StopAfterNEpisodes(k)) on the device, for at
 * most max_steps env steps: budget, *steps_done and *episodes_done as b200rl_onpolicy_run_episodes.  budget < 0: b200rl_replay_run
 * (max_steps) (a sharded ctx is accepted).  budget >= 0: step s* runs with its updates, target sync and controller / explorer
 * counters: what b200rl_replay_run(s*) does.  Chunks of at most min(capacity / 2, 2048) steps (the ring then still holds every frame
 * a chunk pushed) run as b200rl_replay_run; a chunk that could reach the budget first copies the env arrays, the ring (frames,
 * heads, counts, sum tree, sampler streams), the explorer streams and the Q-network (parameters, Adam moments, beta^t, target, last
 * loss / TD) to a shadow allocated by the handle's first call with a budget and kept (about the ring's size again: a configuration
 * near the device's memory can fail here with B200RL_ERR_OOM).  A counting kernel reduces the terminal flags the chunk pushed per
 * step; a crossing before the chunk's last step restores the shadow and the host counters (*ex, *ctl, update and step counters) and
 * runs b200rl_replay_run(s*).  stats4: as b200rl_replay_run, for the last update run.  With a budget, a sharded ctx (world > 1) is
 * refused with B200RL_ERR_UNSUPPORTED before any side effect. */
int b200rl_replay_run_episodes(b200rl_replay* r, uint64_t* explorer_rng_dev, b200rl_explorer* ex, b200rl_insert_sample_ratio* ctl,
                               int64_t max_steps, int64_t budget, float* stats4, int64_t* steps_done, int64_t* episodes_done);
int b200rl_replay_graph_active(b200rl_replay* r, int* out);   /* 1: a "1 step + m updates" unit has been captured and replayed */
int b200rl_replay_destroy(b200rl_replay* r);

/* select the wgmma tensor-core kernels (default, H = 64) or the FP32 CUDA-core kernels for the dense layers */
int b200rl_set_tensor_cores(int enable);
/* 1 (default; B200RL_FUSED_STEP=0 in the environment starts with 0): the on-policy update runs reduce + [peer exchange] + clip +
 * Adam in the tail of the tensor-core loss + backward launch (one launch per optimiser step); 0: a second kernel does it.
 * Both orders of summation over the gradient partials are identical; process-wide, like b200rl_set_tensor_cores. */
int b200rl_set_fused_step(int enable);
/* ---------------------------------------------------------------- multi-GPU -------- */
/* env-index data parallelism: one process per GPU, one sum all-reduce of the flat gradient per
 * optimiser step over NCCL / NVLink (SURVEY §8e).  rank 0 makes the 128-byte id. */
int b200rl_comm_unique_id(void* id128_out);
int b200rl_comm_init(b200rl_ctx* ctx, int nranks, int rank, const void* id128);   /* id128 NULL: no NCCL, peer exchange only */
/* Fused all-reduce over NVLink / NVSwitch peer memory (ranks of one node).  Each rank exports a small exchange region
 * (export), maps every other rank's (open: 64-byte CUDA IPC handle of another process; or the raw pointer when the peer
 * lives in the same process) and attaches the table.  After attach the optimiser step of a sharded run is ONE kernel:
 * reduce the per-CTA gradient partials -> publish to the own region -> read every peer's region -> sum in rank order
 * (bit-identical on all ranks) -> global-norm clip -> Adam; NCCL is then only used for buffers larger than the region. */
int b200rl_comm_p2p_export(b200rl_ctx* ctx, void* handle64_out, void** region_out);
int b200rl_comm_p2p_open(b200rl_ctx* ctx, const void* handle64, void** region_out);
int b200rl_comm_p2p_attach(b200rl_ctx* ctx, void* const* regions);
/* PCI bus id of the ctx's device ("0000:1b:00.0", NUL-terminated, len >= 16): lets the ranks of a job find out whether they
 * all drive different GPUs.  b200rl_comm_p2p_set_exclusive(ctx, 1) then declares it (call after attach, same value on every
 * rank): only with one rank per device may a whole-device kernel wait for its peers inside itself, which is what the fused
 * loss + backward + exchange + optimiser-step launch does; otherwise (default for IPC-mapped peers) the exchange stays in
 * its own small kernel.  attach() sets the flag itself for peers of the same process (raw pointers). */
int b200rl_ctx_pci_bus_id(b200rl_ctx* ctx, char* out, int len);
int b200rl_comm_p2p_set_exclusive(b200rl_ctx* ctx, int exclusive);
int b200rl_comm_allreduce_f32(b200rl_ctx* ctx, float* dev_buf, int64_t n);
/* rank and number of ranks of the ctx's communicator (0 and 1 without one): the column offset rank N and the explorer step
 * stride world N of a sharded QBasedPolicy (b200rl_net_q_explore) */
int b200rl_comm_rank_world(b200rl_ctx* ctx, int* rank, int* world);

#ifdef __cplusplus
}
#endif
#endif /* B200RL_H */
