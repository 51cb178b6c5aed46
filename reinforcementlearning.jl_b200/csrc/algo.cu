// algo.cu — host-side orchestration behind the C ABI: network handle (FluxApproximator +
// optimiser state + TargetNetwork), the on-policy agent (PPO / A2C: plan! -> act! -> push! ->
// optimise!), the DQN update on a prioritised trajectory and the DQN agent loop (plan! -> act! ->
// push! -> optimise! with the updates replayed as CUDA graphs).  All arithmetic is in the
// kernels of nn.cu / returns.cu / traj.cu / env.cu; this file sequences launches on the ctx
// stream and owns the rollout tensors.
//
// Reference anchors: Agent stage pushes RLCore/src/policies/agent/agent_base.jl:45-66;
// FluxApproximator/optimise! policies/learners/flux_approximator.jl:11-46; TargetNetwork
// target_network.jl:27-88; PPO/A2C/DQN update rules: ReinforcementLearningZoo (absent from the
// snapshot; SURVEY Appendix B), hyper-parameters docs/homepage/blog/a_practical_introduction_to_RL.jl/index.html:15238-15286.
#include <map>

#include "greedy.cuh"
#include "internal.h"
#include "nn.cuh"
#include "replay_schedule.h"
#include "ring.cuh"
#include "stop_episodes.cuh"

static void* env_field(b200rl_env* e, int f) { void* p = nullptr; b200rl_env_ptr(e, f, &p); return p; }
// the observation the networks read; refuses a Float64 env that is not wrapped by b200rl_env_set_state_f32 (and Acrobot)
static int learner_obs(b200rl_env* e, const float** obs) {
    *obs = b200rl_env_internal_obs_f32(e);
    REQUIRE(*obs, B200RL_ERR_UNSUPPORTED,
            "the networks read Float32 observations: construct the env with T = Float32 or wrap it in StateTransformedEnv(env, Float32) "
            "(b200rl_env_set_state_f32)");
    return B200RL_OK;
}

namespace {
// D = double: the action a Float64 env receives, Float64(clamp(a, lo, hi))
template <class D>
__global__ void clamp_copy_kernel(D* __restrict__ dst, const float* __restrict__ src, int64_t n, float lo, float hi) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = (D)fminf(fmaxf(src[i], lo), hi);
}
// plan!(greedy policy) on the (nout, N) head outputs: raw action bits (greedy.cuh); clamp != 0: a continuous action is
// handed to the env as clamp(mu, lo, hi)
__global__ void greedy_select_kernel(const float* __restrict__ heads, MlpDesc d, int64_t n, int clamp, float lo, float hi,
                                     uint32_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float z[kOutMax];
#pragma unroll
    for (int o = 0; o < kOutMax; ++o) z[o] = o < d.nout ? heads[(int64_t)d.nout * i + o] : 0.f;
    uint32_t a = greedy::greedy_action(d, z);
    if (clamp) a = __float_as_uint(fminf(fmaxf(__uint_as_float(a), lo), hi));
    out[i] = a;
}
// staged b200rl_evaluate, after each act!: per-env Float32 return (rewards added in step order, like the env's EPISODE_RETURN)
// and length; an episode that ended is recorded in slot cnt (< K) of its env
__global__ void eval_record_kernel(const float* __restrict__ reward, const uint8_t* __restrict__ flags, int64_t n, int K,
                                   float* __restrict__ acc_ret, int32_t* __restrict__ acc_len, int32_t* __restrict__ cnt,
                                   float* __restrict__ returns, int32_t* __restrict__ lengths) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float ret = __fadd_rn(acc_ret[i], reward[i]);
    const int32_t len = acc_len[i] + 1;
    if (flags[i] & 1) {
        const int e = cnt[i];
        if (e < K) {
            if (returns) returns[(size_t)K * i + e] = ret;
            if (lengths) lengths[(size_t)K * i + e] = len;
        }
        cnt[i] = e + 1;
        acc_ret[i] = 0.f;
        acc_len[i] = 0;
    } else {
        acc_ret[i] = ret;
        acc_len[i] = len;
    }
}
__global__ void copy_f32_kernel(float* __restrict__ dst, const float* __restrict__ src, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i];
}
__global__ void stats_row_kernel(float* __restrict__ row, const float* __restrict__ loss4, const float* __restrict__ gnorm,
                                 unsigned int* __restrict__ tick) {
    if (threadIdx.x < 4) row[threadIdx.x] = loss4[threadIdx.x];
    if (threadIdx.x == 4) row[4] = *gnorm;
    if (threadIdx.x == 5 && tick) *tick += 1u;
}
// After GAE: one 32-byte record per rollout sample {state (zero padded to 4), action bits, logp_old, advantage, return}, so the
// randomly permuted minibatch gather of K7 touches ONE DRAM sector per sample instead of one per array (5 arrays: ~4x the
// algorithmic bytes).  Streaming: 32 B read + 32 B written per sample, fully coalesced.
template <int NS>
__global__ void __launch_bounds__(256) pack_records_kernel(float4* __restrict__ rec, const float* __restrict__ states, const uint32_t* __restrict__ actions,
                                                          const float* __restrict__ logp, const float* __restrict__ adv, const float* __restrict__ ret,
                                                          int64_t total) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= total) return;
    float4 st = make_float4(0.f, 0.f, 0.f, 0.f);
    if (NS == 4) st = reinterpret_cast<const float4*>(states)[j];
    else {
        float x[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int i = 0; i < NS; ++i) x[i] = states[(int64_t)NS * j + i];
        st = make_float4(x[0], x[1], x[2], x[3]);
    }
    float4 sc = make_float4(__uint_as_float(actions[j]), logp[j], adv[j], ret[j]);
    // 32 lanes x 32 B = 1 KB contiguous per warp: two 16-byte stores per thread land in the same sector
    rec[2 * j] = st;
    rec[2 * j + 1] = sc;
}
__global__ void sum_norm_partials_kernel(const double* __restrict__ partials, int n, double* __restrict__ out2) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        double a = 0, b = 0;
        for (int k = 0; k < n; ++k) { a += partials[2 * k]; b += partials[2 * k + 1]; }
        out2[0] = a; out2[1] = b;
    }
}
__global__ void finalize_norm2_kernel(const double* __restrict__ sums2, double count, float* __restrict__ out2) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        double mean = sums2[0] / count;
        double var = (sums2[1] - count * mean * mean) / (count - 1.0);
        if (var < 0) var = 0;
        float sd = (float)sqrt(var);
        sd = sd < 1e-8f ? 1e-8f : (sd > 1000.0f ? 1000.0f : sd);
        out2[0] = (float)mean;
        out2[1] = 1.0f / sd;
    }
}
}  // namespace

// a continuous action as the env receives it: clamp(a, lo, hi) of its action space, in the env's T (dst holds N of them)
static int env_action_clamped(b200rl_env* env, const float* a, int64_t N, void* dst) {
    b200rl_ctx* ctx = b200rl_env_internal_ctx(env);
    const float bound = b200rl_env_internal_action_bound(env);
    if (b200rl_env_internal_dtype(env) == B200RL_F64)
        clamp_copy_kernel<double><<<grid_for(N, 256), 256, 0, ctx->stream>>>((double*)dst, a, N, -bound, bound);
    else
        clamp_copy_kernel<float><<<grid_for(N, 256), 256, 0, ctx->stream>>>((float*)dst, a, N, -bound, bound);
    LAUNCH_CHECK(ctx);
    return B200RL_OK;
}

// ------------------------------------------------------------------ network handle ---------
struct b200rl_net {
    b200rl_ctx* ctx;
    int kind;  // 0 actor-critic categorical, 1 actor-critic gaussian, 2 Q-network, 3 dueling Q-network
    MlpDesc actor, critic;
    int64_t np;
    float *params, *grad, *m, *v, *beta_t, *target;
    float* partial; int n_partials;
    float* loss_partial; float* loss4; float* gnorm;
    double* cta_sumsq; unsigned int* counters;
    float lr, b1, b2, eps, max_grad_norm;
    uint64_t n_updates;
};

// The operands of one optimiser step on n with the hyperparameters of an on-policy or DQN config c.  stats_row (may be null, and
// then so is tick): the row {4 loss sums, grad norm} of this step; tick: the device update counter, incremented once by the step.
template <class Config>
static OptStep opt_step(const b200rl_net* n, const Config& c, float* stats_row = nullptr, unsigned int* tick = nullptr) {
    OptStep st = {};
    st.params = n->params; st.grad = n->grad; st.m = n->m; st.v = n->v; st.beta_t = n->beta_t;
    st.loss_out4 = n->loss4; st.stats_row = stats_row; st.gnorm_out = n->gnorm;
    st.cta_sumsq = n->cta_sumsq; st.counters = n->counters; st.tick = tick;
    st.max_norm = c.max_grad_norm; st.lr = c.lr; st.b1 = c.beta1; st.b2 = c.beta2; st.eps = c.eps;
    return st;
}

// One optimiser step on the gradient partials of a loss + backward launch: reduce [-> all-reduce over the ranks] ->
// clip_by_global_norm! -> Adam.  One kernel (nn_reduce_clip_adam) when its CTAs can all be co-resident and the ranks, if any,
// exchange over the peer memory; the staged kernels otherwise.
static int optimiser_step(b200rl_net* n, int n_partials, int n_loss, const OptStep& st) {
    b200rl_ctx* ctx = n->ctx;
    const int world = b200rl_comm_world(ctx);
    P2PTable peers;
    if ((world == 1 || b200rl_comm_p2p_table(ctx, &peers)) && (int)grid_for(n->np, 256) <= ctx->sm_count)
        return nn_reduce_clip_adam(ctx, n->partial, n_partials, n->np, n->loss_partial, n_loss, st);
    TRY(nn_reduce_partials(ctx, n->partial, n_partials, n->np, n->grad, n->loss_partial, n_loss, n->loss4));
    if (world > 1) {
        TRY(b200rl_comm_allreduce_internal(ctx, n->grad, n->np, 0));
        TRY(b200rl_comm_allreduce_internal(ctx, n->loss4, 4, 0));
    }
    TRY(nn_clip_adam(ctx, n->np, st));
    if (st.stats_row) {
        stats_row_kernel<<<1, 32, 0, ctx->stream>>>(st.stats_row, n->loss4, n->gnorm, st.tick);
        LAUNCH_CHECK(ctx);
    }
    return B200RL_OK;
}

// ------------------------------------------------------------------ CUDA-graph replay unit --
// A stretch of launches (the body) that an agent loop runs over and over, replayed as one CUDA graph per unit id.  The first
// use of an id runs the body eagerly (lazy module loading, function attributes, scratch growth), the second captures it, every
// later one launches the graph.  Capture does not execute, so the host counters the captured calls advanced are measured,
// rolled back, and advanced by the same amount on every launch: the host sees what an eager run leaves.  A capture or
// instantiation that fails switches the unit to eager launches for good.
struct HostCounters {
    uint64_t launches, net_updates, env_steps, agent_updates;
    int64_t pushed;
    HostCounters operator-(const HostCounters& o) const {
        return {launches - o.launches, net_updates - o.net_updates, env_steps - o.env_steps, agent_updates - o.agent_updates, pushed - o.pushed};
    }
};
struct CounterSet {   // where a body's host counters live; traj and agent_updates may be null
    b200rl_ctx* ctx; b200rl_net* net; b200rl_env* env; b200rl_traj* traj; uint64_t* agent_updates;
    HostCounters read() const {
        return {ctx->launches, net->n_updates, b200rl_env_internal_steps(env), agent_updates ? *agent_updates : 0,
                traj ? b200rl_traj_internal_pushed(traj) : 0};
    }
    void add(const HostCounters& d) const {
        ctx->launches += d.launches; net->n_updates += d.net_updates;
        b200rl_env_internal_add_steps(env, d.env_steps);
        if (agent_updates) *agent_updates += d.agent_updates;
        if (traj) b200rl_traj_internal_add_pushed(traj, d.pushed);
    }
};
class GraphUnit {
    struct Unit { cudaGraphExec_t exec = nullptr; bool warmed = false; HostCounters delta{}; };
    std::map<int64_t, Unit> units_;
    std::vector<unsigned char> key_;
    bool failed_ = false;
    void drop() {
        for (auto& kv : units_) if (kv.second.exec) { cudaGraphExecDestroy(kv.second.exec); kv.second.exec = nullptr; }
    }
public:
    ~GraphUnit() { drop(); }
    bool active() const {
        for (const auto& kv : units_) if (kv.second.exec) return true;
        return false;
    }
    // what the captured launches bake in besides the handles (compared bytewise): a change re-captures every unit
    void rekey(const void* key, size_t bytes) {
        const unsigned char* k = (const unsigned char*)key;
        if (key_.size() == bytes && memcmp(key_.data(), k, bytes) == 0) return;
        drop();
        key_.assign(k, k + bytes);
    }
    // capturable = false: run the body eagerly (a measurement run, or launches a graph cannot hold)
    template <class Body>
    int run(int64_t id, const CounterSet& cs, bool capturable, Body&& body) {
        b200rl_ctx* ctx = cs.ctx;
        Unit& u = units_[id];
        if (!u.warmed || !capturable || failed_ || ctx->phase_base >= 0) {
            u.warmed = true;
            return body();
        }
        if (!u.exec) {
            const HostCounters c0 = cs.read();
            CUDA_TRY(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
            const int st = body();
            cudaGraph_t g = nullptr;
            const cudaError_t ce = cudaStreamEndCapture(ctx->stream, &g);
            u.delta = cs.read() - c0;
            cs.add(c0 - cs.read());
            cudaError_t ie = cudaErrorUnknown;
            if (st == B200RL_OK && ce == cudaSuccess && g) ie = cudaGraphInstantiate(&u.exec, g, 0);
            if (g) cudaGraphDestroy(g);
            if (ie != cudaSuccess) {
                cudaGetLastError();
                u.exec = nullptr;
                failed_ = true;
                return body();
            }
        }
        CUDA_TRY(cudaGraphLaunch(u.exec, ctx->stream));
        cs.add(u.delta);
        return B200RL_OK;
    }
};

// ------------------------------------------------------------------ fused runs ---------------
// b200rl_onpolicy_run_episodes / b200rl_replay_run_episodes (run_stretches below) run a stretch of steps ahead and roll it back when
// the episode budget is reached inside it (stop_episodes.cuh).  Shadow: the device state such a stretch changes, copied aside
// before it (mark) and copied back (restore) in one launch each.  Its buffer is allocated by the handle's first call with an
// episode budget (stop_buffers).
static size_t round256(size_t b) { return (b + 255) / 256 * 256; }
struct Shadow {
    char* buf = nullptr;
    size_t cap = 0, used = 0;
    stop::Regions g{};
    void clear() { g.n = 0; used = 0; }
    int add(void* p, size_t bytes) {
        REQUIRE(g.n < stop::kMaxRegions && used + round256(bytes) <= cap, B200RL_ERR_INVALID, "shadow buffer too small");
        g.state[g.n] = (char*)p; g.shadow[g.n] = buf + used; g.bytes[g.n] = bytes;
        ++g.n; used += round256(bytes);
        return B200RL_OK;
    }
    int add_regions(const DevRegion* r, int n) {
        for (int k = 0; k < n; ++k) TRY(add(r[k].p, r[k].bytes));
        return B200RL_OK;
    }
    int copy(b200rl_ctx* ctx, bool to_shadow) const {
        size_t most = 0;
        for (int k = 0; k < g.n; ++k) most = g.bytes[k] > most ? g.bytes[k] : most;
        if (!g.n || !most) return B200RL_OK;
        const unsigned cap_x = (unsigned)(4 * (ctx->sm_count > 0 ? ctx->sm_count : 132));
        unsigned x = grid_for((int64_t)((most + 15) / 16), 256);
        stop::copy_regions_kernel<<<dim3(x < cap_x ? x : cap_x, (unsigned)g.n), 256, 0, ctx->stream>>>(g, to_shadow ? 1 : 0);
        LAUNCH_CHECK(ctx);
        return B200RL_OK;
    }
};
// Per-step counts of one stretch and its crossing: `counts` (s + 2 entries; the last two receive {s*, episodes}; zeroed before the
// stretch ran, which may have counted already), `count` launches the counting kernel, the crossing is read back through the pinned
// pair `host` (synchronises: once per stretch).
template <class Count>
static int stop_crossing(b200rl_ctx* ctx, unsigned long long* counts, int64_t s, int64_t remaining, long long* host, Count&& count,
                         StopCrossing* out) {
    TRY(count());
    long long* dev_out = (long long*)(counts + s);
    stop::crossing_kernel<<<1, 1, 0, ctx->stream>>>(counts, s, remaining, dev_out);
    LAUNCH_CHECK(ctx);
    CUDA_TRY(cudaMemcpyAsync(host, dev_out, 2 * sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    *out = StopCrossing{host[0], host[1]};
    return B200RL_OK;
}

// The buffers of a run with an episode budget, allocated by the handle's first such run and kept (an agent that never stops on an
// episode count holds none; later runs allocate nothing): the shadow, per-step counts of the longest stretch + {s*, episodes}, the
// pinned pair.
struct StopBuffers {
    Shadow shadow;
    unsigned long long* counts = nullptr;
    long long* host = nullptr;
    int alloc(b200rl_ctx* ctx, size_t shadow_bytes, int64_t longest) {
        if (shadow.buf) return B200RL_OK;
        CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        CUDA_TRY(cudaMalloc(&counts, (size_t)(longest + 2) * sizeof(unsigned long long)));
        CUDA_TRY(cudaHostAlloc(&host, 2 * sizeof(long long), cudaHostAllocDefault));
        CUDA_TRY(cudaMalloc(&shadow.buf, shadow_bytes));
        shadow.cap = shadow_bytes;
        return B200RL_OK;
    }
    void release() { cudaFree(shadow.buf); cudaFree(counts); cudaFreeHost(host); }
};

/* The one loop of a fused run: at most max_steps env steps of run(agent, env, StopAfterNSteps | StopAfterNEpisodes), cut into
 * stretches by the agent (`ops`: OnPolicyStretches, ReplayStretches, EvalStretches).  budget >= 0: a stretch that could reach the budget
 * (N · s >= budget - episodes so far) is marked first; the terminal flags it wrote are counted; if the budget is reached before its
 * last step, the mark and the host counters are restored and its first s* steps run instead.  budget < 0: nothing is marked or
 * counted — no allocation and no synchronisation per stretch, so a sharded ctx may run it — and the run returns at the agent's
 * last boundary (the end of a rollout) inside max_steps, if there is one: a window of the caller never splits a rollout that
 * would otherwise run as one graph launch.
 * Ops: Saved save() / restore(Saved) of the host counters; shadow_bytes() and longest() (stretch) of the buffers; mark() the
 * device state into the shadow; stretch(left, counting, remaining) -> s; run(s, may_stop), which may add the per-step counts itself
 * (the counts are zeroed before it); count(s, Saved) launches the counting kernel; end_stretch() after the count; at_boundary(left). */
template <class Ops>
static int run_stretches(b200rl_ctx* ctx, StopBuffers& sb, int64_t N, Ops& ops, int64_t max_steps, int64_t budget, int64_t* steps_done,
                         int64_t* episodes_done) {
    const bool counting = budget >= 0;
    if (counting) TRY(sb.alloc(ctx, ops.shadow_bytes(), ops.longest()));
    int64_t done = 0, episodes = 0;
    while (done < max_steps) {
        const int64_t remaining = budget - episodes;
        const int64_t s = ops.stretch(max_steps - done, counting, remaining);
        const typename Ops::Saved saved = ops.save();
        const bool may_stop = counting && remaining <= N * s;   // (a lane ends at most one episode per step)
        if (may_stop) {
            sb.shadow.clear();
            TRY(ops.mark(sb.shadow));
            TRY(sb.shadow.copy(ctx, true));
        }
        if (counting) CUDA_TRY(cudaMemsetAsync(sb.counts, 0, (size_t)s * sizeof(unsigned long long), ctx->stream));
        TRY(ops.run(s, may_stop));
        StopCrossing c{0, 0};
        if (counting) {
            TRY(stop_crossing(ctx, sb.counts, s, remaining, sb.host, [&] { return ops.count(s, saved, sb.counts); }, &c));
            if (c.step != 0 && c.step < s) {   // the stage loop stops after step s* of the stretch: roll back, run s* steps
                TRY(sb.shadow.copy(ctx, false));
                ops.restore(saved);
                TRY(ops.run(c.step, true));
            }
        }
        done += c.step ? c.step : s;
        episodes += c.episodes;
        TRY(ops.end_stretch());
        if (c.step || (!counting && ops.at_boundary(max_steps - done))) break;
    }
    *steps_done = done;
    *episodes_done = episodes;
    return B200RL_OK;
}

// kinds 2 and 3 are Q-networks (one flat vector, a target network, the DQN entry points); 0 and 1 actor-critic pairs
static bool is_q_kind(int kind) { return kind == 2 || kind == 3; }

static int make_descs(const b200rl_net_desc* d, MlpDesc* actor, MlpDesc* critic) {
    REQUIRE(d, B200RL_ERR_INVALID, "null desc");
    REQUIRE(d->kind >= 0 && d->kind <= 3, B200RL_ERR_INVALID,
            "kind must be 0 (actor-critic categorical), 1 (gaussian), 2 (Q-network) or 3 (dueling Q-network)");
    REQUIRE(d->n_in >= 1 && d->n_in <= kInMax, B200RL_ERR_UNSUPPORTED, "n_in must be 1..4");
    REQUIRE(d->hidden == 64 || d->hidden == 128, B200RL_ERR_UNSUPPORTED, "hidden must be 64 or 128");
    REQUIRE(d->act == 0 || d->act == 1, B200RL_ERR_INVALID, "act must be 0 (relu) or 1 (tanh)");
    if (d->kind == 1) REQUIRE(d->n_out == 1, B200RL_ERR_UNSUPPORTED, "gaussian policy supports a 1-d action");
    else if (d->kind == 3) REQUIRE(d->n_out >= 1 && d->n_out + 1 <= kOutMax, B200RL_ERR_UNSUPPORTED, "dueling Q-network: n_out (actions) must be 1..3");
    else REQUIRE(d->n_out >= 1 && d->n_out <= kOutMax, B200RL_ERR_UNSUPPORTED, "n_out must be 1..4");
    *actor = MlpDesc{d->n_in, d->hidden, d->act, d->kind == 1 ? 2 : d->n_out, d->kind == 1 ? 1 : 0, d->kind == 3 ? 1 : 0};
    *critic = MlpDesc{d->n_in, d->hidden, d->act, 1, 0, 0};
    return B200RL_OK;
}

// device buffers of an evaluation window: the records, and the staged path's per-env accumulators, actions and head outputs
struct EvalBufs {
    float* ret;                   // (K, N), null when the caller wants no returns
    int32_t* len;                 // (K, N), null when the caller wants no lengths
    int32_t* cnt;                 // (N)
    float* acc_ret;
    int32_t* acc_len;
    uint32_t* act;
    void* act_clamped;            // (N) T: the clamped continuous action the env receives
    float* heads;                 // (nout, N)
};

// The flow of b200rl_evaluate and b200rl_evaluate_explore after their checks: the device records (the caller's, on_device, or
// scratch holding the caller's values, so that slots the window does not fill keep them), reset!(env; is_force = true) (run.jl:46),
// the fused window fused(bufs) or, where it returns B200RL_ERR_UNSUPPORTED, n_steps x {plan!, act! (auto-reset), record} as staged
// launches without a host sync, then the copy-out.  plan(k, bufs, &a_env) launches plan! of window step k and sets the actions the
// env receives.
template <class Fused, class Plan>
static int eval_window(b200rl_ctx* ctx, b200rl_env* env, int nout, int nsteps, int K, float* returns_out, int32_t* lengths_out,
                       int32_t* counts_out, int on_device, Fused&& fused, Plan&& plan) {
    const int64_t N = b200rl_env_internal_n(env);
    const size_t rec_bytes = (size_t)N * K * 4;
    auto round256 = [](size_t b) { return (b + 255) / 256 * 256; };
    // device buffers: the caller's (on_device) or scratch; the staged path also keeps per-env accumulators and its actions
    size_t off = 0;
    const size_t o_ret = off; off += on_device ? 0 : round256(rec_bytes);
    const size_t o_len = off; off += on_device ? 0 : round256(rec_bytes);
    const size_t o_cnt = off; off += round256((size_t)N * 4);
    const size_t o_acc = off; off += round256((size_t)N * 4) * 2;
    const size_t o_act = off; off += round256((size_t)N * 4) + round256((size_t)N * 8);
    const size_t o_heads = off; off += round256((size_t)N * nout * 4);
    void* sc;
    TRY(ctx_scratch(ctx, off, &sc));
    char* base = (char*)sc;
    EvalBufs b;
    b.ret = returns_out ? (on_device ? returns_out : (float*)(base + o_ret)) : nullptr;
    b.len = lengths_out ? (on_device ? lengths_out : (int32_t*)(base + o_len)) : nullptr;
    b.cnt = (on_device && counts_out) ? counts_out : (int32_t*)(base + o_cnt);
    b.acc_ret = (float*)(base + o_acc);
    b.acc_len = (int32_t*)(base + o_acc + round256((size_t)N * 4));
    b.act = (uint32_t*)(base + o_act);
    b.act_clamped = base + o_act + round256((size_t)N * 4);
    b.heads = (float*)(base + o_heads);
    if (!on_device) {   // record slots the window does not fill keep the caller's values
        if (b.ret && rec_bytes) CUDA_TRY(cudaMemcpyAsync(b.ret, returns_out, rec_bytes, cudaMemcpyHostToDevice, ctx->stream));
        if (b.len && rec_bytes) CUDA_TRY(cudaMemcpyAsync(b.len, lengths_out, rec_bytes, cudaMemcpyHostToDevice, ctx->stream));
    }
    TRY(b200rl_env_reset(env, 1));   // reset!(env; is_force = true), run.jl:46
    int st = nn_tc_enabled() ? fused(b) : B200RL_ERR_UNSUPPORTED;
    if (st == B200RL_ERR_UNSUPPORTED) {   // staged: plan! -> act! (auto-reset) -> record, n_steps times, no host sync
        // (an evaluation is a run of its own: its K1 steps do not write the env's episode log)
        struct LogHold {
            b200rl_env* e;
            ~LogHold() { b200rl_env_internal_log_hold(e, false); }
        } hold{env};
        b200rl_env_internal_log_hold(env, true);
        CUDA_TRY(cudaMemsetAsync(b.cnt, 0, (size_t)N * 4, ctx->stream));
        CUDA_TRY(cudaMemsetAsync(b.acc_ret, 0, round256((size_t)N * 4) * 2, ctx->stream));
        const uint8_t* flags = (const uint8_t*)env_field(env, B200RL_FIELD_FLAGS);
        for (int k = 0; k < nsteps; ++k) {
            const void* a_env = b.act;
            TRY(plan(k, b, &a_env));
            TRY(b200rl_env_step(env, a_env, 1, 1));
            const float* rew;   // (a Float64 env: Float32(reward), as its EPISODE_RETURN adds it)
            TRY(b200rl_env_internal_reward_f32(env, &rew));
            eval_record_kernel<<<grid_for(N, 256), 256, 0, ctx->stream>>>(rew, flags, N, K, b.acc_ret, b.acc_len, b.cnt, b.ret, b.len);
            LAUNCH_CHECK(ctx);
        }
    } else if (st != B200RL_OK) {
        return st;
    }
    if (!on_device) {
        if (returns_out && rec_bytes) CUDA_TRY(cudaMemcpyAsync(returns_out, b.ret, rec_bytes, cudaMemcpyDeviceToHost, ctx->stream));
        if (lengths_out && rec_bytes) CUDA_TRY(cudaMemcpyAsync(lengths_out, b.len, rec_bytes, cudaMemcpyDeviceToHost, ctx->stream));
        if (counts_out) CUDA_TRY(cudaMemcpyAsync(counts_out, b.cnt, (size_t)N * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    }
    return B200RL_OK;
}

extern "C" {

int b200rl_net_nparams(const b200rl_net_desc* d, int64_t* out) {
    MlpDesc a, c;
    TRY(make_descs(d, &a, &c));
    REQUIRE(out, B200RL_ERR_INVALID, "null out");
    *out = is_q_kind(d->kind) ? a.nparams() : a.nparams() + c.nparams();
    return B200RL_OK;
}

int b200rl_net_destroy(b200rl_net* n) {
    if (!n) return B200RL_OK;
    cudaSetDevice(n->ctx->device);
    cudaStreamSynchronize(n->ctx->stream);
    cudaFree(n->params); cudaFree(n->grad); cudaFree(n->m); cudaFree(n->v); cudaFree(n->beta_t); cudaFree(n->target);
    cudaFree(n->partial); cudaFree(n->loss_partial); cudaFree(n->loss4); cudaFree(n->gnorm); cudaFree(n->cta_sumsq); cudaFree(n->counters);
    delete n;
    return B200RL_OK;
}

/* Replaces FluxApproximator(model, optimiser) (+ TargetNetwork for kinds 2 and 3): takes the flat
 * Flux.destructure parameter vector; optimiser = Adam(1e-3, (0.9, 0.999), 1e-8), clip 0.5 until
 * b200rl_net_configure_optimizer is called. */
int b200rl_net_create(b200rl_ctx* ctx, const b200rl_net_desc* d, const float* params_host, b200rl_net** out) {
    TRY(ctx_bind(ctx));
    REQUIRE(out && params_host, B200RL_ERR_INVALID, "null argument");
    b200rl_net* n = new b200rl_net();
    memset(n, 0, sizeof *n);
    n->ctx = ctx; n->kind = d ? d->kind : 0;
    int s = make_descs(d, &n->actor, &n->critic);
    if (s != B200RL_OK) { delete n; return s; }
    n->np = is_q_kind(n->kind) ? n->actor.nparams() : n->actor.nparams() + n->critic.nparams();
    n->lr = 1e-3f; n->b1 = 0.9f; n->b2 = 0.999f; n->eps = 1e-8f; n->max_grad_norm = 0.5f;
    size_t bytes = (size_t)n->np * sizeof(float);
    n->n_partials = is_q_kind(n->kind) ? nn_dqn_max_partials(ctx, n->actor.H) : nn_grid_ctas(ctx, n->actor.H);
    int n_loss_rows = 2 * (n->n_partials > ctx->sm_count ? n->n_partials : ctx->sm_count);
#define NET_TRY(x) CUDA_TRY_OR(x, b200rl_net_destroy(n))
    NET_TRY(cudaMalloc(&n->params, bytes)); NET_TRY(cudaMalloc(&n->grad, bytes)); NET_TRY(cudaMalloc(&n->m, bytes)); NET_TRY(cudaMalloc(&n->v, bytes));
    NET_TRY(cudaMalloc(&n->beta_t, 2 * sizeof(float)));
    if (is_q_kind(n->kind)) NET_TRY(cudaMalloc(&n->target, bytes));
    NET_TRY(cudaMalloc(&n->partial, (size_t)n->n_partials * bytes));
    NET_TRY(cudaMalloc(&n->loss_partial, (size_t)n_loss_rows * 4 * sizeof(float)));
    NET_TRY(cudaMalloc(&n->loss4, 4 * sizeof(float))); NET_TRY(cudaMalloc(&n->gnorm, sizeof(float)));
    NET_TRY(cudaMalloc(&n->cta_sumsq, 256 * sizeof(double))); NET_TRY(cudaMalloc(&n->counters, 4 * sizeof(unsigned int)));
    NET_TRY(cudaMemsetAsync(n->counters, 0, 4 * sizeof(unsigned int), ctx->stream));
    NET_TRY(cudaMemcpyAsync(n->params, params_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    if (is_q_kind(n->kind)) NET_TRY(cudaMemcpyAsync(n->target, params_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    NET_TRY(cudaMemsetAsync(n->grad, 0, bytes, ctx->stream)); NET_TRY(cudaMemsetAsync(n->m, 0, bytes, ctx->stream));
    NET_TRY(cudaMemsetAsync(n->v, 0, bytes, ctx->stream));
    NET_TRY(cudaMemsetAsync(n->partial, 0, (size_t)n->n_partials * bytes, ctx->stream));
    NET_TRY(cudaMemsetAsync(n->loss_partial, 0, (size_t)n_loss_rows * 4 * sizeof(float), ctx->stream));
    float bt[2] = {n->b1, n->b2};
    NET_TRY(cudaMemcpyAsync(n->beta_t, bt, sizeof bt, cudaMemcpyHostToDevice, ctx->stream));
    NET_TRY(cudaStreamSynchronize(ctx->stream));
#undef NET_TRY
    *out = n;
    return B200RL_OK;
}

int b200rl_net_set_critic_act(b200rl_net* n, int act) {
    REQUIRE(n, B200RL_ERR_INVALID, "null net");
    REQUIRE(!is_q_kind(n->kind), B200RL_ERR_INVALID, "only actor-critic networks have a critic trunk");
    REQUIRE(act == 0 || act == 1, B200RL_ERR_INVALID, "act must be 0 (relu) or 1 (tanh)");
    n->critic.act = act;
    return B200RL_OK;
}

int b200rl_net_configure_optimizer(b200rl_net* n, float lr, float beta1, float beta2, float eps, float max_grad_norm) {
    REQUIRE(n, B200RL_ERR_INVALID, "null net");
    TRY(ctx_bind(n->ctx));
    n->lr = lr; n->b1 = beta1; n->b2 = beta2; n->eps = eps; n->max_grad_norm = max_grad_norm;
    if (n->n_updates == 0) {
        float bt[2] = {beta1, beta2};
        CUDA_TRY(cudaMemcpyAsync(n->beta_t, bt, sizeof bt, cudaMemcpyHostToDevice, n->ctx->stream));
        CUDA_TRY(cudaStreamSynchronize(n->ctx->stream));
    }
    return B200RL_OK;
}

/* which: 0 params, 1 last (clipped) gradient, 2 Adam m, 3 Adam v, 4 beta_t (2 floats), 5 target params */
static int net_buf(b200rl_net* n, int which, float** p, int64_t* len) {
    switch (which) {
        case 0: *p = n->params; *len = n->np; return B200RL_OK;
        case 1: *p = n->grad; *len = n->np; return B200RL_OK;
        case 2: *p = n->m; *len = n->np; return B200RL_OK;
        case 3: *p = n->v; *len = n->np; return B200RL_OK;
        case 4: *p = n->beta_t; *len = 2; return B200RL_OK;
        case 5: REQUIRE(n->target, B200RL_ERR_INVALID, "no target network"); *p = n->target; *len = n->np; return B200RL_OK;
    }
    REQUIRE(false, B200RL_ERR_INVALID, "unknown buffer id");
}
/* export / import of parameters and optimiser state (checkpoint hook pattern, docs/src/How_to_use_hooks.md:124-167) */
int b200rl_net_get(b200rl_net* n, int which, float* host_dst, int64_t count) {
    REQUIRE(n && host_dst, B200RL_ERR_INVALID, "null argument");
    TRY(ctx_bind(n->ctx));
    float* p; int64_t len;
    TRY(net_buf(n, which, &p, &len));
    REQUIRE(count >= len, B200RL_ERR_INVALID, "destination too small");
    CUDA_TRY(cudaMemcpyAsync(host_dst, p, (size_t)len * 4, cudaMemcpyDeviceToHost, n->ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(n->ctx->stream));
    return B200RL_OK;
}
int b200rl_net_set(b200rl_net* n, int which, const float* host_src, int64_t count) {
    REQUIRE(n && host_src, B200RL_ERR_INVALID, "null argument");
    TRY(ctx_bind(n->ctx));
    float* p; int64_t len;
    TRY(net_buf(n, which, &p, &len));
    REQUIRE(count >= len, B200RL_ERR_INVALID, "source too small");
    CUDA_TRY(cudaMemcpyAsync(p, host_src, (size_t)len * 4, cudaMemcpyHostToDevice, n->ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(n->ctx->stream));
    return B200RL_OK;
}
int b200rl_net_ptr(b200rl_net* n, int which, void** dptr_out) {
    REQUIRE(n && dptr_out, B200RL_ERR_INVALID, "null argument");
    float* p; int64_t len;
    TRY(net_buf(n, which, &p, &len));
    *dptr_out = p;
    return B200RL_OK;
}

/* optimiser steps taken so far (drives the TargetNetwork's sync_freq phase, target_network.jl:70-88; part of a checkpoint) */
int b200rl_net_get_step(b200rl_net* n, int64_t* out) {
    REQUIRE(n && out, B200RL_ERR_INVALID, "null argument");
    *out = (int64_t)n->n_updates;
    return B200RL_OK;
}
int b200rl_net_set_step(b200rl_net* n, int64_t step) {
    REQUIRE(n && step >= 0, B200RL_ERR_INVALID, "bad argument");
    n->n_updates = (uint64_t)step;
    return B200RL_OK;
}
/* TargetNetwork sync: target = rho*target + (1-rho)*model (rho = 0: hard copy) — target_network.jl:70-88 */
int b200rl_net_target_sync(b200rl_net* n, float rho) {
    REQUIRE(n && n->target, B200RL_ERR_INVALID, "no target network");
    TRY(ctx_bind(n->ctx));
    return nn_target_sync(n->ctx, n->target, n->params, n->np, rho);
}

// the loss scalars of an agent's config; kSamplerHyper: what plan! outside an agent samples with (b200rl_net_act, b200rl_evaluate)
static AcHyper ac_hyper(const b200rl_onpolicy_config& c) {
    return AcHyper{c.clip_range, c.w_actor, c.w_critic, c.w_entropy, c.min_sigma, c.max_sigma, c.normalize_advantage, c.algo};
}
static constexpr AcHyper kSamplerHyper{0.1f, 1.f, 0.5f, 0.001f, 0.f, __builtin_inff(), 0, 0};
// per-minibatch stats row [actor_loss, critic_loss, entropy, loss, grad_norm, 0] from the device row s = {4 loss sums, grad norm}
static void decode_stats_row(const b200rl_onpolicy_config& c, const float* s, float invB, float* o) {
    o[0] = s[0] * invB; o[1] = s[2] * invB; o[2] = s[1] * invB;
    o[3] = c.w_actor * o[0] + c.w_critic * o[1] - c.w_entropy * o[2];
    o[4] = s[4]; o[5] = 0.f;
}

static int stage_obs(b200rl_net* n, const float* obs, int64_t N, int on_device, const float** dev, size_t extra, void** extra_dev) {
    size_t ob = (size_t)N * n->actor.in * 4;
    if (on_device && extra == 0) { *dev = obs; return B200RL_OK; }
    void* s;
    TRY(ctx_scratch(n->ctx, ob + extra + 512, &s));
    if (!on_device) { CUDA_TRY(cudaMemcpyAsync(s, obs, ob, cudaMemcpyHostToDevice, n->ctx->stream)); *dev = (const float*)s; }
    else *dev = obs;
    if (extra_dev) *extra_dev = (char*)s + ((ob + 255) / 256) * 256;
    return B200RL_OK;
}

/* plan!(policy, env) for a batch of observations (in, N): action (int32 1-based | float), log-prob and V(s).
 * rng = (4, N) uint64 DEVICE policy streams (advanced in place).  Outputs may be NULL.  on_device applies to obs and outputs. */
int b200rl_net_act(b200rl_net* n, const float* obs, int64_t N, uint64_t* rng_dev, void* action_out, float* logp_out, float* value_out,
                   float* heads_out, int on_device) {
    REQUIRE(n && obs && rng_dev && !is_q_kind(n->kind), B200RL_ERR_INVALID, "bad argument (actor-critic nets only)");
    TRY(ctx_bind(n->ctx));
    const AcHyper& hp = kSamplerHyper;
    const float* dobs;
    size_t ho = (size_t)N * n->actor.nout * 4;
    void* ex = nullptr;
    TRY(stage_obs(n, obs, N, on_device, &dobs, on_device ? 0 : (size_t)N * 12 + ho + 1024, &ex));
    if (on_device)
        return nn_policy_act(n->ctx, n->actor, n->critic, n->params, hp, dobs, N, (unsigned long long*)rng_dev, action_out, logp_out, value_out,
                             heads_out, nullptr);
    float* da = (float*)ex; float* dl = da + N; float* dv = dl + N; float* dh = dv + N;
    TRY(nn_policy_act(n->ctx, n->actor, n->critic, n->params, hp, dobs, N, (unsigned long long*)rng_dev, da, dl, dv, heads_out ? dh : nullptr, nullptr));
    if (action_out) CUDA_TRY(cudaMemcpyAsync(action_out, da, (size_t)N * 4, cudaMemcpyDeviceToHost, n->ctx->stream));
    if (logp_out) CUDA_TRY(cudaMemcpyAsync(logp_out, dl, (size_t)N * 4, cudaMemcpyDeviceToHost, n->ctx->stream));
    if (value_out) CUDA_TRY(cudaMemcpyAsync(value_out, dv, (size_t)N * 4, cudaMemcpyDeviceToHost, n->ctx->stream));
    if (heads_out) CUDA_TRY(cudaMemcpyAsync(heads_out, dh, ho, cudaMemcpyDeviceToHost, n->ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(n->ctx->stream));
    return B200RL_OK;
}

/* critic V(s) (kinds 0/1: out (N)) or Q(s, .) (kinds 2, 3: out (n_out, N); kind 3 the combined Q); use_target selects the target network */
int b200rl_net_values(b200rl_net* n, const float* obs, int64_t N, float* out, int use_target, int on_device) {
    REQUIRE(n && obs && out, B200RL_ERR_INVALID, "null argument");
    TRY(ctx_bind(n->ctx));
    const MlpDesc& d = is_q_kind(n->kind) ? n->actor : n->critic;
    const float* p = is_q_kind(n->kind) ? (use_target ? n->target : n->params) : n->params + n->actor.nparams();
    REQUIRE(p, B200RL_ERR_INVALID, "no target network");
    const float* dobs;
    size_t ob = (size_t)N * d.nout * 4;
    void* ex = nullptr;
    TRY(stage_obs(n, obs, N, on_device, &dobs, on_device ? 0 : ob + 256, &ex));
    if (on_device) return nn_mlp_forward(n->ctx, d, p, dobs, N, out);
    TRY(nn_mlp_forward(n->ctx, d, p, dobs, N, (float*)ex));
    CUDA_TRY(cudaMemcpyAsync(out, ex, ob, cudaMemcpyDeviceToHost, n->ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(n->ctx->stream));
    return B200RL_OK;
}

/* epsilon-greedy action selection on Q(s, .) (EpsilonGreedyExplorer / QBasedPolicy plan!); all pointers DEVICE */
int b200rl_net_q_act(b200rl_net* n, const float* obs_dev, int64_t N, uint64_t* rng_dev, float epsilon, int32_t* action_out_dev) {
    REQUIRE(n && obs_dev && action_out_dev && is_q_kind(n->kind), B200RL_ERR_INVALID, "bad argument (Q-network only)");
    REQUIRE(epsilon <= 0.f || rng_dev, B200RL_ERR_INVALID, "rng required for epsilon > 0");
    TRY(ctx_bind(n->ctx));
    void* s;
    TRY(ctx_scratch(n->ctx, (size_t)N * n->actor.nout * 4 + 256, &s));
    return nn_q_act(n->ctx, n->actor, n->params, obs_dev, N, (unsigned long long*)rng_dev, epsilon, action_out_dev, (float*)s);
}

// the explorer fields a kind reads: a known kind, a schedule with epsilons in [0, 1] (kinds 0 / 1), a finite beta (kind 2).  The
// fields kinds 2-4 do not read must be zero, so that a struct filled for one explorer is not silently run as another.
static int check_explorer(const b200rl_explorer* ex) {
    REQUIRE(ex->kind >= 0 && ex->kind <= 4, B200RL_ERR_INVALID, "unknown explorer kind (0 :linear, 1 :exp, 2 speedy, 3 weighted softmax, 4 Gumbel softmax)");
    if (ex->kind <= 1) {
        REQUIRE(ex->warmup_steps >= 0 && ex->decay_steps >= 0, B200RL_ERR_INVALID, "bad explorer schedule");
        REQUIRE(ex->eps_stable >= 0.0 && ex->eps_stable <= 1.0 && ex->eps_init >= 0.0 && ex->eps_init <= 1.0, B200RL_ERR_INVALID, "epsilon outside [0, 1]");
        return B200RL_OK;
    }
    REQUIRE(ex->eps_stable == 0.0 && ex->eps_init == 0.0 && ex->warmup_steps == 0 && ex->decay_steps == 0 && ex->is_break_tie == 0,
            B200RL_ERR_INVALID, "explorer kinds 2-4 take no epsilon schedule or break-tie (those fields must be 0)");
    if (ex->kind == 2) REQUIRE(std::isfinite(ex->beta), B200RL_ERR_INVALID, "EpsilonSpeedyExplorer beta must be finite");
    else REQUIRE(ex->beta == 0.0, B200RL_ERR_INVALID, "the softmax explorers take no beta (must be 0)");
    return B200RL_OK;
}

/* BatchExplorer(explorer) with the explorer's schedule evaluated per column on the device; all pointers DEVICE */
int b200rl_net_q_explore(b200rl_net* n, const float* obs_dev, int64_t N, uint64_t* rng_dev, const b200rl_explorer* ex, int32_t* action_out_dev) {
    REQUIRE(n && obs_dev && action_out_dev && rng_dev && ex && is_q_kind(n->kind), B200RL_ERR_INVALID, "bad argument (Q-network only)");
    REQUIRE(N > 0, B200RL_ERR_INVALID, "empty batch");
    TRY(check_explorer(ex));
    TRY(ctx_bind(n->ctx));
    void* s;
    TRY(ctx_scratch(n->ctx, (size_t)N * n->actor.nout * 4 + 256, &s));
    return nn_q_explore(n->ctx, n->actor, n->params, obs_dev, N, (unsigned long long*)rng_dev, *ex, action_out_dev, (float*)s);
}

/* plan!(greedy policy, obs): findmax of the logits / Q-values (kinds 0, 2, 3), mu (kind 1); no RNG.  Same forward pass as
 * b200rl_net_values / the head outputs of b200rl_net_act. */
int b200rl_net_act_greedy(b200rl_net* n, const float* obs, int64_t N, void* action_out, int on_device) {
    REQUIRE(n && obs && action_out, B200RL_ERR_INVALID, "null argument");
    REQUIRE(N > 0, B200RL_ERR_INVALID, "empty batch");
    TRY(ctx_bind(n->ctx));
    const size_t hb = ((size_t)N * n->actor.nout * 4 + 255) / 256 * 256;
    const float* dobs;
    void* ex = nullptr;
    TRY(stage_obs(n, obs, N, on_device, &dobs, hb + (size_t)N * 4 + 256, &ex));
    float* heads = (float*)ex;
    uint32_t* da = on_device ? (uint32_t*)action_out : (uint32_t*)((char*)ex + hb);
    TRY(nn_mlp_forward(n->ctx, n->actor, n->params, dobs, N, heads));
    greedy_select_kernel<<<grid_for(N, 256), 256, 0, n->ctx->stream>>>(heads, n->actor, N, 0, 0.f, 0.f, da);
    LAUNCH_CHECK(n->ctx);
    if (!on_device) {
        CUDA_TRY(cudaMemcpyAsync(action_out, da, (size_t)N * 4, cudaMemcpyDeviceToHost, n->ctx->stream));
        CUDA_TRY(cudaStreamSynchronize(n->ctx->stream));
    }
    return B200RL_OK;
}

/* run(policy, env, StopAfterNSteps(n_steps)) with the network's greedy (mode 0) or sampling (mode 1) policy; see b200rl.h.
 * Fused into one launch (fwd_tc.cu) for H = 64 on the tensor-core path, otherwise staged launches with the same arithmetic. */
int b200rl_evaluate(b200rl_net* n, b200rl_env* env, const b200rl_eval_config* cfg, uint64_t* policy_rng_dev, float* returns_out,
                    int32_t* lengths_out, int32_t* counts_out, int on_device) {
    REQUIRE(n && env && cfg, B200RL_ERR_INVALID, "null argument");
    REQUIRE(b200rl_env_internal_ctx(env) == n->ctx, B200RL_ERR_INVALID, "net/env belong to another ctx");
    const float* obs;
    TRY(learner_obs(env, &obs));
    REQUIRE(b200rl_env_internal_kind(env) != B200RL_ENV_ACROBOT, B200RL_ERR_UNSUPPORTED, "AcrobotEnv has 6 observations (networks take at most 4)");
    REQUIRE(cfg->mode == 0 || cfg->mode == 1, B200RL_ERR_INVALID, "mode must be 0 (greedy) or 1 (sample)");
    REQUIRE(!(cfg->mode == 1 && is_q_kind(n->kind)), B200RL_ERR_UNSUPPORTED, "mode 1 samples a policy head: evaluate a Q-network with mode 0 or QBasedPolicy");
    REQUIRE(b200rl_env_internal_nobs(env) == n->actor.in, B200RL_ERR_INVALID, "network input width != observation width");
    const bool cont = b200rl_env_internal_continuous(env);
    REQUIRE(cont == (n->kind == 1), B200RL_ERR_INVALID, "head kind != action-space kind (Gaussian head <-> continuous actions)");
    REQUIRE(cont || n->actor.nout == b200rl_env_internal_n_actions(env), B200RL_ERR_INVALID, "head width != number of discrete actions");
    REQUIRE(cfg->n_steps >= 1, B200RL_ERR_INVALID, "n_steps must be >= 1");
    REQUIRE(cfg->max_episodes >= 0, B200RL_ERR_INVALID, "max_episodes must be >= 0");
    REQUIRE(cfg->mode == 0 || policy_rng_dev, B200RL_ERR_INVALID, "mode 1 needs the (4, N) device policy streams");
    TRY(ctx_bind(n->ctx));
    b200rl_ctx* ctx = n->ctx;
    const int64_t N = b200rl_env_internal_n(env);
    const int K = cfg->max_episodes, mode = cfg->mode, nsteps = cfg->n_steps;
    const AcHyper& hp = kSamplerHyper;
    unsigned long long* prng = (unsigned long long*)policy_rng_dev;
    const float bound = b200rl_env_internal_action_bound(env);
    const bool f64 = b200rl_env_internal_dtype(env) == B200RL_F64;
    return eval_window(
        ctx, env, n->actor.nout, nsteps, K, returns_out, lengths_out, counts_out, on_device,
        [&](const EvalBufs& b) -> int { return nn_tc_evaluate(ctx, env, n->actor, n->params, hp, mode, nsteps, K, prng, b.ret, b.len, b.cnt); },
        [&](int, const EvalBufs& b, const void** a_env) -> int {
            if (mode == 0) {
                TRY(nn_mlp_forward(ctx, n->actor, n->params, obs, N, b.heads));
                greedy_select_kernel<<<grid_for(N, 256), 256, 0, ctx->stream>>>(b.heads, n->actor, N, cont ? 1 : 0, -bound, bound, b.act);
                LAUNCH_CHECK(ctx);
                if (cont && f64) {   // Float64 of the clamped mu
                    TRY(env_action_clamped(env, (const float*)b.act, N, b.act_clamped));
                    *a_env = b.act_clamped;
                }
            } else {
                TRY(nn_policy_act(ctx, n->actor, n->critic, n->params, hp, obs, N, prng, b.act, nullptr, nullptr, nullptr, nullptr));
                if (cont) {
                    TRY(env_action_clamped(env, (const float*)b.act, N, b.act_clamped));
                    *a_env = b.act_clamped;
                }
            }
            return B200RL_OK;
        });
}

/* run(QBasedPolicy(learner, explorer), env, StopAfterNSteps(n_steps)); see b200rl.h.  Fused into one launch (fwd_tc.cu) for H = 64
 * on the tensor-core path, otherwise q_explore | q_act, act! and record launches per step with the same arithmetic. */
int b200rl_evaluate_explore(b200rl_net* n, b200rl_env* env, int32_t n_steps, int32_t max_episodes, b200rl_explorer* ex,
                            uint64_t* explorer_rng_dev, float* returns_out, int32_t* lengths_out, int32_t* counts_out, int on_device) {
    REQUIRE(n && env, B200RL_ERR_INVALID, "null argument");
    REQUIRE(b200rl_env_internal_ctx(env) == n->ctx, B200RL_ERR_INVALID, "net/env belong to another ctx");
    const float* obs;
    TRY(learner_obs(env, &obs));
    REQUIRE(b200rl_env_internal_kind(env) != B200RL_ENV_ACROBOT, B200RL_ERR_UNSUPPORTED, "AcrobotEnv has 6 observations (networks take at most 4)");
    REQUIRE(!b200rl_env_internal_continuous(env), B200RL_ERR_UNSUPPORTED, "QBasedPolicy needs a discrete action space");
    REQUIRE(is_q_kind(n->kind), B200RL_ERR_INVALID, "needs a Q-network (kind 2 or 3)");
    REQUIRE(b200rl_env_internal_nobs(env) == n->actor.in, B200RL_ERR_INVALID, "network input width != observation width");
    REQUIRE(n->actor.nout == b200rl_env_internal_n_actions(env), B200RL_ERR_INVALID, "Q head width != number of discrete actions");
    REQUIRE(n_steps >= 1, B200RL_ERR_INVALID, "n_steps must be >= 1");
    REQUIRE(max_episodes >= 0, B200RL_ERR_INVALID, "max_episodes must be >= 0");
    const int64_t N = b200rl_env_internal_n(env);
    const int64_t NW = N * b200rl_comm_world(n->ctx);   // columns of one plan! over the ranks' union (DESIGN.md §3)
    if (ex) {
        REQUIRE(explorer_rng_dev, B200RL_ERR_INVALID, "an explorer other than GreedyExplorer needs the (4, N) device explorer streams");
        TRY(check_explorer(ex));
        REQUIRE(n_steps <= ((1ll << 62) - (ex->step > 0 ? ex->step : 0)) / NW, B200RL_ERR_INVALID, "explorer step would overflow");
    }
    TRY(ctx_bind(n->ctx));
    b200rl_ctx* ctx = n->ctx;
    unsigned long long* xrng = (unsigned long long*)explorer_rng_dev;
    TRY(eval_window(
        ctx, env, n->actor.nout, n_steps, max_episodes, returns_out, lengths_out, counts_out, on_device,
        [&](const EvalBufs& b) -> int {
            return nn_tc_evaluate(ctx, env, n->actor, n->params, kSamplerHyper, 2, n_steps, max_episodes, xrng, b.ret, b.len, b.cnt, ex);
        },
        [&](int k, const EvalBufs& b, const void**) -> int {
            if (!ex) return nn_q_act(ctx, n->actor, n->params, obs, N, nullptr, 0.0f, (int32_t*)b.act, b.heads);   // GreedyExplorer
            b200rl_explorer e = *ex;
            e.step = ex->step + (int64_t)k * NW;    // BatchExplorer: the inner explorer's step moved N · world times per plan!
            return nn_q_explore(ctx, n->actor, n->params, obs, N, xrng, e, (int32_t*)b.act, b.heads);
        }));
    if (ex) ex->step += (int64_t)n_steps * NW;
    return B200RL_OK;
}

}  // extern "C"

// ------------------------------------------------------------------ evaluation policies under run() ---------
// run(EvaluationPolicy | QBasedPolicy, env, StopAfterNSteps | StopAfterNEpisodes, hook) on the fused evaluation kernel: the handle
// holds the StopBuffers of run_stretches across the windows of a run (and the runs of a policy).  mode 0 greedy, 1 sampled
// (kinds 0 / 1), 2 a Q-network planned by an explorer (kinds 2 / 3).
struct b200rl_eval {
    b200rl_ctx* ctx;
    b200rl_net* net;
    b200rl_env* env;
    int mode;
    StopBuffers stop;
};

// the net <-> env <-> mode checks of b200rl_evaluate / b200rl_evaluate_explore, with their statuses
static int eval_check(b200rl_net* n, b200rl_env* env, int mode) {
    REQUIRE(b200rl_env_internal_ctx(env) == n->ctx, B200RL_ERR_INVALID, "net/env belong to another ctx");
    const float* obs;
    TRY(learner_obs(env, &obs));
    REQUIRE(b200rl_env_internal_kind(env) != B200RL_ENV_ACROBOT, B200RL_ERR_UNSUPPORTED, "AcrobotEnv has 6 observations (networks take at most 4)");
    REQUIRE(mode >= 0 && mode <= 2, B200RL_ERR_INVALID, "mode must be 0 (greedy), 1 (sample) or 2 (QBasedPolicy)");
    REQUIRE(!(mode == 1 && is_q_kind(n->kind)), B200RL_ERR_UNSUPPORTED, "mode 1 samples a policy head: evaluate a Q-network with mode 0 or QBasedPolicy");
    const bool cont = b200rl_env_internal_continuous(env);
    if (mode == 2) {
        REQUIRE(!cont, B200RL_ERR_UNSUPPORTED, "QBasedPolicy needs a discrete action space");
        REQUIRE(is_q_kind(n->kind), B200RL_ERR_INVALID, "needs a Q-network (kind 2 or 3)");
    }
    REQUIRE(b200rl_env_internal_nobs(env) == n->actor.in, B200RL_ERR_INVALID, "network input width != observation width");
    REQUIRE(mode == 2 || cont == (n->kind == 1), B200RL_ERR_INVALID, "head kind != action-space kind (Gaussian head <-> continuous actions)");
    REQUIRE(cont || n->actor.nout == b200rl_env_internal_n_actions(env), B200RL_ERR_INVALID, "head width != number of discrete actions");
    return B200RL_OK;
}

// One stretch of s steps from the env's current state: the fused evaluation kernel (RUN instantiations) or, where it returns
// B200RL_ERR_UNSUPPORTED, s x {plan!, act! (auto-reset, episode log), count} as staged launches without a host sync — plan! with the
// launches of the stage loop's EvaluationPolicy / QBasedPolicy (b200rl_net_act_greedy | b200rl_net_act | b200rl_net_q_act |
// b200rl_net_q_explore).  counts (may be null): counts[j] += lanes terminal after step j + 1.  ex->step is not advanced here.
static int eval_run_stretch(b200rl_eval* h, unsigned long long* prng, const b200rl_explorer* ex, int64_t s, unsigned long long* counts) {
    b200rl_ctx* ctx = h->ctx;
    b200rl_net* n = h->net;
    b200rl_env* env = h->env;
    const int mode = h->mode;
    int st = nn_tc_enabled() ? nn_tc_eval_run(ctx, env, n->actor, n->params, kSamplerHyper, mode, (int)s, prng, ex, counts)
                             : B200RL_ERR_UNSUPPORTED;
    if (st != B200RL_ERR_UNSUPPORTED) return st;
    const int64_t N = b200rl_env_internal_n(env);
    const int64_t NW = N * b200rl_comm_world(ctx);
    const float* obs;
    TRY(learner_obs(env, &obs));
    const bool cont = b200rl_env_internal_continuous(env), f64 = b200rl_env_internal_dtype(env) == B200RL_F64;
    const float bound = b200rl_env_internal_action_bound(env);
    void* sc;
    TRY(ctx_scratch(ctx, round256((size_t)N * 4) + round256((size_t)N * 8) + round256((size_t)N * n->actor.nout * 4), &sc));
    uint32_t* act = (uint32_t*)sc;
    void* act_clamped = (char*)sc + round256((size_t)N * 4);
    float* heads = (float*)((char*)sc + round256((size_t)N * 4) + round256((size_t)N * 8));
    const uint8_t* flags = (const uint8_t*)env_field(env, B200RL_FIELD_FLAGS);
    for (int64_t k = 0; k < s; ++k) {
        const void* a_env = act;
        if (mode == 0) {
            TRY(nn_mlp_forward(ctx, n->actor, n->params, obs, N, heads));
            greedy_select_kernel<<<grid_for(N, 256), 256, 0, ctx->stream>>>(heads, n->actor, N, cont ? 1 : 0, -bound, bound, act);
            LAUNCH_CHECK(ctx);
            if (cont && f64) {   // Float64 of the clamped mu
                TRY(env_action_clamped(env, (const float*)act, N, act_clamped));
                a_env = act_clamped;
            }
        } else if (mode == 1) {
            TRY(nn_policy_act(ctx, n->actor, n->critic, n->params, kSamplerHyper, obs, N, prng, act, nullptr, nullptr, nullptr, nullptr));
            if (cont) {
                TRY(env_action_clamped(env, (const float*)act, N, act_clamped));
                a_env = act_clamped;
            }
        } else if (!ex) {   // GreedyExplorer
            TRY(nn_q_act(ctx, n->actor, n->params, obs, N, nullptr, 0.0f, (int32_t*)act, heads));
        } else {
            b200rl_explorer e = *ex;
            e.step = ex->step + k * NW;    // BatchExplorer: the inner explorer's step moved N · world times per plan!
            TRY(nn_q_explore(ctx, n->actor, n->params, obs, N, prng, e, (int32_t*)act, heads));
        }
        TRY(b200rl_env_step(env, a_env, 1, 1));
        if (counts) {
            stop::count_columns_kernel<<<dim3(grid_for(N, stop::kCountBlock), 1), stop::kCountBlock, 0, ctx->stream>>>(flags, N, 0, 1, counts + k);
            LAUNCH_CHECK(ctx);
        }
    }
    return B200RL_OK;
}

/* The evaluation policy's part of run_stretches: stretches of stop::eval_stretch steps, each of which counts as it runs
 * (eval_run_stretch).  The shadow is the env's step regions and the (4, N) policy or explorer streams; a rollback restores the env's step
 * counter and the explorer step. */
struct EvalStretches {
    b200rl_eval* h;
    unsigned long long* prng;      // (4, N) policy streams (mode 1), explorer streams (mode 2 with an explorer), or null
    b200rl_explorer* ex;           // mode 2; null: GreedyExplorer
    bool counting;
    int64_t N, NW;
    struct Saved { int64_t ex_step; uint64_t env_steps; };
    Saved save() const { return {ex ? ex->step : 0, b200rl_env_internal_steps(h->env)}; }
    void restore(const Saved& s0) const {
        if (ex) ex->step = s0.ex_step;
        b200rl_env_internal_add_steps(h->env, s0.env_steps - b200rl_env_internal_steps(h->env));
    }
    size_t shadow_bytes() const { return b200rl_env_internal_step_bytes_max(h->env) + round256((size_t)N * 32); }
    int64_t longest() const { return stop::kEvalStretchMax; }
    int mark(Shadow& sh) const {
        DevRegion er[kEnvStepRegionsMax];
        TRY(sh.add_regions(er, b200rl_env_internal_step_regions(h->env, er)));
        return prng ? sh.add(prng, (size_t)N * 32) : B200RL_OK;
    }
    int64_t stretch(int64_t left, bool c, int64_t remaining) const { return stop::eval_stretch(left, remaining, N, c); }
    int run(int64_t s, bool) {
        TRY(eval_run_stretch(h, prng, ex, s, counting ? h->stop.counts : nullptr));
        if (ex) ex->step += s * NW;
        return B200RL_OK;
    }
    int count(int64_t, const Saved&, unsigned long long*) const { return B200RL_OK; }   // (counted by run)
    int end_stretch() const { return B200RL_OK; }
    bool at_boundary(int64_t) const { return false; }
};

extern "C" {

int b200rl_eval_create(b200rl_net* net, b200rl_env* env, int32_t mode, b200rl_eval** out) {
    REQUIRE(net && env && out, B200RL_ERR_INVALID, "null argument");
    TRY(eval_check(net, env, mode));
    b200rl_eval* h = new b200rl_eval();
    h->ctx = net->ctx; h->net = net; h->env = env; h->mode = mode;
    *out = h;
    return B200RL_OK;
}

int b200rl_eval_destroy(b200rl_eval* h) {
    if (!h) return B200RL_OK;
    cudaSetDevice(h->ctx->device);
    cudaStreamSynchronize(h->ctx->stream);
    h->stop.release();
    delete h;
    return B200RL_OK;
}

/* run(policy, env, StopAfterNSteps | StopAfterNEpisodes(k)) for at most max_steps env steps (include/b200rl.h): run_stretches */
int b200rl_eval_run_episodes(b200rl_eval* h, uint64_t* rng_dev, b200rl_explorer* ex, int64_t max_steps, int64_t budget, int64_t* steps_done,
                             int64_t* episodes_done) {
    REQUIRE(h && steps_done && episodes_done, B200RL_ERR_INVALID, "null argument");
    REQUIRE(max_steps >= 1, B200RL_ERR_INVALID, "max_steps must be >= 1");
    REQUIRE(budget < 0 || b200rl_comm_world(h->ctx) == 1, B200RL_ERR_UNSUPPORTED,
            "StopAfterNEpisodes counts the episodes of every rank: a sharded ctx keeps the stage loop");
    TRY(eval_check(h->net, h->env, h->mode));   // (the Float32 wrapper may have been removed since create)
    REQUIRE(h->mode == 2 || !ex, B200RL_ERR_INVALID, "an explorer plans a Q-network: mode 2 only");
    REQUIRE(h->mode != 1 || rng_dev, B200RL_ERR_INVALID, "mode 1 needs the (4, N) device policy streams");
    const int64_t N = b200rl_env_internal_n(h->env);
    const int64_t NW = N * b200rl_comm_world(h->ctx);   // columns of one plan! over the ranks' union (DESIGN.md §3)
    int64_t run_steps = max_steps;
    if (ex) {
        REQUIRE(rng_dev, B200RL_ERR_INVALID, "an explorer other than GreedyExplorer needs the (4, N) device explorer streams");
        TRY(check_explorer(ex));
        const int64_t room = ((1ll << 62) - (ex->step > 0 ? ex->step : 0)) / NW;   // steps before the explorer step overflows
        REQUIRE(budget < 0 ? max_steps <= room : room >= 1, B200RL_ERR_INVALID, "explorer step would overflow");
        if (room < run_steps) run_steps = room;   // (with a budget the run stops there; the next call is refused)
    }
    TRY(ctx_bind(h->ctx));
    unsigned long long* prng = (h->mode == 1 || ex) ? (unsigned long long*)rng_dev : nullptr;
    EvalStretches ops{h, prng, ex, budget >= 0, N, NW};
    return run_stretches(h->ctx, h->stop, N, ops, run_steps, budget, steps_done, episodes_done);
}

/* One optimiser step from explicit on-policy minibatch arrays (all HOST; test / generic entry):
 * loss + gradient (K7), global-norm clip + Adam (K8).  losses_out[6] = actor_loss, critic_loss,
 * entropy, loss, grad_norm (pre-clip), 0.  apply_update = 0 leaves the parameters untouched (gradient only). */
int b200rl_net_ac_step(b200rl_net* n, const b200rl_onpolicy_config* cfg, const float* states, const void* actions, const float* logp_old,
                       const float* adv, const float* ret, int64_t total, const int32_t* idx, int64_t B, float adv_mean, float adv_inv_std,
                       int apply_update, float* losses_out) {
    REQUIRE(n && cfg && states && actions && adv && ret && !is_q_kind(n->kind), B200RL_ERR_INVALID, "bad argument");
    TRY(ctx_bind(n->ctx));
    b200rl_ctx* ctx = n->ctx;
    int ns = n->actor.in;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
    const int64_t Beff = idx ? B : total;
    size_t o_s = take((size_t)total * ns * 4), o_a = take((size_t)total * 4), o_l = take((size_t)total * 4), o_ad = take((size_t)total * 4),
           o_r = take((size_t)total * 4), o_i = take((size_t)Beff * 4), o_n = take(8);
    void* sc;
    TRY(ctx_scratch(ctx, off, &sc));
    char* base = (char*)sc;
    std::vector<int32_t> iota;
    if (!idx) {  // identity order
        iota.resize((size_t)total);
        for (int64_t k = 0; k < total; ++k) iota[(size_t)k] = (int32_t)k;
        idx = iota.data();
    }
    CUDA_TRY(cudaMemcpyAsync(base + o_s, states, (size_t)total * ns * 4, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(base + o_a, actions, (size_t)total * 4, cudaMemcpyHostToDevice, ctx->stream));
    if (logp_old) CUDA_TRY(cudaMemcpyAsync(base + o_l, logp_old, (size_t)total * 4, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(base + o_ad, adv, (size_t)total * 4, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(base + o_r, ret, (size_t)total * 4, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(base + o_i, idx, (size_t)Beff * 4, cudaMemcpyHostToDevice, ctx->stream));
    float nm[2] = {adv_mean, adv_inv_std};
    CUDA_TRY(cudaMemcpyAsync(base + o_n, nm, 8, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));  // host buffers (incl. the local iota) are borrowed for this call only
    const AcHyper hp = ac_hyper(*cfg);
    AcBatch b{(const float*)(base + o_s), ns, base + o_a, logp_old ? (const float*)(base + o_l) : nullptr, (const float*)(base + o_ad),
              (const float*)(base + o_r), (const int32_t*)(base + o_i), (uint32_t)total, 0u, 0u, nullptr, nullptr, Beff, 1.0f / (float)Beff,
              (const float*)(base + o_n)};
    int ctas = nn_ac_loss_grad(ctx, n->actor, n->critic, n->params, hp, b, n->partial, n->loss_partial);
    if (ctas < 0) return ctas;
    TRY(nn_reduce_partials(ctx, n->partial, ctas, n->np, n->grad, n->loss_partial, 2 * ctas, n->loss4));
    if (apply_update) {
        TRY(nn_clip_adam(ctx, n->np, opt_step(n, *cfg)));
        n->n_updates += 1;
    }
    if (losses_out) {
        float s[5] = {};   // {4 loss sums, grad norm}
        CUDA_TRY(cudaMemcpyAsync(s, n->loss4, 16, cudaMemcpyDeviceToHost, ctx->stream));
        if (apply_update) CUDA_TRY(cudaMemcpyAsync(s + 4, n->gnorm, 4, cudaMemcpyDeviceToHost, ctx->stream));
        CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        decode_stats_row(*cfg, s, 1.0f / (float)Beff, losses_out);
    }
    return B200RL_OK;
}

}  // extern "C"

// ------------------------------------------------------------------ on-policy agent --------
struct b200rl_onpolicy {
    b200rl_ctx* ctx;
    b200rl_net* net;
    b200rl_env* env;
    b200rl_onpolicy_config cfg;
    int64_t N;
    int T, t, ns;
    bool continuous;
    bool bootstrap_done;   // column T of states / values already written by the fused rollout
    unsigned long long* rng;
    float* states; void* actions; float* logp; float* rewards; uint8_t* terminals; float* values; float* adv; float* ret;
    void* act_clamped;           // (N) T: the clamped continuous action the env receives
    double* norm_partials; double* norm_sums; float* norm2;
    int32_t* perm_dev;
    float* stats_dev; int stats_rows;
    float4* rec;                 // packed 32-byte records of the rollout (written after GAE, gathered by K7)
    unsigned int* upd_dev;       // device copy of n_updates: keys the minibatch permutation, ticked by the last optimiser step of an update
    uint64_t n_updates;
    GraphUnit graph;             // one whole iteration (collect(T) + update) for b200rl_onpolicy_iterate
    StopBuffers stop;            // b200rl_onpolicy_run_episodes with a budget: env arrays, policy streams and rollout columns
};

// the (n_epochs * n_microbatches, 6) stats rows of the last update (synchronises)
static int read_stats(b200rl_onpolicy* a, float* stats_host) {
    std::vector<float> tmp((size_t)a->stats_rows * 8);
    CUDA_TRY(cudaMemcpyAsync(tmp.data(), a->stats_dev, tmp.size() * 4, cudaMemcpyDeviceToHost, a->ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(a->ctx->stream));
    const float invB = 1.0f / ((float)(a->N * a->T / a->cfg.n_microbatches) * (float)b200rl_comm_world(a->ctx));
    for (int r = 0; r < a->stats_rows; ++r) decode_stats_row(a->cfg, tmp.data() + (size_t)r * 8, invB, stats_host + (size_t)r * 6);
    return B200RL_OK;
}

/* rollout tensors by field id: 0 state (ns, N, T+1) | 1 action (N, T) | 2 logp (N, T) | 3 reward (N, T) | 4 terminal (N, T) u8 |
 * 5 value (N, T+1) | 6 advantage (N, T) | 7 return (N, T) | 8 policy rng (4, N) u64 | 9 advantage norm {mean, inv_std} */
static int rollout_field(b200rl_onpolicy* a, int field, void** p, size_t* bytes) {
    const size_t N = (size_t)a->N, T = (size_t)a->T;
    switch (field) {
        case 0: *p = a->states; *bytes = N * a->ns * (T + 1) * 4; return B200RL_OK;
        case 1: *p = a->actions; *bytes = N * T * 4; return B200RL_OK;
        case 2: *p = a->logp; *bytes = N * T * 4; return B200RL_OK;
        case 3: *p = a->rewards; *bytes = N * T * 4; return B200RL_OK;
        case 4: *p = a->terminals; *bytes = N * T; return B200RL_OK;
        case 5: *p = a->values; *bytes = N * (T + 1) * 4; return B200RL_OK;
        case 6: *p = a->adv; *bytes = N * T * 4; return B200RL_OK;
        case 7: *p = a->ret; *bytes = N * T * 4; return B200RL_OK;
        case 8: *p = a->rng; *bytes = N * 32; return B200RL_OK;
        case 9: *p = a->norm2; *bytes = 8; return B200RL_OK;
    }
    REQUIRE(false, B200RL_ERR_INVALID, "unknown field");
}

extern "C" {

int b200rl_onpolicy_destroy(b200rl_onpolicy* a) {
    if (!a) return B200RL_OK;
    cudaSetDevice(a->ctx->device);
    cudaStreamSynchronize(a->ctx->stream);
    b200rl_env_internal_set_traj_targets(a->env, nullptr, nullptr);
    cudaFree(a->rng); cudaFree(a->states); cudaFree(a->actions); cudaFree(a->logp); cudaFree(a->rewards); cudaFree(a->terminals);
    cudaFree(a->values); cudaFree(a->adv); cudaFree(a->ret); cudaFree(a->act_clamped); cudaFree(a->norm_partials); cudaFree(a->norm_sums);
    cudaFree(a->norm2); cudaFree(a->perm_dev); cudaFree(a->stats_dev); cudaFree(a->rec); cudaFree(a->upd_dev);
    a->stop.release();
    delete a;
    return B200RL_OK;
}

/* Agent(policy = PPOPolicy / A2CPolicy, trajectory = PPOTrajectory(capacity = update_freq)):
 * rollout tensors (N, T) env-fastest live on the device.  policy_rng: (4, N) host uint64, one
 * Xoshiro stream per env for action sampling (the reference draws a whole batch from one stream). */
int b200rl_onpolicy_create(b200rl_ctx* ctx, b200rl_net* net, b200rl_env* env, const b200rl_onpolicy_config* cfg, const uint64_t* policy_rng,
                           b200rl_onpolicy** out) {
    TRY(ctx_bind(ctx));
    REQUIRE(net && env && cfg && policy_rng && out, B200RL_ERR_INVALID, "null argument");
    REQUIRE(!is_q_kind(net->kind), B200RL_ERR_INVALID, "needs an actor-critic network");
    REQUIRE(net->ctx == ctx && b200rl_env_internal_ctx(env) == ctx, B200RL_ERR_INVALID, "net/env belong to another ctx");
    const float* obs;
    TRY(learner_obs(env, &obs));
    REQUIRE(cfg->update_freq >= 1 && cfg->n_epochs >= 1 && cfg->n_microbatches >= 1, B200RL_ERR_INVALID, "bad config");
    int nobs = b200rl_env_internal_nobs(env);
    REQUIRE(nobs == net->actor.in, B200RL_ERR_INVALID, "network input width != observation width");
    bool cont = b200rl_env_internal_continuous(env);
    REQUIRE(cont == (net->kind == 1), B200RL_ERR_INVALID, "categorical policy needs a discrete env, gaussian a continuous one");
    int64_t N = b200rl_env_internal_n(env);
    REQUIRE((N * cfg->update_freq) % cfg->n_microbatches == 0, B200RL_ERR_INVALID, "N*T must be divisible by n_microbatches");
    REQUIRE(N * (int64_t)cfg->update_freq < (1ll << 31), B200RL_ERR_UNSUPPORTED, "rollout too large for 32-bit sample indices");
    b200rl_onpolicy* a = new b200rl_onpolicy();   // (value-initialised: every pointer and counter starts at zero)
    a->ctx = ctx; a->net = net; a->env = env; a->cfg = *cfg; a->N = N; a->T = cfg->update_freq; a->t = 0; a->ns = nobs; a->continuous = cont;
    size_t NT_ = (size_t)N * a->T;
#define A_TRY(x) CUDA_TRY_OR(x, b200rl_onpolicy_destroy(a))
    A_TRY(cudaMalloc(&a->rng, (size_t)N * 32));
    A_TRY(cudaMalloc(&a->states, (size_t)N * nobs * (a->T + 1) * 4));
    A_TRY(cudaMalloc(&a->actions, NT_ * 4)); A_TRY(cudaMalloc(&a->logp, NT_ * 4)); A_TRY(cudaMalloc(&a->rewards, NT_ * 4));
    A_TRY(cudaMalloc(&a->terminals, NT_)); A_TRY(cudaMalloc(&a->values, (size_t)N * (a->T + 1) * 4));
    A_TRY(cudaMalloc(&a->adv, NT_ * 4)); A_TRY(cudaMalloc(&a->ret, NT_ * 4));
    A_TRY(cudaMalloc(&a->act_clamped, (size_t)N * 8));   // (N) T
    A_TRY(cudaMalloc(&a->norm_partials, (size_t)b200rl_gae_fused_partials_count(N) * sizeof(double)));
    A_TRY(cudaMalloc(&a->norm_sums, 2 * sizeof(double))); A_TRY(cudaMalloc(&a->norm2, 2 * sizeof(float)));
    a->stats_rows = cfg->n_epochs * cfg->n_microbatches;
    A_TRY(cudaMalloc(&a->stats_dev, (size_t)a->stats_rows * 8 * sizeof(float)));
    // staging for host-supplied shuffle!() results; allocated here because a device allocation inside update would
    // synchronise the device (and with it another rank of the same process that is waiting in the peer exchange)
    A_TRY(cudaMalloc(&a->perm_dev, (size_t)a->cfg.n_epochs * NT_ * 4));
    A_TRY(cudaMalloc(&a->rec, NT_ * 32));
    A_TRY(cudaMalloc(&a->upd_dev, sizeof(unsigned int)));
    A_TRY(cudaMemsetAsync(a->upd_dev, 0, sizeof(unsigned int), ctx->stream));
    A_TRY(cudaMemsetAsync(a->stats_dev, 0, (size_t)a->stats_rows * 8 * sizeof(float), ctx->stream));
    A_TRY(cudaMemcpyAsync(a->rng, policy_rng, (size_t)N * 32, cudaMemcpyHostToDevice, ctx->stream));
    A_TRY(cudaStreamSynchronize(ctx->stream));
#undef A_TRY
    TRY(b200rl_net_configure_optimizer(net, cfg->lr, cfg->beta1, cfg->beta2, cfg->eps, cfg->max_grad_norm));
    *out = a;
    return B200RL_OK;
}

/* RLBase.plan!(agent, env) + push!(agent, PreActStage): K6 on the env's current observation;
 * stores state / log-prob / V(s) into column t of the rollout and arms the env so that the
 * next act! writes reward / terminal into the same column.  actions_host (N) may be NULL. */
int b200rl_onpolicy_plan(b200rl_onpolicy* a, void* actions_host) {
    REQUIRE(a, B200RL_ERR_INVALID, "null agent");
    REQUIRE(a->t < a->T, B200RL_ERR_INVALID, "rollout is full: call b200rl_onpolicy_update first");
    TRY(ctx_bind(a->ctx));
    a->bootstrap_done = false;
    int64_t N = a->N;
    const float* obs;
    TRY(learner_obs(a->env, &obs));
    char* act_col = (char*)a->actions + (size_t)N * a->t * 4;
    TRY(nn_policy_act(a->ctx, a->net->actor, a->net->critic, a->net->params, ac_hyper(a->cfg), obs, N, a->rng, act_col, a->logp + (size_t)N * a->t,
                      a->values + (size_t)N * a->t, nullptr, a->states + (size_t)N * a->ns * a->t));
    TRY(b200rl_env_internal_set_traj_targets(a->env, a->rewards + (size_t)N * a->t, a->terminals + (size_t)N * a->t));
    if (actions_host) {
        CUDA_TRY(cudaMemcpyAsync(actions_host, act_col, (size_t)N * 4, cudaMemcpyDeviceToHost, a->ctx->stream));
        CUDA_TRY(cudaStreamSynchronize(a->ctx->stream));
    }
    return B200RL_OK;
}
/* RLBase.act!(env, planned action) device-to-device (auto-reset fused) */
int b200rl_onpolicy_act(b200rl_onpolicy* a) {
    REQUIRE(a, B200RL_ERR_INVALID, "null agent");
    TRY(ctx_bind(a->ctx));
    char* act_col = (char*)a->actions + (size_t)a->N * a->t * 4;
    if (a->continuous) {  // the env asserts a in its action space; the stored (unclamped) action keeps its log-prob
        TRY(env_action_clamped(a->env, (const float*)act_col, a->N, a->act_clamped));
        return b200rl_env_step(a->env, a->act_clamped, 1, 1);
    }
    return b200rl_env_step(a->env, act_col, 1, 1);
}
/* push!(agent, PostActStage, env, action): the transition of column t is complete */
int b200rl_onpolicy_push(b200rl_onpolicy* a) {
    REQUIRE(a, B200RL_ERR_INVALID, "null agent");
    REQUIRE(a->t < a->T, B200RL_ERR_INVALID, "rollout is full");
    a->t += 1;
    b200rl_env_internal_set_traj_targets(a->env, nullptr, nullptr);
    return B200RL_OK;
}
/* n x (plan! -> act! -> push!) without leaving the device */
int b200rl_onpolicy_collect(b200rl_onpolicy* a, int n_steps) {
    REQUIRE(a && n_steps >= 0, B200RL_ERR_INVALID, "bad argument");
    if (n_steps > 0 && nn_tc_enabled()) {   // one launch for the whole stretch (fwd_tc.cu)
        REQUIRE(a->t + n_steps <= a->T, B200RL_ERR_INVALID, "rollout is full: call b200rl_onpolicy_update first");
        const float* obs;
        TRY(learner_obs(a->env, &obs));   // (the wrapper may have been removed since create)
        TRY(ctx_bind(a->ctx));
        const int fin = a->t + n_steps == a->T ? 1 : 0;
        int st = nn_tc_rollout(a->ctx, a->env, a->net->actor, a->net->critic, a->net->params, ac_hyper(a->cfg), a->rng, a->t, n_steps, a->T, fin, a->states,
                               a->actions, a->logp, a->values, a->rewards, a->terminals);
        if (st == B200RL_OK) {
            a->t += n_steps;
            a->bootstrap_done = fin != 0;
            return B200RL_OK;
        }
        if (st != B200RL_ERR_UNSUPPORTED) return st;
    }
    for (int k = 0; k < n_steps; ++k) {
        TRY(b200rl_onpolicy_plan(a, nullptr));
        TRY(b200rl_onpolicy_act(a));
        TRY(b200rl_onpolicy_push(a));
    }
    return B200RL_OK;
}
int b200rl_onpolicy_fill(b200rl_onpolicy* a, int* t_out, int* T_out) {
    REQUIRE(a, B200RL_ERR_INVALID, "null agent");
    if (t_out) *t_out = a->t;
    if (T_out) *T_out = a->T;
    return B200RL_OK;
}

/* optimise!(agent): V(s_{T+1}), GAE (+returns, advantage normalisation), then n_epochs x
 * n_microbatches of {loss+grad, reduce, [all-reduce], clip + Adam}.  perm_host: optional
 * (n_epochs, N*T) int32 0-based permutations (the host's shuffle!); NULL = device Feistel
 * permutation keyed by (update counter, epoch).  stats_host: optional (n_epochs*n_microbatches, 6)
 * floats [actor_loss, critic_loss, entropy, loss, grad_norm, 0] (forces a sync). */
int b200rl_onpolicy_update(b200rl_onpolicy* a, const int32_t* perm_host, float* stats_host) {
    REQUIRE(a, B200RL_ERR_INVALID, "null agent");
    REQUIRE(a->t == a->T, B200RL_ERR_INVALID, "rollout not full yet");
    TRY(ctx_bind(a->ctx));
    b200rl_ctx* ctx = a->ctx;
    b200rl_net* n = a->net;
    const b200rl_onpolicy_config& c = a->cfg;
    int64_t N = a->N, T = a->T, NT_ = N * T;
    int world = b200rl_comm_world(ctx);
    // measurement aid (b200rl_debug_phase_slots): events between the phases, eager path only
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    CUDA_TRY(cudaStreamIsCapturing(ctx->stream, &cap));
    const int pb = (cap == cudaStreamCaptureStatusNone && ctx->phase_base + 3 + 2 * a->stats_rows <= b200rl_ctx::kTimerSlots) ? ctx->phase_base : -1;
    auto phase = [&](int k) -> int { return pb >= 0 ? b200rl_timer_record(ctx, pb + k) : B200RL_OK; };
    TRY(phase(0));
    // bootstrap value of the state after the last step
    const float* obs;
    TRY(learner_obs(a->env, &obs));
    // (a copy kernel, not cudaMemcpyAsync D2D: device-to-device copies are on CUDA's implicit-synchronisation list)
    if (!a->bootstrap_done) {   // (the fused rollout has already written column T of states / values)
        copy_f32_kernel<<<grid_for(N * a->ns, 256), 256, 0, ctx->stream>>>(a->states + (size_t)N * a->ns * T, obs, N * a->ns);
        LAUNCH_CHECK(ctx);
        TRY(nn_mlp_forward(ctx, n->critic, n->params + n->actor.nparams(), obs, N, a->values + (size_t)N * T));
    }
    a->bootstrap_done = false;
    // GAE + returns + normalisation sums
    int n_part = b200rl_gae_fused_partials_count(N) / 2;
    TRY(b200rl_gae_fused_internal(ctx, a->adv, a->ret, a->rewards, a->values, a->terminals, c.gamma, c.lambda, N, T,
                                  c.normalize_advantage ? a->norm_partials : nullptr));
    if (c.algo == 1) {  // A2C: critic target = discounted gains bootstrapped with V(s_{T+1})
        TRY(b200rl_discount_rewards_f32(ctx, a->ret, a->rewards, a->terminals, a->values + (size_t)N * T, c.gamma, N, T, 2, 1));
    }
    if (c.normalize_advantage) {
        sum_norm_partials_kernel<<<1, 32, 0, ctx->stream>>>(a->norm_partials, n_part, a->norm_sums);
        LAUNCH_CHECK(ctx);
        if (world > 1) TRY(b200rl_comm_allreduce_internal(ctx, a->norm_sums, 2, 1));
        finalize_norm2_kernel<<<1, 32, 0, ctx->stream>>>(a->norm_sums, (double)NT_ * (double)world, a->norm2);
        LAUNCH_CHECK(ctx);
    }
    {   // one 32-byte record per sample for the permuted minibatch gathers (n_epochs x n_microbatches of them follow)
        const unsigned g = grid_for(NT_, 256);
        const uint32_t* act = (const uint32_t*)a->actions;
        switch (a->ns) {
            case 1: pack_records_kernel<1><<<g, 256, 0, ctx->stream>>>(a->rec, a->states, act, a->logp, a->adv, a->ret, NT_); break;
            case 2: pack_records_kernel<2><<<g, 256, 0, ctx->stream>>>(a->rec, a->states, act, a->logp, a->adv, a->ret, NT_); break;
            case 3: pack_records_kernel<3><<<g, 256, 0, ctx->stream>>>(a->rec, a->states, act, a->logp, a->adv, a->ret, NT_); break;
            default: pack_records_kernel<4><<<g, 256, 0, ctx->stream>>>(a->rec, a->states, act, a->logp, a->adv, a->ret, NT_); break;
        }
        LAUNCH_CHECK(ctx);
    }
    if (perm_host) {
        CUDA_TRY(cudaMemcpyAsync(a->perm_dev, perm_host, (size_t)c.n_epochs * NT_ * 4, cudaMemcpyHostToDevice, ctx->stream));
    }
    TRY(phase(1));
    const AcHyper hp = ac_hyper(c);
    int64_t B = NT_ / c.n_microbatches;
    int row = 0;
    for (int e = 0; e < c.n_epochs; ++e) {
        for (int mb = 0; mb < c.n_microbatches; ++mb, ++row) {
            // permutation key = n_updates * 1000003 + e * 7919 + 12345; the update counter is read from device memory (upd_dev)
            // so that a captured iteration can be replayed
            AcBatch b{a->states, a->ns, a->actions, a->logp, a->adv, a->ret,
                      perm_host ? a->perm_dev + (size_t)e * NT_ + (size_t)mb * B : nullptr,
                      (uint32_t)NT_, (uint32_t)e * 7919u + 12345u, (uint32_t)(mb * B), a->upd_dev, a->rec, B,
                      1.0f / ((float)B * (float)world), a->norm2};
            float* stats_row = a->stats_dev + (size_t)row * 8;
            unsigned int* tick = row == a->stats_rows - 1 ? a->upd_dev : nullptr;   // the last optimiser step closes the update
            // one launch: loss + backward + [peer exchange] + clip + Adam (tensor-core path); otherwise loss + backward, then the
            // optimiser step
            const OptStep st = opt_step(n, c, stats_row, tick);
            int ctas = nn_ac_loss_grad_step(ctx, n->actor, n->critic, hp, b, n->partial, n->loss_partial, st);
            const bool staged = ctas == B200RL_ERR_UNSUPPORTED;
            if (staged) ctas = nn_ac_loss_grad(ctx, n->actor, n->critic, n->params, hp, b, n->partial, n->loss_partial);
            if (ctas < 0) return ctas;
            TRY(phase(2 + 2 * row));
            if (staged) TRY(optimiser_step(n, ctas, 2 * ctas, st));
            TRY(phase(3 + 2 * row));
            n->n_updates += 1;
        }
    }
    a->n_updates += 1;
    a->t = 0;
    if (stats_host) TRY(read_stats(a, stats_host));
    return B200RL_OK;
}

/* n_iters x { collect(T); update } — the whole PPO / A2C iteration (fused rollout, bootstrap, GAE, record packing, n_epochs x
 * n_microbatches x {loss + backward, [peer exchange +] clip + Adam}) replayed as ONE CUDA graph launch per iteration, so
 * the ranks of a sharded run cannot drift apart on host launch jitter (they meet 17 times per iteration inside the peer
 * exchange).  Needs an empty rollout (t = 0).  Every per-launch counter lives in device memory (update counter, exchange
 * sequence numbers, self-resetting grid barrier), so the captured launches are replayable as they are.  The first
 * iteration ever runs eagerly (lazy module loading, scratch growth, function attributes), the second is captured.
 * stats_host: optional (n_epochs * n_microbatches, 6) rows of the LAST iteration (forces a sync).
 * Falls back to eager launches when capture is impossible (NCCL path without the peer exchange). */
int b200rl_onpolicy_iterate(b200rl_onpolicy* a, int n_iters, float* stats_host) {
    REQUIRE(a && n_iters >= 0, B200RL_ERR_INVALID, "bad argument");
    REQUIRE(a->t == 0, B200RL_ERR_INVALID, "iterate needs an empty rollout (t = 0)");
    const float* obs;
    TRY(learner_obs(a->env, &obs));
    TRY(ctx_bind(a->ctx));
    b200rl_ctx* ctx = a->ctx;
    P2PTable peers;
    const bool capturable = b200rl_comm_world(ctx) == 1 || b200rl_comm_p2p_table(ctx, &peers);
    // launch arguments the graph bakes in
    struct { int tc, max_timeout, state_f32, pad; uint64_t log[4]; } key = {nn_tc_enabled() ? 1 : 0, b200rl_env_internal_max_timeout(a->env),
                                                                             b200rl_env_internal_state_f32(a->env) ? 1 : 0, 0, {}};
    b200rl_env_internal_log_key(a->env, key.log);
    a->graph.rekey(&key, sizeof key);
    const CounterSet counters{ctx, a->net, a->env, nullptr, &a->n_updates};
    for (int it = 0; it < n_iters; ++it) {
        TRY(a->graph.run(0, counters, capturable, [&]() -> int {
            a->t = 0; a->bootstrap_done = false;   // (a no-op, unless a capture that failed part-way left the rollout filled)
            TRY(b200rl_onpolicy_collect(a, a->T));
            return b200rl_onpolicy_update(a, nullptr, nullptr);
        }));
    }
    if (stats_host && n_iters > 0) TRY(read_stats(a, stats_host));
    return B200RL_OK;
}
/* The on-policy agent's part of run_stretches.  A stretch is the rest of the rollout (collect(T - t), capped by max_steps); a whole
 * rollout that cannot reach the budget runs as one graph launch (b200rl_onpolicy_iterate), whose update leaves the terminal columns as
 * they are.  A full rollout is updated, as optimise! at the PostActStage of its last step would; the update of a stretch that could
 * reach the budget runs only after the count, so the network never needs a shadow. */
struct OnPolicyStretches {
    b200rl_onpolicy* a;
    bool whole = false, updated = false;
    struct Saved { int t; bool bootstrap_done; uint64_t env_steps; };
    Saved save() const { return {a->t, a->bootstrap_done, b200rl_env_internal_steps(a->env)}; }
    void restore(const Saved& s0) const {
        a->t = s0.t;
        a->bootstrap_done = s0.bootstrap_done;
        b200rl_env_internal_add_steps(a->env, s0.env_steps - b200rl_env_internal_steps(a->env));
    }
    size_t shadow_bytes() const {
        size_t bytes = b200rl_env_internal_step_bytes_max(a->env) + round256((size_t)a->N * 32);
        for (int f = 0; f <= 5; ++f) {
            void* p; size_t b;
            rollout_field(a, f, &p, &b);
            bytes += round256(b);
        }
        return bytes;
    }
    int64_t longest() const { return a->T; }
    int mark(Shadow& sh) const {
        DevRegion er[kEnvStepRegionsMax];
        TRY(sh.add_regions(er, b200rl_env_internal_step_regions(a->env, er)));
        TRY(sh.add(a->rng, (size_t)a->N * 32));
        for (int f = 0; f <= 5; ++f) {
            void* p; size_t bytes;
            TRY(rollout_field(a, f, &p, &bytes));
            TRY(sh.add(p, bytes));
        }
        return B200RL_OK;
    }
    int64_t stretch(int64_t left, bool, int64_t) const { return a->T - a->t < left ? a->T - a->t : left; }
    int run(int64_t s, bool may_stop) {
        whole = !may_stop && a->t == 0 && s == a->T;
        if (!whole) return b200rl_onpolicy_collect(a, (int)s);
        updated = true;
        return b200rl_onpolicy_iterate(a, 1, nullptr);
    }
    int count(int64_t s, const Saved& s0, unsigned long long* counts) const {
        b200rl_ctx* ctx = a->ctx;
        stop::count_columns_kernel<<<dim3(grid_for(a->N, stop::kCountBlock), (unsigned)(s < 65535 ? s : 65535)), stop::kCountBlock, 0,
                                      ctx->stream>>>(a->terminals, a->N, s0.t, (int)s, counts);
        LAUNCH_CHECK(ctx);
        return B200RL_OK;
    }
    int end_stretch() {
        if (whole || a->t != a->T) return B200RL_OK;
        updated = true;
        return b200rl_onpolicy_update(a, nullptr, nullptr);
    }
    bool at_boundary(int64_t left) const { return a->t == 0 && left < a->T; }
};

/* run(agent, env, StopAfterNSteps | StopAfterNEpisodes(k)) for at most max_steps env steps (include/b200rl.h): run_stretches */
int b200rl_onpolicy_run_episodes(b200rl_onpolicy* a, int64_t max_steps, int64_t budget, float* stats_host, int64_t* steps_done,
                                 int64_t* episodes_done) {
    REQUIRE(a && steps_done && episodes_done && max_steps >= 1, B200RL_ERR_INVALID, "bad argument");
    REQUIRE(budget < 0 || b200rl_comm_world(a->ctx) == 1, B200RL_ERR_UNSUPPORTED,
            "StopAfterNEpisodes counts the episodes of every rank: a sharded ctx keeps the stage loop");
    const float* obs;
    TRY(learner_obs(a->env, &obs));
    TRY(ctx_bind(a->ctx));
    OnPolicyStretches ops{a};
    TRY(run_stretches(a->ctx, a->stop, a->N, ops, max_steps, budget, steps_done, episodes_done));
    if (stats_host && ops.updated) TRY(read_stats(a, stats_host));
    return B200RL_OK;
}

/* 1 when b200rl_onpolicy_iterate replays a captured graph, 0 when it launches eagerly (diagnostic for tests / bench) */
int b200rl_onpolicy_graph_active(b200rl_onpolicy* a, int* out) {
    REQUIRE(a && out, B200RL_ERR_INVALID, "null argument");
    *out = a->graph.active() ? 1 : 0;
    return B200RL_OK;
}

/* rollout tensors for inspection / parity tests (fields: rollout_field) */
int b200rl_onpolicy_get(b200rl_onpolicy* a, int field, void* host_dst, size_t bytes) {
    REQUIRE(a && host_dst, B200RL_ERR_INVALID, "null argument");
    TRY(ctx_bind(a->ctx));
    void* src;
    size_t need;
    TRY(rollout_field(a, field, &src, &need));
    REQUIRE(bytes >= need, B200RL_ERR_INVALID, "destination too small");
    CUDA_TRY(cudaMemcpyAsync(host_dst, src, need, cudaMemcpyDeviceToHost, a->ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(a->ctx->stream));
    return B200RL_OK;
}

/* checkpoint import: fields 0-5 and 8 of b200rl_onpolicy_get (advantages / returns / normalisation are recomputed by update) */
int b200rl_onpolicy_set(b200rl_onpolicy* a, int field, const void* host_src, size_t bytes) {
    REQUIRE(a && host_src, B200RL_ERR_INVALID, "null argument");
    REQUIRE(field != 6 && field != 7 && field != 9, B200RL_ERR_INVALID, "field not settable");
    TRY(ctx_bind(a->ctx));
    void* dst;
    size_t need;
    TRY(rollout_field(a, field, &dst, &need));
    REQUIRE(bytes >= need, B200RL_ERR_INVALID, "source too small");
    CUDA_TRY(cudaMemcpyAsync(dst, host_src, need, cudaMemcpyHostToDevice, a->ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(a->ctx->stream));
    return B200RL_OK;
}
int b200rl_onpolicy_export_state(b200rl_onpolicy* a, int64_t* c3) {
    REQUIRE(a && c3, B200RL_ERR_INVALID, "null argument");
    c3[0] = a->t; c3[1] = (int64_t)a->n_updates; c3[2] = (int64_t)a->net->n_updates;
    return B200RL_OK;
}
int b200rl_onpolicy_import_state(b200rl_onpolicy* a, const int64_t* c3) {
    REQUIRE(a && c3, B200RL_ERR_INVALID, "null argument");
    REQUIRE(c3[0] >= 0 && c3[0] <= a->T && c3[1] >= 0 && c3[2] >= 0, B200RL_ERR_INVALID, "counters out of range");
    a->t = (int)c3[0]; a->n_updates = (uint64_t)c3[1]; a->net->n_updates = (uint64_t)c3[2];
    TRY(ctx_bind(a->ctx));
    const unsigned int upd = (unsigned int)a->n_updates;   // the device copy keys the minibatch permutation
    CUDA_TRY(cudaMemcpyAsync(a->upd_dev, &upd, sizeof upd, cudaMemcpyHostToDevice, a->ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(a->ctx->stream));
    a->bootstrap_done = false;   // column T of states / values is rewritten from the env's observation by the next update
    b200rl_env_internal_set_traj_targets(a->env, nullptr, nullptr);
    return B200RL_OK;
}

/* Measurement aid (bench.py roofline): average device time of `reps` back-to-back launches of one
 * hot-path kernel on the agent's current tensors, CUDA events on the ctx stream.
 * which: 0 loss+backward minibatch kernel (K7) | 1 policy inference (K6) | 2 env step (K1, mutates the env) |
 * 3 fused GAE (K5) | 4 partial reduce + clip + Adam (K8) */
int b200rl_onpolicy_time_kernel(b200rl_onpolicy* a, int which, int reps, float* avg_ms_out) {
    REQUIRE(a && avg_ms_out && reps >= 1, B200RL_ERR_INVALID, "bad argument");
    TRY(ctx_bind(a->ctx));
    b200rl_ctx* ctx = a->ctx;
    b200rl_net* n = a->net;
    const b200rl_onpolicy_config& c = a->cfg;
    int64_t N = a->N, T = a->T, NT_ = N * T, B = NT_ / c.n_microbatches;
    const AcHyper hp = ac_hyper(c);
    const float* obs;
    TRY(learner_obs(a->env, &obs));
    int ctas = (nn_tc_enabled() && nn_tc_bwd_supported(n->actor, n->critic)) ? nn_tc_partial_rows(2 * (ctx->sm_count / 2), n->actor, hp, B) : nn_grid_ctas(ctx, n->actor.H);
    void* rng_copy = nullptr;
    if (which == 1) {
        TRY(ctx_scratch(ctx, (size_t)N * 32 + (size_t)N * 12 + 256, &rng_copy));
        CUDA_TRY(cudaMemcpyAsync(rng_copy, a->rng, (size_t)N * 32, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    auto once = [&]() -> int {
        switch (which) {
            case 0: {
                AcBatch b{a->states, a->ns, a->actions, a->logp, a->adv, a->ret, nullptr, (uint32_t)NT_, 12345u, 0u, nullptr, a->rec, B, 1.0f / (float)B,
                          a->norm2};
                int st = nn_ac_loss_grad(ctx, n->actor, n->critic, n->params, hp, b, n->partial, n->loss_partial);
                return st < 0 ? st : B200RL_OK;
            }
            case 1: {
                float* o = (float*)((char*)rng_copy + (size_t)N * 32);
                return nn_policy_act(ctx, n->actor, n->critic, n->params, hp, obs, N, (unsigned long long*)rng_copy, o, o + N, o + 2 * N, nullptr, nullptr);
            }
            case 2: return b200rl_env_step(a->env, a->actions, 1, 1);
            case 3: return b200rl_gae_fused_internal(ctx, a->adv, a->ret, a->rewards, a->values, a->terminals, c.gamma, c.lambda, N, T, a->norm_partials);
            // the optimiser step as update() runs it (lr = 0: parameters stay put), incl. the peer exchange of a sharded run
            case 4: {
                OptStep st = opt_step(n, c);
                st.lr = 0.0f;
                return optimiser_step(n, ctas, 2 * ctas, st);
            }
        }
        b200rl_set_error("unknown kernel id");
        return B200RL_ERR_INVALID;
    };
    REQUIRE(!(which == 2 && a->continuous), B200RL_ERR_UNSUPPORTED, "env-step timing uses the discrete action column");
    TRY(once());  // warm-up
    CUDA_TRY(cudaEventRecord(ctx->ev0, ctx->stream));
    for (int r = 0; r < reps; ++r) TRY(once());
    CUDA_TRY(cudaEventRecord(ctx->ev1, ctx->stream));
    CUDA_TRY(cudaEventSynchronize(ctx->ev1));
    float ms = 0.f;
    CUDA_TRY(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
    *avg_ms_out = ms / (float)reps;
    return B200RL_OK;
}

// ------------------------------------------------------------------ DQN ---------------------
/* push!(trajectory, env): append the env's last transition (action, reward, terminal, next obs) — all on device.
 * first_state_only 1: episode-start frame for every lane (PreEpisodeStage); 2: only for the lanes whose last transition was terminal */
int b200rl_traj_push_env(b200rl_traj* t, b200rl_env* env, int first_state_only) {
    REQUIRE(t && env, B200RL_ERR_INVALID, "null argument");
    REQUIRE(b200rl_traj_internal_lanes(t) == b200rl_env_internal_n(env), B200RL_ERR_INVALID, "trajectory lanes != number of envs");
    const float* obs;   // (the trajectory stores Float32 states)
    TRY(learner_obs(env, &obs));
    if (first_state_only == 2) return b200rl_traj_push_episode_start(t, obs, 1, 1);   // only the lanes whose episode has ended (soft reset)
    if (first_state_only) return b200rl_traj_push_state(t, obs, 1);
    const float* rew;
    TRY(b200rl_env_internal_reward_f32(env, &rew));
    return b200rl_traj_push(t, (const int32_t*)env_field(env, B200RL_FIELD_ACTION), rew, (const uint8_t*)env_field(env, B200RL_FIELD_FLAGS), obs, 1);
}

/* optimise!(DQNLearner / PrioritizedDQNLearner, batch): sample + gather (K4), TD loss + backward
 * (K7), clip + Adam (K8), priority write-back, target sync every target_update_freq updates.
 * upd_dev (may be null): the sync phase is counted on the device (nn_target_sync_counted) instead of by a host `if`, so the
 * sequence can be captured and replayed; n->n_updates advances either way.  td_keep (may be null): copy of the TD errors. */
static int dqn_update_seq(b200rl_net* n, b200rl_traj* t, const b200rl_dqn_config* cfg, unsigned long long* upd_dev, float* td_keep,
                          float** td_out) {
    b200rl_ctx* ctx = n->ctx;
    TRY(b200rl_traj_sample(t, cfg->per_beta));
    TrajBatchView b = b200rl_traj_internal_batch(t);
    REQUIRE(b.ns == n->actor.in, B200RL_ERR_INVALID, "state width mismatch");
    void* sc;
    // scratch: [Q tables: 2*B*nout] used inside nn_dqn_loss_grad, td after them
    size_t q_bytes = (size_t)b.B * n->actor.nout * 4 * 2 + 256;
    TRY(ctx_scratch(ctx, q_bytes + (size_t)b.B * 4 + 256, &sc));
    float* td = (float*)((char*)sc + q_bytes);
    int world = b200rl_comm_world(ctx);
    int np_ = nn_dqn_loss_grad(ctx, n->actor, n->params, n->target, b.s, b.a, b.r, b.t, b.s2, b.w, b.B, 1.0f / ((float)b.B * (float)world), cfg->gamma,
                               cfg->huber, cfg->double_dqn, n->partial, n->loss_partial, td, b200rl_traj_internal_discount(t));
    if (np_ < 0) return np_;
    TRY(optimiser_step(n, np_, np_, opt_step(n, *cfg)));
    if (b200rl_traj_internal_prioritized(t)) TRY(b200rl_traj_internal_priority_from_td(t, td, cfg->per_eps, cfg->per_alpha));
    n->n_updates += 1;
    if (upd_dev) TRY(nn_target_sync_counted(ctx, n->target, n->params, n->np, cfg->rho, upd_dev, cfg->target_update_freq));
    else if (cfg->target_update_freq > 0 && n->n_updates % (uint64_t)cfg->target_update_freq == 0) TRY(nn_target_sync(ctx, n->target, n->params, n->np, cfg->rho));
    if (td_keep) {
        copy_f32_kernel<<<grid_for(b.B, 256), 256, 0, ctx->stream>>>(td_keep, td, b.B);
        LAUNCH_CHECK(ctx);
    }
    if (td_out) *td_out = td;
    return B200RL_OK;
}
// an n-step sampler discounts its windows by its own γ: the learner's must be the same one
static int check_nstep_gamma(b200rl_traj* t, const b200rl_dqn_config* cfg) {
    int ns; float g;
    b200rl_traj_internal_nstep(t, &ns, &g);
    REQUIRE(ns == 1 || g == cfg->gamma, B200RL_ERR_INVALID, "the trajectory's n-step gamma differs from the learner's gamma");
    return B200RL_OK;
}
// stats4 = loss, grad_norm, mean |td|, n_updates of the update that wrote loss4 / gnorm / td (synchronises)
static int dqn_stats(b200rl_net* n, const float* td, int64_t B, float* stats4) {
    b200rl_ctx* ctx = n->ctx;
    float l4[4], gn;
    std::vector<float> tdh((size_t)B);
    CUDA_TRY(cudaMemcpyAsync(l4, n->loss4, 16, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(&gn, n->gnorm, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(tdh.data(), td, (size_t)B * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    double s = 0;
    for (float x : tdh) s += x < 0 ? -x : x;
    const int world = b200rl_comm_world(ctx);
    stats4[0] = l4[0] / ((float)B * (float)world); stats4[1] = gn; stats4[2] = (float)(s / (double)B);
    stats4[3] = (float)n->n_updates;
    return B200RL_OK;
}

int b200rl_dqn_update(b200rl_net* n, b200rl_traj* t, const b200rl_dqn_config* cfg, float* stats_host) {
    REQUIRE(n && t && cfg && is_q_kind(n->kind), B200RL_ERR_INVALID, "bad argument (needs a Q-network)");
    REQUIRE(n->ctx == b200rl_traj_internal_ctx(t), B200RL_ERR_INVALID, "net/trajectory belong to different ctx");
    TRY(check_nstep_gamma(t, cfg));
    TRY(ctx_bind(n->ctx));
    float* td = nullptr;
    TRY(dqn_update_seq(n, t, cfg, nullptr, nullptr, &td));
    if (stats_host) TRY(dqn_stats(n, td, b200rl_traj_internal_batch(t).B, stats_host));
    return B200RL_OK;
}
/* TD errors (B floats) of the batch used by the last b200rl_dqn_update (for parity tests) */
int b200rl_dqn_last_td(b200rl_net* n, b200rl_traj* t, float* host_dst, int64_t count) {
    REQUIRE(n && t && host_dst, B200RL_ERR_INVALID, "null argument");
    TRY(ctx_bind(n->ctx));
    TrajBatchView b = b200rl_traj_internal_batch(t);
    REQUIRE(count >= b.B, B200RL_ERR_INVALID, "destination too small");
    size_t q_bytes = (size_t)b.B * n->actor.nout * 4 * 2 + 256;
    REQUIRE(n->ctx->scratch_bytes >= q_bytes + (size_t)b.B * 4, B200RL_ERR_INVALID, "no update has run yet");
    CUDA_TRY(cudaMemcpyAsync(host_dst, (char*)n->ctx->scratch + q_bytes, (size_t)b.B * 4, cudaMemcpyDeviceToHost, n->ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(n->ctx->stream));
    return B200RL_OK;
}

}  // extern "C"

// ------------------------------------------------------------------ DQN agent loop ---------
namespace {
__global__ void add_i64_kernel(long long* __restrict__ v, long long d) { *v += d; }
}  // namespace

constexpr int64_t kStopChunkMax = 2048;   // steps per chunk of b200rl_replay_run_episodes (its counts sit in shared memory)
constexpr int kAgree = 21;   // values of the agreement exchange of a sharded run (replay_agree)
// what the captured launches bake in besides the handles: a change means re-capture
struct ReplayKey {
    int tc, max_timeout, greedy, state_f32;
    int nstep_n; float nstep_gamma;  // the sampler's n-step setting (picks the sample kernel and its window arguments)
    b200rl_explorer ex;          // step zeroed (it lives in device memory)
    const void* rng;
    const void* scratch;
    const void* keys;
    uint64_t log[4];             // the env's episode log
};
struct b200rl_replay {
    b200rl_ctx* ctx;
    b200rl_net* net;
    b200rl_env* env;
    b200rl_traj* traj;
    b200rl_dqn_config cfg;
    int64_t N, B;
    int32_t* action;              // (N) planned actions
    long long* ex_step_dev;       // explorer step, advanced by N · world per step on the device
    unsigned long long* upd_dev;  // optimiser steps of the Q-network (the target-sync phase), advanced per update on the device
    float* td_keep;               // TD errors of the last update
    int64_t* keys; float* vals;   // (stride, N) sum-tree leaves a fused collect window touched (prioritised ring)
    int stride_cap;               // rows of keys / vals allocated
    long long h_counters[2];
    double* agree_dev;            // (world, 2 kAgree) table of the agreement exchange (sharded ctx)
    GraphUnit graphs;             // "1 step + m updates" units, by m
    StopBuffers stop;             // b200rl_replay_run_episodes with a budget: env arrays, ring, explorer streams, Q-network
    int64_t stop_chunk;           // longest chunk whose pushes the ring still holds: 2 s + 1 <= cap + 1 frames
};

// plan! -> act! -> push!(trajectory): the launches of the stage protocol (QBasedPolicy.plan_device, env.act_, Agent.push)
static int replay_collect_step(b200rl_replay* r, uint64_t* rng, const b200rl_explorer* ex) {
    b200rl_ctx* ctx = r->ctx;
    b200rl_net* n = r->net;
    const float* obs;
    TRY(learner_obs(r->env, &obs));
    void* s;
    TRY(ctx_scratch(ctx, (size_t)r->N * n->actor.nout * 4 + 256, &s));
    if (ex) {
        TRY(nn_q_explore(ctx, n->actor, n->params, obs, r->N, (unsigned long long*)rng, *ex, r->action, (float*)s, r->ex_step_dev));
        add_i64_kernel<<<1, 1, 0, ctx->stream>>>(r->ex_step_dev, (long long)r->N * b200rl_comm_world(ctx));
        LAUNCH_CHECK(ctx);
    } else {
        TRY(nn_q_act(ctx, n->actor, n->params, obs, r->N, nullptr, 0.0f, r->action, (float*)s));
    }
    TRY(b200rl_env_step(r->env, r->action, 1, 1));
    return b200rl_traj_push_env(r->traj, r->env, 0);
}
static int replay_stride(const b200rl_replay* r, int64_t k) {
    const int64_t F = b200rl_traj_internal_ring(r->traj).frames();
    return (int)(2 * k + 1 < F ? 2 * k + 1 : F);
}
// scratch every launch of the loop needs: the update's Q tables and TD errors, the staged collect's Q values
static size_t replay_scratch_bytes(const b200rl_replay* r) {
    const size_t q_bytes = (size_t)r->B * r->net->actor.nout * 4 * 2 + 256;
    const size_t need_upd = q_bytes + (size_t)r->B * 4 + 256, need_q = (size_t)r->N * r->net->actor.nout * 4 + 256;
    return need_upd > need_q ? need_upd : need_q;
}
// (stride, N) touched-leaf keys / vals for collect stretches up to `stride` rows (prioritised ring)
static int replay_grow_keys(b200rl_replay* r, int stride) {
    if (stride <= r->stride_cap) return B200RL_OK;
    CUDA_TRY(cudaStreamSynchronize(r->ctx->stream));
    cudaFree(r->keys); cudaFree(r->vals);
    r->keys = nullptr; r->vals = nullptr; r->stride_cap = 0;
    CUDA_TRY(cudaMalloc(&r->keys, (size_t)stride * r->N * 8));
    CUDA_TRY(cudaMalloc(&r->vals, (size_t)stride * r->N * 4));
    r->stride_cap = stride;
    return B200RL_OK;
}
// k collect steps: one fused launch (H = 64 on the tensor-core path; + one sum-tree rebuild for a prioritised ring), otherwise k x
// the staged launches
static int replay_collect(b200rl_replay* r, uint64_t* rng, const b200rl_explorer* ex, int64_t k) {
    b200rl_ctx* ctx = r->ctx;
    b200rl_net* n = r->net;
    const bool prio = b200rl_traj_internal_prioritized(r->traj);
    const int stride = replay_stride(r, k);
    if (nn_tc_enabled() && (!prio || stride <= r->stride_cap)) {
        int st = nn_tc_replay_collect(ctx, r->env, n->actor, n->params, ex, r->ex_step_dev, (unsigned long long*)rng, b200rl_traj_internal_ring(r->traj),
                                      b200rl_traj_internal_default_priority(r->traj), prio ? 1 : 0, (int)k, r->keys, r->vals, stride);
        if (st == B200RL_OK) {
            if (ex) {
                add_i64_kernel<<<1, 1, 0, ctx->stream>>>(r->ex_step_dev, (long long)r->N * b200rl_comm_world(ctx) * k);
                LAUNCH_CHECK(ctx);
            }
            b200rl_traj_internal_add_pushed(r->traj, k);
            if (prio) TRY(b200rl_traj_internal_tree_rebuild(r->traj, r->keys, r->vals, (int64_t)stride * r->N));
            return B200RL_OK;
        }
        if (st != B200RL_ERR_UNSUPPORTED) return st;
    }
    for (int64_t j = 0; j < k; ++j) TRY(replay_collect_step(r, rng, ex));
    return B200RL_OK;
}
// The values the ranks of a sharded b200rl_replay_run must agree on (DESIGN.md §3): ranks that ran different numbers of updates
// would wait for each other in the gradient exchange for ever.  Each 64-bit value travels as its two 32-bit halves (exact in
// Float64) in the rank's own row of a (world, 2 kAgree) table; one sum all-reduce of the table hands every rank every row.
static uint64_t f64_bits(double d) { uint64_t b; memcpy(&b, &d, 8); return b; }
static int replay_agree(b200rl_replay* r, const b200rl_explorer* ex, const b200rl_insert_sample_ratio* ctl, int64_t n_steps, bool local_ok,
                        bool* agree) {
    b200rl_ctx* ctx = r->ctx;
    const int world = b200rl_comm_world(ctx), rank = b200rl_comm_rank(ctx);
    uint64_t cfg_digest = 1469598103934665603ull;   // FNV-1a of the DQN config's bytes (floats and int32s, no padding)
    const unsigned char* cb = (const unsigned char*)&r->cfg;
    for (size_t j = 0; j < sizeof r->cfg; ++j) cfg_digest = (cfg_digest ^ cb[j]) * 1099511628211ull;
    int ns; float ng;
    b200rl_traj_internal_nstep(r->traj, &ns, &ng);
    const b200rl_explorer e = ex ? *ex : b200rl_explorer{};
    const uint64_t v[kAgree] = {local_ok ? 1ull : 0ull, (uint64_t)r->N, (uint64_t)r->B, (uint64_t)n_steps,
                                f64_bits(ctl->ratio), (uint64_t)ctl->threshold, (uint64_t)ctl->n_inserted, (uint64_t)ctl->n_sampled,
                                ex ? 1ull : 0ull, (uint64_t)e.kind, f64_bits(e.eps_stable), f64_bits(e.eps_init), (uint64_t)e.warmup_steps,
                                (uint64_t)e.decay_steps, (uint64_t)e.step, (uint64_t)e.is_break_tie, f64_bits(e.beta), cfg_digest,
                                (uint64_t)ns, (uint64_t)f64_bits((double)ng), b200rl_env_internal_state_f32(r->env) ? 1ull : 0ull};
    const int W = 2 * kAgree;
    std::vector<double> tab((size_t)world * W, 0.0);
    for (int j = 0; j < kAgree; ++j) {
        tab[(size_t)rank * W + 2 * j] = (double)(uint32_t)(v[j] >> 32);
        tab[(size_t)rank * W + 2 * j + 1] = (double)(uint32_t)v[j];
    }
    CUDA_TRY(cudaMemcpyAsync(r->agree_dev, tab.data(), tab.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    TRY(b200rl_comm_allreduce_internal(ctx, r->agree_dev, (int64_t)tab.size(), 1));
    CUDA_TRY(cudaMemcpyAsync(tab.data(), r->agree_dev, tab.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    *agree = true;
    for (int q = 0; q < world; ++q)
        for (int j = 0; j < W; ++j) *agree = *agree && tab[(size_t)q * W + j] == tab[(size_t)rank * W + j];
    return B200RL_OK;
}
static int replay_unit(b200rl_replay* r, uint64_t* rng, const b200rl_explorer* ex, int64_t m) {
    TRY(replay_collect(r, rng, ex, 1));
    for (int64_t k = 0; k < m; ++k) TRY(dqn_update_seq(r->net, r->traj, &r->cfg, r->upd_dev, r->td_keep, nullptr));
    return B200RL_OK;
}

/* The replay agent's part of run_stretches: b200rl_replay_run per stretch — with a budget chunks of at most stop_chunk steps (the
 * ring then still holds every frame a chunk pushed, which count_ring_kernel reads), without one the whole window.  A rollback
 * restores the host counters b200rl_replay_run advanced: *ex, *ctl, env steps, pushed frames, optimiser steps. */
struct ReplayStretches {
    b200rl_replay* r;
    uint64_t* rng;
    b200rl_explorer* ex;
    b200rl_insert_sample_ratio* ctl;
    struct Saved { b200rl_explorer ex; b200rl_insert_sample_ratio ctl; uint64_t env_steps, net_updates; int64_t pushed; };
    Saved save() const {
        return {ex ? *ex : b200rl_explorer{}, *ctl, b200rl_env_internal_steps(r->env), r->net->n_updates, b200rl_traj_internal_pushed(r->traj)};
    }
    void restore(const Saved& s0) const {
        if (ex) *ex = s0.ex;
        *ctl = s0.ctl;
        b200rl_env_internal_add_steps(r->env, s0.env_steps - b200rl_env_internal_steps(r->env));
        b200rl_traj_internal_add_pushed(r->traj, s0.pushed - b200rl_traj_internal_pushed(r->traj));
        r->net->n_updates = s0.net_updates;
    }
    size_t shadow_bytes() const {
        DevRegion tr[kTrajStateRegionsMax];
        const int nt = b200rl_traj_internal_state_regions(r->traj, tr);
        size_t bytes = b200rl_env_internal_step_bytes_max(r->env) + round256((size_t)r->N * 32) + 4 * round256((size_t)r->net->np * 4) +
                       3 * 256 + round256((size_t)r->B * 4);
        for (int k = 0; k < nt; ++k) bytes += round256(tr[k].bytes);
        return bytes;
    }
    int64_t longest() const { return r->stop_chunk; }
    int mark(Shadow& sh) const {
        b200rl_net* n = r->net;
        DevRegion rg[kEnvStepRegionsMax > kTrajStateRegionsMax ? kEnvStepRegionsMax : kTrajStateRegionsMax];
        TRY(sh.add_regions(rg, b200rl_env_internal_step_regions(r->env, rg)));
        TRY(sh.add_regions(rg, b200rl_traj_internal_state_regions(r->traj, rg)));
        if (ex && rng) TRY(sh.add(rng, (size_t)r->N * 32));
        const size_t pb = (size_t)n->np * 4;
        TRY(sh.add(n->params, pb)); TRY(sh.add(n->m, pb)); TRY(sh.add(n->v, pb)); TRY(sh.add(n->target, pb));
        TRY(sh.add(n->beta_t, 2 * 4)); TRY(sh.add(n->loss4, 4 * 4)); TRY(sh.add(n->gnorm, 4));
        return sh.add(r->td_keep, (size_t)r->B * 4);
    }
    int64_t stretch(int64_t left, bool counting, int64_t) const { return counting && r->stop_chunk < left ? r->stop_chunk : left; }
    int run(int64_t s, bool) const { return b200rl_replay_run(r, rng, ex, ctl, s, nullptr); }
    int count(int64_t s, const Saved&, unsigned long long* counts) const {
        b200rl_ctx* ctx = r->ctx;
        stop::count_ring_kernel<<<grid_for(r->N, stop::kCountBlock), stop::kCountBlock, (size_t)s * sizeof(int), ctx->stream>>>(
            b200rl_traj_internal_ring(r->traj), (int)s, counts);
        LAUNCH_CHECK(ctx);
        return B200RL_OK;
    }
    int end_stretch() const { return B200RL_OK; }
    bool at_boundary(int64_t) const { return false; }
};

extern "C" {

int b200rl_replay_destroy(b200rl_replay* r) {
    if (!r) return B200RL_OK;
    cudaSetDevice(r->ctx->device);
    cudaStreamSynchronize(r->ctx->stream);
    cudaFree(r->action); cudaFree(r->ex_step_dev); cudaFree(r->upd_dev); cudaFree(r->td_keep); cudaFree(r->keys); cudaFree(r->vals);
    cudaFree(r->agree_dev);
    r->stop.release();
    delete r;
    return B200RL_OK;
}

int b200rl_replay_create(b200rl_ctx* ctx, b200rl_net* q, b200rl_env* env, b200rl_traj* traj, const b200rl_dqn_config* cfg, b200rl_replay** out) {
    TRY(ctx_bind(ctx));
    REQUIRE(q && env && traj && cfg && out, B200RL_ERR_INVALID, "null argument");
    REQUIRE(is_q_kind(q->kind), B200RL_ERR_INVALID, "needs a Q-network (kind 2 or 3)");
    REQUIRE(q->ctx == ctx && b200rl_env_internal_ctx(env) == ctx && b200rl_traj_internal_ctx(traj) == ctx, B200RL_ERR_INVALID,
            "net/env/trajectory belong to another ctx");
    const float* obs;
    TRY(learner_obs(env, &obs));
    REQUIRE(b200rl_env_internal_kind(env) != B200RL_ENV_ACROBOT, B200RL_ERR_UNSUPPORTED, "AcrobotEnv has 6 observations (networks take at most 4)");
    REQUIRE(!b200rl_env_internal_continuous(env), B200RL_ERR_UNSUPPORTED, "QBasedPolicy needs a discrete action space");
    REQUIRE(b200rl_env_internal_nobs(env) == q->actor.in, B200RL_ERR_INVALID, "network input width != observation width");
    REQUIRE(q->actor.nout == b200rl_env_internal_n_actions(env), B200RL_ERR_INVALID, "Q head width != number of discrete actions");
    const int64_t N = b200rl_env_internal_n(env);
    REQUIRE(b200rl_traj_internal_lanes(traj) == N, B200RL_ERR_INVALID, "trajectory lanes != number of envs");
    TrajBatchView b = b200rl_traj_internal_batch(traj);
    REQUIRE(b.B > 0, B200RL_ERR_INVALID, "the trajectory was created without a sampler (batch_size = 0)");
    REQUIRE(b.ns == q->actor.in, B200RL_ERR_INVALID, "trajectory state width != network input width");
    const int world = b200rl_comm_world(ctx);
    P2PTable peers;
    REQUIRE(world == 1 || b200rl_comm_p2p_table(ctx, &peers) || b200rl_comm_has_nccl(ctx), B200RL_ERR_UNSUPPORTED,
            "a sharded ctx needs the peer exchange attached or an NCCL communicator");
    TRY(check_nstep_gamma(traj, cfg));
    b200rl_replay* r = new b200rl_replay();   // (value-initialised: every pointer and counter starts at zero)
    r->ctx = ctx; r->net = q; r->env = env; r->traj = traj; r->cfg = *cfg; r->N = N; r->B = b.B;
#define R_TRY(x) CUDA_TRY_OR(x, b200rl_replay_destroy(r))
    R_TRY(cudaMalloc(&r->action, (size_t)N * 4));
    R_TRY(cudaMalloc(&r->ex_step_dev, sizeof(long long)));
    R_TRY(cudaMalloc(&r->upd_dev, sizeof(unsigned long long)));
    R_TRY(cudaMalloc(&r->td_keep, (size_t)b.B * 4));
    if (world > 1) R_TRY(cudaMalloc(&r->agree_dev, (size_t)world * 2 * kAgree * sizeof(double)));
    {   // StopAfterNEpisodes (b200rl_replay_run_episodes): the chunk length; its buffers are allocated by the first run with a budget
        const int64_t cap = b200rl_traj_internal_ring(traj).cap;
        r->stop_chunk = cap / 2 < kStopChunkMax ? cap / 2 : kStopChunkMax;
    }
#undef R_TRY
    if (world > 1) {
        // A sharded run allocates nothing: a device allocation serialises with the kernels running on the device, and the ranks of
        // one process may share it — a rank allocating while a peer rank's kernel waits for it inside the exchange would never
        // finish.  So the loop's scratch and the touched-leaf lists of the longest possible stretch are allocated here.
        void* sc;
        int st = ctx_scratch(ctx, replay_scratch_bytes(r), &sc);
        if (st == B200RL_OK && b200rl_traj_internal_prioritized(traj)) st = replay_grow_keys(r, (int)b200rl_traj_internal_ring(traj).frames());
        if (st != B200RL_OK) { b200rl_replay_destroy(r); return st; }
    }
    *out = r;
    return B200RL_OK;
}

int b200rl_replay_run(b200rl_replay* r, uint64_t* explorer_rng_dev, b200rl_explorer* ex, b200rl_insert_sample_ratio* ctl, int64_t n_steps, float* stats4) {
    REQUIRE(r && ctl, B200RL_ERR_INVALID, "null argument");
    const int world = b200rl_comm_world(r->ctx);
    const int64_t NW = r->N * world;   // columns of one plan! over the ranks' union (DESIGN.md §3)
    auto local_checks = [&]() -> int {
        REQUIRE(n_steps >= 0, B200RL_ERR_INVALID, "n_steps must be >= 0");
        if (ex) {
            REQUIRE(explorer_rng_dev, B200RL_ERR_INVALID, "an explorer other than GreedyExplorer needs the (4, N) device explorer streams");
            TRY(check_explorer(ex));
            REQUIRE(n_steps <= ((1ll << 62) - (ex->step > 0 ? ex->step : 0)) / NW, B200RL_ERR_INVALID, "explorer step would overflow");
        }
        REQUIRE(replay::controller_ok(*ctl), B200RL_ERR_INVALID, "bad controller values (ratio finite in [0, 1e6], counters >= 0)");
        REQUIRE(ctl->n_inserted + n_steps < (1ll << 52), B200RL_ERR_INVALID, "controller counters too large");
        const float* obs;
        TRY(learner_obs(r->env, &obs));   // (the wrapper may have been removed since create)
        return check_nstep_gamma(r->traj, &r->cfg);
    };
    const int local = local_checks();
    TRY(ctx_bind(r->ctx));
    b200rl_ctx* ctx = r->ctx;
    b200rl_net* n = r->net;
    if (world > 1) {   // every rank takes part in the exchange, a rank that refuses too, so that no rank waits for it
        bool agree = false;
        TRY(replay_agree(r, ex, ctl, n_steps, local == B200RL_OK, &agree));
        if (local != B200RL_OK) return local;
        REQUIRE(agree, B200RL_ERR_INVALID,
                "the ranks of a sharded run disagree on N, batch size, n_steps, controller, explorer, DQN config, n-step setting or the "
                "StateTransformedEnv(env, Float32) wrapper "
                "(or another rank refused the run)");
    }
    if (local != B200RL_OK) return local;
    if (n_steps == 0) return B200RL_OK;
    // every scratch user of the loop at its final size now, so that no captured launch sees the buffer move
    void* sc;
    TRY(ctx_scratch(ctx, replay_scratch_bytes(r), &sc));
    // the schedule of the window: m updates after each step; stretches of steps without an update become one collect launch
    b200rl_insert_sample_ratio c = *ctl;
    std::vector<int64_t> ms((size_t)n_steps);
    int64_t longest = 1, run = 0;
    for (int64_t j = 0; j < n_steps; ++j) {
        ms[(size_t)j] = replay::insert_then_sample(c);
        run = ms[(size_t)j] == 0 ? run + 1 : 0;
        if (run > longest) longest = run;
    }
    if (b200rl_traj_internal_prioritized(r->traj)) TRY(replay_grow_keys(r, replay_stride(r, longest)));   // touched-leaf lists of a window
    ReplayKey key;
    memset(&key, 0, sizeof key);
    key.tc = nn_tc_enabled() ? 1 : 0;
    key.max_timeout = b200rl_env_internal_max_timeout(r->env);
    key.greedy = ex ? 0 : 1;
    key.state_f32 = b200rl_env_internal_state_f32(r->env) ? 1 : 0;
    b200rl_traj_internal_nstep(r->traj, &key.nstep_n, &key.nstep_gamma);
    if (ex) { key.ex = *ex; key.ex.step = 0; }
    key.rng = explorer_rng_dev;
    key.scratch = ctx->scratch;
    key.keys = r->keys;
    b200rl_env_internal_log_key(r->env, key.log);
    r->graphs.rekey(&key, sizeof key);
    // device copies of the counters the launches read
    r->h_counters[0] = ex ? (long long)ex->step : 0;
    r->h_counters[1] = (long long)n->n_updates;
    CUDA_TRY(cudaMemcpyAsync(r->ex_step_dev, &r->h_counters[0], sizeof(long long), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(r->upd_dev, &r->h_counters[1], sizeof(long long), cudaMemcpyHostToDevice, ctx->stream));
    const CounterSet counters{ctx, n, r->env, r->traj, nullptr};
    // Captured when every rank owns its device.  Eager launches otherwise: NCCL collectives (no peer exchange) are not captured, and
    // where ranks share a device, instantiating or uploading a graph may wait for the device's running kernels — one of them a peer's
    // exchange waiting for this rank.
    P2PTable peers;
    const bool capturable = world == 1 || (b200rl_comm_p2p_table(ctx, &peers) && peers.exclusive);
    bool updated = false;
    for (int64_t j = 0; j < n_steps;) {
        const int64_t m = ms[(size_t)j];
        if (m == 0) {   // a stretch of steps without an update: one collect window
            int64_t k = 1;
            while (j + k < n_steps && ms[(size_t)(j + k)] == 0) ++k;
            TRY(replay_collect(r, explorer_rng_dev, ex, k));
            j += k;
            continue;
        }
        ++j;
        updated = true;
        TRY(r->graphs.run(m, counters, capturable, [&] { return replay_unit(r, explorer_rng_dev, ex, m); }));
    }
    *ctl = c;
    if (ex) ex->step += n_steps * NW;
    if (stats4 && updated) TRY(dqn_stats(n, r->td_keep, r->B, stats4));
    return B200RL_OK;
}

/* run(agent, env, StopAfterNSteps | StopAfterNEpisodes(k)) for at most max_steps env steps (include/b200rl.h): run_stretches */
int b200rl_replay_run_episodes(b200rl_replay* r, uint64_t* explorer_rng_dev, b200rl_explorer* ex, b200rl_insert_sample_ratio* ctl,
                               int64_t max_steps, int64_t budget, float* stats4, int64_t* steps_done, int64_t* episodes_done) {
    REQUIRE(r && ctl && steps_done && episodes_done && max_steps >= 1, B200RL_ERR_INVALID, "bad argument");
    REQUIRE(budget < 0 || b200rl_comm_world(r->ctx) == 1, B200RL_ERR_UNSUPPORTED,
            "StopAfterNEpisodes counts the episodes of every rank: a sharded ctx keeps the stage loop");
    TRY(ctx_bind(r->ctx));
    const uint64_t updates0 = r->net->n_updates;
    ReplayStretches ops{r, explorer_rng_dev, ex, ctl};
    TRY(run_stretches(r->ctx, r->stop, r->N, ops, max_steps, budget, steps_done, episodes_done));
    if (stats4 && r->net->n_updates != updates0) TRY(dqn_stats(r->net, r->td_keep, r->B, stats4));
    return B200RL_OK;
}

int b200rl_replay_graph_active(b200rl_replay* r, int* out) {
    REQUIRE(r && out, B200RL_ERR_INVALID, "null argument");
    *out = r->graphs.active() ? 1 : 0;
    return B200RL_OK;
}

}  // extern "C"
