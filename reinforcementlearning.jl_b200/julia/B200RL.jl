# B200RL.jl — the Julia side of the drop-in: new `AbstractEnv` / `AbstractPolicy` subtypes whose
# methods `ccall` libb200rl.so (include/b200rl.h).  Pure ccall: no CUDA.jl, no codegen.
#
# STATUS: written against ReinforcementLearning.jl v0.11 (RLBase 0.13.1 / RLCore 0.15.4) but NOT
# executed — the build image has no `julia` binary (DESIGN.md §1).  The Python mirror in this
# package drives the identical C ABI and is what the tests and bench exercise.
#
# Usage (what replaces `MultiThreadEnv([CartPoleEnv(T=Float32, rng=...) for i in 1:N])` + PPOPolicy):
#
#   using ReinforcementLearning, Random
#   include("B200RL.jl"); using .B200RL
#   ctx  = B200Context(0)
#   env  = B200VecEnv(ctx, :CartPole, 65_536; seeds = [Xoshiro(hash(123 + i)) for i in 1:65_536], auto_reset = true)
#   net  = B200Network(ctx, n_in = 4, hidden = 64, n_out = 2, params = Flux.destructure(model)[1])
#   agent = B200OnPolicyAgent(ctx, net, env; update_freq = 32, n_epochs = 4, n_microbatches = 4,
#                             policy_seeds = [Xoshiro(hash(7 + i)) for i in 1:65_536])
#   run(agent, env, StopAfterNSteps(10_000), BatchStepsPerEpisode(65_536))
module B200RL

using Random
using TimerOutputs: @timeit_debug             # the reference's debug tracing (RLCore/src/core/run.jl:46-72); enable with
                                              # TimerOutputs.enable_debug_timings(B200RL); labels land in RLCore.timer
import ReinforcementLearningBase as RLBase
import ReinforcementLearningCore as RLCore
import ReinforcementLearningEnvironments as RLEnvs
using ReinforcementLearningBase: AbstractEnv, AbstractPolicy, Observation, DefaultPlayer, (..), ×   # `..` / `×`: DomainSets, re-exported by RLBase (space.jl:6)
using ReinforcementLearningCore: AbstractStage, PreExperimentStage, PostExperimentStage, PreActStage, PostActStage,
    AbstractStopCondition, AbstractHook, AbstractResetCondition, ResetIfEnvTerminated, StopAfterNEpisodes, StopAfterNSteps,
    EpsilonGreedyExplorer, GreedyExplorer, AbstractExplorer, WeightedSoftmaxExplorer, GumbelSoftmaxExplorer

export B200Context, B200VecEnv, B200Network, B200OnPolicyAgent, B200RandomPolicy, B200Trajectory, B200DQNLearner, B200QBasedPolicy,
    B200Agent, B200EpisodeStats, B200EpisodeLog, InsertSampleRatio, B200GreedyPolicy, evaluate, replay!, set_nstep!

const LIB = get(ENV, "B200RL_LIB", joinpath(@__DIR__, "..", "libb200rl.so"))

# ---- error convention: every entry point returns 0 or a negative status ---------------------
function check(status::Cint)
    status == 0 && return nothing
    msg = unsafe_string(ccall((:b200rl_last_error, LIB), Cstring, ()))
    error("b200rl status $status: $msg")
end

mutable struct B200Context
    h::Ptr{Cvoid}
    function B200Context(device::Integer = 0)
        out = Ref{Ptr{Cvoid}}(C_NULL)
        check(ccall((:b200rl_init, LIB), Cint, (Cint, Ref{Ptr{Cvoid}}), device, out))
        ctx = new(out[])
        finalizer(c -> (c.h == C_NULL || ccall((:b200rl_destroy, LIB), Cvoid, (Ptr{Cvoid},), c.h); c.h = C_NULL), ctx)
    end
end
sync(ctx::B200Context) = check(ccall((:b200rl_sync, LIB), Cint, (Ptr{Cvoid},), ctx.h))

# raw Xoshiro256++ state of a Julia `Xoshiro` (fields s0..s3) -> (4, N) UInt64
raw_states(rngs::AbstractVector{Xoshiro}) = reduce(hcat, [UInt64[r.s0, r.s1, r.s2, r.s3] for r in rngs])

# ---- params structs: pass the FINAL field values of the reference's own constructors ----------
struct CartPoleParamsC
    gravity::Cdouble; masscart::Cdouble; masspole::Cdouble; totalmass::Cdouble; halflength::Cdouble
    polemasslength::Cdouble; forcemag::Cdouble; dt::Cdouble; thetathreshold::Cdouble; xthreshold::Cdouble
    max_steps::Int64
end
struct PendulumParamsC
    max_speed::Cdouble; max_torque::Cdouble; g::Cdouble; m::Cdouble; l::Cdouble; dt::Cdouble
    max_steps::Int64; n_actions::Int64; continuous::Int32
end
struct MountainCarParamsC
    min_pos::Cdouble; max_pos::Cdouble; max_speed::Cdouble; goal_pos::Cdouble; goal_velocity::Cdouble; power::Cdouble; gravity::Cdouble
    max_steps::Int64
end
# built from RLEnvs' own params structs so the reference constructors stay the source of truth (their fields are already rounded to T;
# Float64 embeds Float32 exactly):  B200VecEnv(ctx, :CartPole, N; params = CartPoleParamsC(RLEnvs.CartPoleEnvParams{Float32}(; max_steps = 500)), ...)
CartPoleParamsC(p::RLEnvs.CartPoleEnvParams) = CartPoleParamsC(p.gravity, p.masscart, p.masspole, p.totalmass, p.halflength, p.polemasslength,
                                                                p.forcemag, p.dt, p.thetathreshold, p.xthreshold, p.max_steps)
PendulumParamsC(p::RLEnvs.PendulumEnvParams; n_actions::Integer = 3, continuous::Bool = true) =
    PendulumParamsC(p.max_speed, p.max_torque, p.g, p.m, p.l, p.dt, p.max_steps, n_actions, continuous)
MountainCarParamsC(p::RLEnvs.MountainCarEnvParams) =
    MountainCarParamsC(p.min_pos, p.max_pos, p.max_speed, p.goal_pos, p.goal_velocity, p.power, p.gravity, p.max_steps)
struct AcrobotParamsC   # b200rl_acrobot_params
    link_length_a::Cdouble; link_length_b::Cdouble; link_mass_a::Cdouble; link_mass_b::Cdouble; link_com_pos_a::Cdouble; link_com_pos_b::Cdouble
    link_moi::Cdouble; max_torque_noise::Cdouble; max_vel_a::Cdouble; max_vel_b::Cdouble; g::Cdouble; dt::Cdouble
    max_steps::Int64; book::Int32
end
AcrobotParamsC(p::RLEnvs.AcrobotEnvParams; book_or_nips::AbstractString = "book") =
    AcrobotParamsC(p.link_length_a, p.link_length_b, p.link_mass_a, p.link_mass_b, p.link_com_pos_a, p.link_com_pos_b, p.link_moi, p.max_torque_noise,
                   p.max_vel_a, p.max_vel_b, p.g, p.dt, p.max_steps, book_or_nips == "book" ? 1 : 0)

# 3 / 4: CartPoleEnv(continuous = true) / ContinuousMountainCarEnv (CartPoleEnv.jl:74-79, MountainCarEnv.jl:83), Float32 actions in -1.0..1.0
# 5: AcrobotEnv{Float64} (3rd_party/AcrobotEnv.jl): pass T = Float64; one classical RK4 step per act! (DESIGN.md §7)
const KINDS = Dict(:CartPole => 0, :Pendulum => 1, :MountainCar => 2, :ContinuousCartPole => 3, :ContinuousMountainCar => 4, :Acrobot => 5)
const NS = Dict(0 => 4, 1 => 2, 2 => 2, 3 => 4, 4 => 2, 5 => 4)
const NOBS = Dict(0 => 4, 1 => 3, 2 => 2, 3 => 4, 4 => 2, 5 => 6)
@enum Field STATE = 0 OBS = 1 REWARD = 2 TERMINAL = 3 TSTEP = 4 RNG = 5 FLAGS = 6 ACTION = 7 OBS_F32 = 10

"""
    B200VecEnv(ctx, kind, N; T = Float32, seeds, auto_reset = true, params = nothing)

N classic-control envs stepped by one kernel launch.  Plays the role of `MultiThreadEnv`:
`state(env)` is `(NOBS, N)`, `reward(env)` / `is_terminated(env)` are length-N vectors.
"""
mutable struct B200VecEnv{T} <: AbstractEnv
    ctx::B200Context
    h::Ptr{Cvoid}
    kind::Int
    n::Int
    auto_reset::Bool
    continuous::Bool
    n_actions::Int         # discrete spaces: Base.OneTo(n_actions)
    # host mirrors, refreshed lazily (state(env) may alias a reused buffer: interface.jl:515-517)
    obs::Matrix{T}
    rewards::Vector{T}
    terminals::Vector{UInt8}
    state_f32::Bool        # StateTransformedEnv(env, Float32): state(env) is the Float32 mirror
    obs32::Matrix{Float32}
end

function B200VecEnv(ctx::B200Context, kind::Symbol, n::Integer; T = Float32, seeds::AbstractVector{Xoshiro},
                    auto_reset::Bool = true, params = nothing, continuous::Bool = (kind in (:Pendulum, :ContinuousCartPole, :ContinuousMountainCar)),
                    n_actions::Integer = kind in (:MountainCar, :Pendulum, :Acrobot) ? 3 : 2)
    length(seeds) == n || throw(ArgumentError("need one Xoshiro per env"))
    k = KINDS[kind]
    st = raw_states(seeds)
    out = Ref{Ptr{Cvoid}}(C_NULL)
    # `params`: `nothing` (the reference constructors' defaults) or one of the *ParamsC structs above (an isbits struct, passed by reference)
    pref = params === nothing ? nothing : Ref(params)
    pptr = pref === nothing ? C_NULL : Base.unsafe_convert(Ptr{Cvoid}, pref)
    GC.@preserve st pref check(ccall((:b200rl_env_create, LIB), Cint,
        (Ptr{Cvoid}, Cint, Cint, Int64, Ptr{Cvoid}, Ptr{UInt64}, Ref{Ptr{Cvoid}}),
        ctx.h, k, T === Float64 ? 1 : 0, n, pptr, st, out))
    env = B200VecEnv{T}(ctx, out[], k, n, auto_reset, continuous, n_actions, zeros(T, NOBS[k], n), zeros(T, n), zeros(UInt8, n),
                          false, zeros(Float32, NOBS[k], n))
    finalizer(e -> (e.h == C_NULL || ccall((:b200rl_env_destroy, LIB), Cint, (Ptr{Cvoid},), e.h); e.h = C_NULL), env)
end

"""
    MaxTimeoutEnv(env::B200VecEnv, max_t)

The reference wrapper (wrappers/MaxTimeoutEnv.jl:17-28) as a flag on the batched env: `is_terminated` also fires once an
episode has taken `max_t` interactions; `reward` still forwards to the wrapped env.  Returns `env`.
"""
function RLEnvs.MaxTimeoutEnv(env::B200VecEnv, max_t::Integer)
    check(ccall((:b200rl_env_set_max_timeout, LIB), Cint, (Ptr{Cvoid}, Int64), env.h, max_t))
    env
end

"""
    StateTransformedEnv(env::B200VecEnv, Float32)

`StateTransformedEnv(env; state_mapping = s -> Float32.(s))` (wrappers/StateTransformedEnv.jl:15-19) as a flag on a Float64 batched
env: `state(env)` is the Float32 observation mirror (the round to nearest of the Float64 observation), which the learners,
trajectories and the policies' `plan!` read; the dynamics stay the Float64 env's.  Returns `env`.
"""
function RLEnvs.StateTransformedEnv(env::B200VecEnv, ::Type{Float32})
    check(ccall((:b200rl_env_set_state_f32, LIB), Cint, (Ptr{Cvoid}, Cint), env.h, 1))
    env.state_f32 = true
    env
end

function fetch!(env::B200VecEnv, field::Field, dst::Array)
    GC.@preserve dst check(ccall((:b200rl_env_get, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{Cvoid}, Csize_t),
                                 env.h, Int(field), dst, sizeof(dst)))
    dst
end

# ---- RLBase verbs (interface.jl:435-597) -------------------------------------------------------
RLBase.reset!(env::B200VecEnv; is_force::Bool = true) =
    check(ccall((:b200rl_env_reset, LIB), Cint, (Ptr{Cvoid}, Cint), env.h, is_force))

function RLBase.act!(env::B200VecEnv, actions::AbstractVector{<:Integer})
    a = convert(Vector{Int32}, actions)                     # device dtype is Int32, 1-based like Base.OneTo(n)
    GC.@preserve a check(ccall((:b200rl_env_step, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Cint), env.h, a, 0, env.auto_reset))
end
function RLBase.act!(env::B200VecEnv{T}, actions::AbstractVector{<:AbstractFloat}) where {T}
    a = convert(Vector{T}, actions)                         # a continuous action is a T (Float64 for the constructors' default T)
    GC.@preserve a check(ccall((:b200rl_env_step, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Cint), env.h, a, 0, env.auto_reset))
end
struct FusedRandomAction end                                  # plan!(B200RandomPolicy) token
RLBase.act!(env::B200VecEnv, ::FusedRandomAction) =
    check(ccall((:b200rl_env_step_random, LIB), Cint, (Ptr{Cvoid}, Cint), env.h, env.auto_reset))

RLBase.state(env::B200VecEnv, ::Observation, ::DefaultPlayer) = RLBase.state(env)
RLBase.state(env::B200VecEnv) = env.state_f32 ? fetch!(env, OBS_F32, env.obs32) : fetch!(env, OBS, env.obs)
RLBase.reward(env::B200VecEnv) = fetch!(env, REWARD, env.rewards)
RLBase.is_terminated(env::B200VecEnv) = (fetch!(env, TERMINAL, env.terminals); env.terminals .!= 0)
# CartPoleEnv.jl:95-96, PendulumEnv.jl:73-74, MountainCarEnv.jl:85-86 (one sub-env's space; every sub-env has the same)
RLBase.action_space(env::B200VecEnv) =
    !env.continuous ? Base.OneTo(env.n_actions) : env.kind == 1 ? (-2.0 .. 2.0) : (-1.0 .. 1.0)
# CartPoleEnv.jl:88-93, PendulumEnv.jl:75-79, MountainCarEnv.jl:87-90 with the default parameters (one sub-env's space)
function RLBase.state_space(env::B200VecEnv{T}) where {T}
    if env.kind == 0 || env.kind == 3
        xt, tt = T(2.4), T(12 * π / 180)
        ((-2 * xt) .. (2 * xt)) × (typemin(T) .. typemax(T)) × ((-2 * tt) .. (2 * tt)) × (typemin(T) .. typemax(T))
    elseif env.kind == 1
        (-1.0 .. 1.0) × (-1.0 .. 1.0) × (-T(8) .. T(8))
    else
        (T(-1.2) .. T(0.6)) × (-T(0.07) .. T(0.07))
    end
end
Base.length(env::B200VecEnv) = env.n
function Random.seed!(env::B200VecEnv, seeds::AbstractVector{Xoshiro})
    st = raw_states(seeds)
    GC.@preserve st check(ccall((:b200rl_env_seed, LIB), Cint, (Ptr{Cvoid}, Ptr{UInt64}), env.h, st))
end
function Base.copy(env::B200VecEnv{T}) where {T}
    out = Ref{Ptr{Cvoid}}(C_NULL)
    check(ccall((:b200rl_env_copy, LIB), Cint, (Ptr{Cvoid}, Ref{Ptr{Cvoid}}), env.h, out))
    e = B200VecEnv{T}(env.ctx, out[], env.kind, env.n, env.auto_reset, env.continuous, env.n_actions, copy(env.obs), copy(env.rewards), copy(env.terminals),
                          env.state_f32, copy(env.obs32))
    finalizer(x -> (x.h == C_NULL || ccall((:b200rl_env_destroy, LIB), Cint, (Ptr{Cvoid},), x.h); x.h = C_NULL), e)
end
"Zero-copy device pointer of an env field for fused consumers (b200rl_env_ptr)."
function device_ptr(env::B200VecEnv, field::Field)
    out = Ref{Ptr{Cvoid}}(C_NULL)
    check(ccall((:b200rl_env_ptr, LIB), Cint, (Ptr{Cvoid}, Cint, Ref{Ptr{Cvoid}}), env.h, Int(field), out))
    out[]
end
struct DeviceActions; ptr::Ptr{Cvoid}; end                   # plan! token: the actions already sit in device memory
RLBase.act!(env::B200VecEnv, a::DeviceActions) =
    check(ccall((:b200rl_env_step, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint, Cint), env.h, a.ptr, 1, env.auto_reset))

"""
    B200EpisodeStats()

Device-side reduction of `TotalRewardPerEpisode` / `BatchStepsPerEpisode` (hooks.jl:146-231): the step kernel accumulates
finished episodes, their returns and lengths; the hook reads four numbers at the end of the experiment — no per-step copy.
`hook[]` = (episodes, return_sum, length_sum, env_steps).
"""
mutable struct B200EpisodeStats <: AbstractHook
    stats::NTuple{4,Float64}
    B200EpisodeStats() = new((0.0, 0.0, 0.0, 0.0))
end
Base.getindex(h::B200EpisodeStats) = h.stats
function episode_stats(env::B200VecEnv; reset::Bool = false)
    out = zeros(Float64, 4)
    GC.@preserve out check(ccall((:b200rl_env_episode_stats, LIB), Cint, (Ptr{Cvoid}, Ptr{Float64}, Cint), env.h, out, reset))
    (out[1], out[2], out[3], out[4])
end
Base.push!(h::B200EpisodeStats, ::PreExperimentStage, ::AbstractPolicy, env::B200VecEnv) = (episode_stats(env; reset = true); nothing)
Base.push!(h::B200EpisodeStats, ::PostExperimentStage, ::AbstractPolicy, env::B200VecEnv) = (h.stats = episode_stats(env); nothing)

"""
    B200EpisodeLog(batchsize; capacity = 64)

`TotalRewardPerEpisode` + `BatchStepsPerEpisode` (hooks.jl:146-231) kept on the device (b200rl_env_episode_log): `rewards` and
`steps` are per-env vectors, filled from a ring of `capacity` records per env without a host copy per step.  `_run` splits its
fused loops into windows of at most `capacity` env steps and flushes after each; the stage loop flushes every `capacity`
`PostActStage` pushes.  A flush is read one flush later (or at `PostExperimentStage`).  Returns are the env's Float32 step-order
sums; `evaluate` is not logged; on a sharded ctx the records carry `rank * N + i` and the vectors are indexed by the local env.
`hook[]` = (rewards, steps).
"""
mutable struct B200EpisodeLog <: AbstractHook
    rewards::Vector{Vector{Float32}}
    steps::Vector{Vector{Int}}
    capacity::Int
    env::Union{Nothing,B200VecEnv}
    bufs::Vector{Ptr{Cvoid}}     # two pinned buffers of 16 + 16 * N * capacity bytes
    next::Int
    pending::Int                 # buffer whose flush is not read yet (0: none)
    acts::Int
    base::Int                    # rank * N
    B200EpisodeLog(batchsize::Integer; capacity::Integer = 64) =
        new([Float32[] for _ in 1:batchsize], [Int[] for _ in 1:batchsize], capacity, nothing, Ptr{Cvoid}[], 1, 0, 0, 0)
end
Base.getindex(h::B200EpisodeLog) = (h.rewards, h.steps)
log_records(h::B200EpisodeLog) = h.env.n * h.capacity
function log_detach!(h::B200EpisodeLog)
    h.env === nothing && return
    check(ccall((:b200rl_env_episode_log, LIB), Cint, (Ptr{Cvoid}, Int32), h.env.h, 0))
    foreach(b -> check(ccall((:b200rl_host_free, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), h.env.ctx.h, b)), h.bufs)
    h.env, h.bufs = nothing, Ptr{Cvoid}[]
end
function log_read!(h::B200EpisodeLog)
    h.pending == 0 && return
    buf, n = h.bufs[h.pending], Ref{Int64}(0)
    h.pending = 0
    check(ccall((:b200rl_env_episode_log_read, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ref{Int64}), h.env.h, buf, n))
    for k in 0:n[]-1                                      # b200rl_episode_record: int64 env, float32 ret, int32 len
        rec = buf + 16 + 16k
        i = unsafe_load(Ptr{Int64}(rec)) - h.base + 1
        push!(h.rewards[i], unsafe_load(Ptr{Float32}(rec + 8)))
        push!(h.steps[i], Int(unsafe_load(Ptr{Int32}(rec + 12))))
    end
end
function log_flush!(h::B200EpisodeLog)
    h.env === nothing && return
    check(ccall((:b200rl_env_episode_log_flush, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Int64), h.env.h, h.bufs[h.next], log_records(h)))
    log_read!(h)
    h.pending, h.next, h.acts = h.next, 3 - h.next, 0
end
function Base.push!(h::B200EpisodeLog, ::PreExperimentStage, ::AbstractPolicy, env::B200VecEnv)
    log_detach!(h)
    check(ccall((:b200rl_env_episode_log, LIB), Cint, (Ptr{Cvoid}, Int32), env.h, h.capacity))
    h.env = env
    rank, world = Ref{Cint}(0), Ref{Cint}(1)
    check(ccall((:b200rl_comm_rank_world, LIB), Cint, (Ptr{Cvoid}, Ref{Cint}, Ref{Cint}), env.ctx.h, rank, world))
    h.base = rank[] * env.n
    h.bufs = map(1:2) do _
        p = Ref{Ptr{Cvoid}}(C_NULL)
        check(ccall((:b200rl_host_alloc, LIB), Cint, (Ptr{Cvoid}, Csize_t, Ref{Ptr{Cvoid}}), env.ctx.h, 16 + 16 * log_records(h), p))
        p[]
    end
    h.next, h.pending, h.acts = 1, 0, 0
    nothing
end
function Base.push!(h::B200EpisodeLog, ::PostActStage, ::AbstractPolicy, ::B200VecEnv)
    h.acts += 1
    h.acts >= h.capacity && log_flush!(h)
    nothing
end
Base.push!(h::B200EpisodeLog, ::PostExperimentStage, ::AbstractPolicy, ::B200VecEnv) = (log_flush!(h); log_read!(h); log_detach!(h); nothing)

# ---- run-loop impedance (SURVEY §7 "Run-loop impedance") --------------------------------------
# the kernel resets finished sub-envs itself; the scalar reset condition must never fire
RLCore.check!(::ResetIfEnvTerminated, ::AbstractPolicy, ::B200VecEnv) = false
# StopAfterNEpisodes counts every finished sub-episode (stop_conditions.jl:104-118 for a vector env)
function RLCore.check!(s::StopAfterNEpisodes{Nothing}, agent, env::B200VecEnv)
    s.cur += count(RLBase.is_terminated(env))
    s.cur >= s.episode
end
function RLCore.check!(s::StopAfterNEpisodes, agent, env::B200VecEnv)     # is_show_progress = true (the default)
    n = count(RLBase.is_terminated(env))
    s.cur += n
    n > 0 && RLCore.ProgressMeter.update!(s.progress, min(s.cur, s.episode))
    s.cur >= s.episode
end
# the historical MultiThreadEnv `_run` (no episode stages), run.jl:36-78 specialised on the env type
function RLCore._run(policy::AbstractPolicy, env::B200VecEnv, stop_condition::AbstractStopCondition, hook::AbstractHook,
                     reset_condition::AbstractResetCondition)
    push!(hook, PreExperimentStage(), policy, env)
    push!(policy, PreExperimentStage(), env)
    RLBase.reset!(env; is_force = true)
    push!(policy, PreEpisodeStage(), env)                      # run.jl:47-49: every lane starts an episode
    # Fused path (the Python mirror's run(), core.py): a device-resident agent, a hook with nothing to do per step and a stop
    # condition that counts steps or episodes let whole stretches of the loop run on the device, with the stage loop's results.
    # Windows of at most a B200EpisodeLog's capacity, each one library call (episodes!) followed by a flush of the log; the library
    # cuts a window into stretches.  A StopAfterNEpisodes window stops at the crossing of the remaining budget (an episode count on
    # a sharded ctx keeps the stage loop), a StopAfterNSteps one (budget -1) may end early at the end of a rollout.  A policy that
    # does not train (B200GreedyPolicy, a B200QBasedPolicy on its own) runs on the fused evaluation kernel (b200rl_eval_run_episodes).
    window = hook isa B200EpisodeLog ? hook.capacity : typemax(Int)
    if hook isa Union{B200EpisodeStats,B200EpisodeLog,RLCore.EmptyHook} && reset_condition isa ResetIfEnvTerminated && env.auto_reset &&
       (stop_condition isa StopAfterNSteps || (stop_condition isa StopAfterNEpisodes && ctx_world(env) == 1)) &&
       ((policy isa B200OnPolicyAgent && policy.fused) || (policy isa B200Agent && replay!(policy, env, 0)) ||
        (policy isa Union{B200GreedyPolicy,B200QBasedPolicy} && eval_fusable(policy, env)))
        while true
            if stop_condition isa StopAfterNSteps                  # check! is true once cur >= step, then cur += 1
                steps, _ = episodes!(policy, env, min(window, max(1, stop_condition.step - stop_condition.cur + 1)), -1)
                stop_condition.cur += steps
                done, progress = stop_condition.cur > stop_condition.step, min(stop_condition.cur, stop_condition.step)
            else
                _, n = episodes!(policy, env, window, max(0, stop_condition.episode - stop_condition.cur))   # (0: one step)
                stop_condition.cur += n
                done, progress = stop_condition.cur >= stop_condition.episode, min(stop_condition.cur, stop_condition.episode)
            end
            hook isa B200EpisodeLog && log_flush!(hook)
            stop_condition.progress === nothing || RLCore.ProgressMeter.update!(stop_condition.progress, progress)
            done && break
        end
        push!(policy, PostExperimentStage(), env)
        push!(hook, PostExperimentStage(), policy, env)
        check(ccall((:b200rl_env_check, LIB), Cint, (Ptr{Cvoid},), env.h))
        return hook
    end
    timer = RLCore.timer                                       # same labels as run.jl:46-72
    while true
        did_reset = false
        while RLCore.check!(reset_condition, policy, env)      # ResetAfterNSteps: the whole batch is force-reset (ResetIfEnvTerminated never fires)
            @timeit_debug timer "reset!"                        RLBase.reset!(env; is_force = true)
            @timeit_debug timer "push!(policy) PreEpisodeStage" push!(policy, PreEpisodeStage(), env)
            did_reset = true
        end
        (did_reset || env.auto_reset) || @timeit_debug timer "reset!" RLBase.reset!(env; is_force = false)
        @timeit_debug timer "push!(policy) PreActStage"         push!(policy, PreActStage(), env)
        @timeit_debug timer "optimise! PreActStage"             RLBase.optimise!(policy, PreActStage())
        @timeit_debug timer "push!(hook) PreActStage"           push!(hook, PreActStage(), policy, env)
        action = @timeit_debug timer "plan!"                    RLBase.plan!(policy, env)
        @timeit_debug timer "act!"                              RLBase.act!(env, action)
        @timeit_debug timer "push!(policy) PostActStage"        push!(policy, PostActStage(), env, action)
        @timeit_debug timer "optimise! PostActStage"            RLBase.optimise!(policy, PostActStage())
        @timeit_debug timer "push!(hook) PostActStage"          push!(hook, PostActStage(), policy, env)
        RLCore.check!(stop_condition, policy, env) && break
    end
    push!(policy, PostExperimentStage(), env)
    push!(hook, PostExperimentStage(), policy, env)
    check(ccall((:b200rl_env_check, LIB), Cint, (Ptr{Cvoid},), env.h))   # the reference's `@assert a in action_space(env)`
    hook
end

# ---- policies ---------------------------------------------------------------------------------
"RandomPolicy() sharing each env's RNG stream (random_policy.jl:18-32): the draw is fused into the step kernel."
struct B200RandomPolicy <: AbstractPolicy end
RLBase.plan!(::B200RandomPolicy, ::B200VecEnv) = FusedRandomAction()

struct NetDescC
    n_in::Int32; hidden::Int32; act::Int32; n_out::Int32; kind::Int32
end
mutable struct B200Network
    ctx::B200Context
    h::Ptr{Cvoid}
    desc::NetDescC
end
"""FluxApproximator stand-in: `params` is `Flux.destructure(ActorCritic(actor, critic))[1]` (Float32).
`kind`: `:categorical`, `:gaussian`, `:q` (a Q-network) or `:dueling` (`DuelingNetwork(base = Chain(Dense(n_in, hidden, act),
Dense(hidden, hidden, act)), val = Dense(hidden, 1), adv = Dense(hidden, n_out))`, networks.jl:500-522; `n_out` = number of
actions, 1..3; `params = Flux.destructure(model)[1]` as it is).  `:q` and `:dueling` carry a target network."""
function B200Network(ctx::B200Context; n_in, hidden, n_out, params::Vector{Float32}, act::Symbol = :relu, kind::Symbol = :categorical)
    k = kind === :categorical ? 0 : kind === :gaussian ? 1 : kind === :dueling ? 3 : 2
    d = NetDescC(n_in, hidden, act === :relu ? 0 : 1, n_out, k)
    out = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve params check(ccall((:b200rl_net_create, LIB), Cint, (Ptr{Cvoid}, Ref{NetDescC}, Ptr{Float32}, Ref{Ptr{Cvoid}}),
                                    ctx.h, Ref(d), params, out))
    net = B200Network(ctx, out[], d)
    finalizer(n -> (n.h == C_NULL || ccall((:b200rl_net_destroy, LIB), Cint, (Ptr{Cvoid},), n.h); n.h = C_NULL), net)
end
"Read back parameters / optimiser state (JLD2 checkpoint hooks, docs/src/How_to_use_hooks.md:124-167)."
function Base.getindex(net::B200Network, which::Integer, n::Integer)
    out = Vector{Float32}(undef, n)
    GC.@preserve out check(ccall((:b200rl_net_get, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{Float32}, Int64), net.h, which, out, n))
    out
end

"Import parameters / optimiser state (`which`: 0 params | 2 Adam m | 3 Adam v | 4 beta^t (2) | 5 target params)."
function Base.setindex!(net::B200Network, v::Vector{Float32}, which::Integer)
    GC.@preserve v check(ccall((:b200rl_net_set, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{Float32}, Int64), net.h, which, v, length(v)))
    v
end
"optimise!(::TargetNetwork): target = ρ * target + (1 - ρ) * model (target_network.jl:70-88); ρ = 0 is the hard copy."
target_sync!(net::B200Network, ρ::Real = 0f0) = check(ccall((:b200rl_net_target_sync, LIB), Cint, (Ptr{Cvoid}, Cfloat), net.h, ρ))

struct OnPolicyConfigC
    gamma::Cfloat; lambda::Cfloat; clip_range::Cfloat; max_grad_norm::Cfloat; w_actor::Cfloat; w_critic::Cfloat; w_entropy::Cfloat
    lr::Cfloat; beta1::Cfloat; beta2::Cfloat; eps::Cfloat; min_sigma::Cfloat; max_sigma::Cfloat
    normalize_advantage::Int32; n_epochs::Int32; n_microbatches::Int32; update_freq::Int32; algo::Int32
end

"Agent(policy = PPOPolicy | A2C, trajectory = PPOTrajectory) living on the device."
mutable struct B200OnPolicyAgent <: AbstractPolicy
    ctx::B200Context
    h::Ptr{Cvoid}
    net::B200Network
    env::B200VecEnv
    T::Int
    t::Int
    fused::Bool            # true: actions never visit the host (plan! returns a device token, run() may fuse whole stretches)
    actions::Vector{Int32}
    stats::Matrix{Float32}
end
function B200OnPolicyAgent(ctx, net::B200Network, env::B200VecEnv; policy_seeds::AbstractVector{Xoshiro}, fused::Bool = false,
        γ = 0.99f0, λ = 0.95f0, clip_range = 0.1f0, max_grad_norm = 0.5f0, actor_loss_weight = 1f0, critic_loss_weight = 0.5f0,
        entropy_loss_weight = 0.001f0, lr = 1f-3, update_freq = 32, n_epochs = 4, n_microbatches = 4, normalize_advantage = true,
        algo::Symbol = :ppo)
    cfg = OnPolicyConfigC(γ, λ, clip_range, max_grad_norm, actor_loss_weight, critic_loss_weight, entropy_loss_weight, lr, 0.9f0, 0.999f0,
                          1f-8, 0f0, Inf32, normalize_advantage, n_epochs, n_microbatches, update_freq, algo === :ppo ? 0 : 1)
    st = raw_states(policy_seeds)
    out = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve st check(ccall((:b200rl_onpolicy_create, LIB), Cint,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{OnPolicyConfigC}, Ptr{UInt64}, Ref{Ptr{Cvoid}}), ctx.h, net.h, env.h, Ref(cfg), st, out))
    a = B200OnPolicyAgent(ctx, out[], net, env, update_freq, 0, fused, zeros(Int32, env.n), zeros(Float32, 6, n_epochs * n_microbatches))
    finalizer(x -> (x.h == C_NULL || ccall((:b200rl_onpolicy_destroy, LIB), Cint, (Ptr{Cvoid},), x.h); x.h = C_NULL), a)
end
# plan!(agent, env) (agent_base.jl:52-54): K6 on the current observation; actions come back to the host
struct FusedPolicyAction; agent::Ptr{Cvoid}; end              # plan!(fused agent) token: act! without leaving the device
RLBase.act!(::B200VecEnv, f::FusedPolicyAction) = check(ccall((:b200rl_onpolicy_act, LIB), Cint, (Ptr{Cvoid},), f.agent))
function RLBase.plan!(a::B200OnPolicyAgent, ::B200VecEnv)
    if a.fused
        check(ccall((:b200rl_onpolicy_plan, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), a.h, C_NULL))
        return FusedPolicyAction(a.h)
    end
    GC.@preserve a check(ccall((:b200rl_onpolicy_plan, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), a.h, a.actions))
    a.actions
end
"n_steps x {plan!, act!, push!} in one kernel launch (fused rollout)."
function collect!(a::B200OnPolicyAgent, n_steps::Integer)
    check(ccall((:b200rl_onpolicy_collect, LIB), Cint, (Ptr{Cvoid}, Cint), a.h, n_steps))
    a.t += n_steps
end
# push!(agent, PostActStage, env, action) (agent_base.jl:56-59): reward/terminal were written in-kernel
function Base.push!(a::B200OnPolicyAgent, ::PostActStage, ::B200VecEnv, action)
    check(ccall((:b200rl_onpolicy_push, LIB), Cint, (Ptr{Cvoid},), a.h))
    a.t += 1
end
Base.push!(::B200OnPolicyAgent, ::AbstractStage, ::B200VecEnv) = nothing
# optimise!(agent, PostActStage) (agent_base.jl:34-41): GAE + n_epochs x n_microbatches updates once the rollout is full
function RLBase.optimise!(a::B200OnPolicyAgent, ::PostActStage)
    a.t == a.T || return nothing
    GC.@preserve a check(ccall((:b200rl_onpolicy_update, LIB), Cint, (Ptr{Cvoid}, Ptr{Int32}, Ptr{Float32}), a.h, C_NULL, a.stats))
    a.t = 0
    nothing
end
RLBase.optimise!(::B200OnPolicyAgent, ::AbstractStage) = nothing

# ---- checkpoint / resume (the JLD2 hook pattern, docs/src/How_to_use_hooks.md:124-167) ---------------
# `DoEveryNSteps(n = 10_000) do t, agent, env; JLD2.jldsave("ckpt_$t.jld2"; B200RL.checkpoint(agent)...) end`
const ENV_FIELDS = (state = 0, obs = 1, reward = 2, flags = 6, t = 4, rng = 5, action = 7, episode_return = 8, episode_stats = 9)
function env_field_array(env::B200VecEnv{T}, name::Symbol) where {T}
    n = env.n
    name === :state ? Matrix{T}(undef, NS[env.kind], n) : name === :obs ? Matrix{T}(undef, NOBS[env.kind], n) :
    name === :reward ? Vector{T}(undef, n) : name === :flags ? Vector{UInt8}(undef, n) : name === :t ? Vector{Int32}(undef, n) :
    name === :rng ? Matrix{UInt64}(undef, 4, n) : name === :action ? (env.continuous ? Vector{Float32}(undef, n) : Vector{Int32}(undef, n)) :
    name === :episode_return ? Vector{Float32}(undef, n) : Vector{Float64}(undef, 4)
end
"Copy the whole device state of an on-policy run out: NamedTuple of plain arrays (`JLD2.jldsave(path; ckpt...)`)."
function checkpoint(a::B200OnPolicyAgent)
    env, net = a.env, a.net
    envs = map(keys(ENV_FIELDS)) do name
        dst = env_field_array(env, name)
        GC.@preserve dst check(ccall((:b200rl_env_get, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{Cvoid}, Csize_t), env.h, ENV_FIELDS[name], dst, sizeof(dst)))
        dst
    end
    np = Ref{Int64}(0)
    check(ccall((:b200rl_net_nparams, LIB), Cint, (Ref{NetDescC}, Ref{Int64}), Ref(net.desc), np))
    counters = zeros(Int64, 3)
    GC.@preserve counters check(ccall((:b200rl_onpolicy_export_state, LIB), Cint, (Ptr{Cvoid}, Ptr{Int64}), a.h, counters))
    rng = Matrix{UInt64}(undef, 4, env.n)
    GC.@preserve rng check(ccall((:b200rl_onpolicy_get, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{Cvoid}, Csize_t), a.h, 8, rng, sizeof(rng)))
    # in the middle of a rollout (counters[1] = t > 0; e.g. DoEveryNSteps(n = 10_000) with update_freq = 32) the columns 0..t-1 of the
    # rollout tensors are part of the state: fields 0-5 of b200rl_onpolicy_get (state, action, logp, reward, terminal, value)
    rollout = counters[1] == 0 ? nothing : map(0:5) do f
        dst = rollout_field_array(a, f)
        GC.@preserve dst check(ccall((:b200rl_onpolicy_get, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{Cvoid}, Csize_t), a.h, f, dst, sizeof(dst)))
        dst
    end
    (env = NamedTuple{keys(ENV_FIELDS)}(envs), params = net[0, np[]], adam_m = net[2, np[]], adam_v = net[3, np[]], beta_t = net[4, 2],
     counters = counters, policy_rng = rng, rollout = rollout)
end
"Host array shaped like rollout field `f` of `b200rl_onpolicy_get` (0 state (ns, N, T+1) | 1 action | 2 logp | 3 reward | 4 terminal | 5 value (N, T+1))."
function rollout_field_array(a::B200OnPolicyAgent, f::Integer)
    n, T, ns = a.env.n, a.T, NOBS[a.env.kind]
    f == 0 ? Array{Float32}(undef, ns, n, T + 1) : f == 1 ? (a.env.continuous ? Matrix{Float32}(undef, n, T) : Matrix{Int32}(undef, n, T)) :
    f == 4 ? Matrix{UInt8}(undef, n, T) : f == 5 ? Matrix{Float32}(undef, n, T + 1) : Matrix{Float32}(undef, n, T)
end
"Put a `checkpoint` back into a freshly constructed agent (same env kind / N, same network shape, same hyper-parameters)."
function restore!(a::B200OnPolicyAgent, ck)
    for name in keys(ENV_FIELDS)
        name === :obs && a.env.kind != 1 && continue            # the observation is the state (one buffer) except for Pendulum
        src = getfield(ck.env, name)
        GC.@preserve src check(ccall((:b200rl_env_set, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{Cvoid}, Csize_t), a.env.h, ENV_FIELDS[name], src, sizeof(src)))
    end
    a.net[0] = ck.params; a.net[2] = ck.adam_m; a.net[3] = ck.adam_v; a.net[4] = ck.beta_t
    rng, counters = ck.policy_rng, ck.counters
    GC.@preserve rng check(ccall((:b200rl_onpolicy_set, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{Cvoid}, Csize_t), a.h, 8, rng, sizeof(rng)))
    if counters[1] > 0    # mid-rollout checkpoint: the first t columns must come back, or the next update would read uninitialised memory
        hasproperty(ck, :rollout) && ck.rollout !== nothing ||
            error("B200RL.restore!: the checkpoint was taken at rollout step t = $(counters[1]) but holds no rollout columns")
        for (f, src) in zip(0:5, ck.rollout)
            GC.@preserve src check(ccall((:b200rl_onpolicy_set, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{Cvoid}, Csize_t), a.h, f, src, sizeof(src)))
        end
    end
    GC.@preserve counters check(ccall((:b200rl_onpolicy_import_state, LIB), Cint, (Ptr{Cvoid}, Ptr{Int64}), a.h, counters))
    a.t = Int(counters[1])
    a
end

# ---- DQN: device trajectory + learner + explorer (BASELINE config 5) --------------------------------
# InsertSampleRatioController(ratio, threshold) (RLTrajectories 0.4; docs/src/How_to_implement_a_new_algorithm.md:108); one insertion = one frame
Base.@kwdef mutable struct InsertSampleRatio
    ratio::Float64 = 1.0
    threshold::Int = 1
    n_inserted::Int = 0
    n_sampled::Int = 0
end
function on_sample!(c::InsertSampleRatio)
    if c.n_inserted >= c.threshold && c.n_sampled <= (c.n_inserted - c.threshold) * c.ratio
        c.n_sampled += 1
        return true
    end
    false
end
"""
    B200Trajectory(ctx; state_size, lanes, capacity, batch_size, sampler_seeds, prioritized = false, default_priority = 1f0,
                   controller = InsertSampleRatio(), n_step = 1, γ = 0.99f0)

`Trajectory(container = CircularArraySARTSTraces(capacity) [wrapped in CircularPrioritizedTraces], sampler = BatchSampler(batch_size)
| NStepBatchSampler(n_step, γ, batch_size), controller = InsertSampleRatioController(ratio, threshold))` (ReinforcementLearningTrajectories
0.4) resident on the device: a ring of `capacity + 1` frames of `lanes` sub-envs; `next_state` of frame j is frame j + 1.  With
`n_step > 1` a sampled entry's reward / terminal / next_state come from its n-step window, `discount = γ^m` and `horizon = m` say how
long it was (DESIGN.md §3), and the learner's γ must be the same.
"""
mutable struct B200Trajectory
    ctx::B200Context
    h::Ptr{Cvoid}
    lanes::Int
    batch_size::Int
    controller::InsertSampleRatio
    state_size::Int
    n_step::Int
    γ::Float32
end
function B200Trajectory(ctx::B200Context; state_size::Integer, lanes::Integer, capacity::Integer, batch_size::Integer,
                        sampler_seeds::AbstractVector{Xoshiro}, prioritized::Bool = false, default_priority = 1f0,
                        controller = InsertSampleRatio(), n_step::Integer = 1, γ = 0.99f0)
    length(sampler_seeds) == batch_size || throw(ArgumentError("need one Xoshiro per batch slot"))
    st = raw_states(sampler_seeds)
    out = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve st check(ccall((:b200rl_traj_create, LIB), Cint,
        (Ptr{Cvoid}, Cint, Int64, Int64, Cint, Cfloat, Ptr{UInt64}, Int64, Ref{Ptr{Cvoid}}),
        ctx.h, state_size, lanes, capacity, prioritized, default_priority, st, batch_size, out))
    t = B200Trajectory(ctx, out[], lanes, batch_size, controller, state_size, 1, 0.99f0)
    finalizer(x -> (x.h == C_NULL || ccall((:b200rl_traj_destroy, LIB), Cint, (Ptr{Cvoid},), x.h); x.h = C_NULL), t)
    n_step == 1 || set_nstep!(t, n_step, γ)
    t
end
"`NStepBatchSampler(n, γ)` from the next sample on (`n = 1`: the BatchSampler); refused unless 1 ≤ n ≤ min(32, capacity), γ ∈ [0, 1]."
function set_nstep!(t::B200Trajectory, n::Integer, γ)
    check(ccall((:b200rl_traj_set_nstep, LIB), Cint, (Ptr{Cvoid}, Int32, Cfloat), t.h, n, γ))
    t.n_step, t.γ = Int(n), Float32(γ)
    t
end
"The last sampled batch: `(state, action, reward, terminal, next_state, key, priority, weight, discount, horizon)`."
function batch(t::B200Trajectory)
    B, ns = t.batch_size, t.state_size
    field!(f, a) = (GC.@preserve a check(ccall((:b200rl_traj_batch_get, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{Cvoid}, Csize_t),
                                                t.h, f, a, sizeof(a))); a)
    (state = field!(0, Matrix{Float32}(undef, ns, B)), action = field!(1, Vector{Int32}(undef, B)), reward = field!(2, Vector{Float32}(undef, B)),
     terminal = field!(3, Vector{UInt8}(undef, B)) .!= 0, next_state = field!(4, Matrix{Float32}(undef, ns, B)), key = field!(5, Vector{Int64}(undef, B)),
     priority = field!(6, Vector{Float32}(undef, B)), weight = field!(7, Vector{Float32}(undef, B)), discount = field!(9, Vector{Float32}(undef, B)),
     horizon = field!(10, Vector{Int32}(undef, B)))
end
function Base.length(t::B200Trajectory)
    n = Ref{Int64}(0)
    check(ccall((:b200rl_traj_length, LIB), Cint, (Ptr{Cvoid}, Ref{Int64}), t.h, n))
    Int(n[])
end
# push!(trajectory, (state = s0,)) / push!(trajectory, (state = s', action, reward, terminal)) reading the env's device fields
# mode 0: the transition; 1: episode-start frame for every lane; 2: episode-start frame for the lanes whose last transition was terminal
push_env!(t::B200Trajectory, env::B200VecEnv; mode::Integer = 0) =
    check(ccall((:b200rl_traj_push_env, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Cint), t.h, env.h, mode))
"`length(container)` per lane (== steps + episodes - 1, RLCore/test/core/base.jl:20)"
function lane_lengths(t::B200Trajectory)
    out = Vector{Int64}(undef, t.lanes)
    GC.@preserve out check(ccall((:b200rl_traj_lane_lengths, LIB), Cint, (Ptr{Cvoid}, Ptr{Int64}), t.h, out))
    out
end

struct DQNConfigC
    gamma::Cfloat; lr::Cfloat; beta1::Cfloat; beta2::Cfloat; eps::Cfloat; max_grad_norm::Cfloat; rho::Cfloat
    per_alpha::Cfloat; per_beta::Cfloat; per_eps::Cfloat
    huber::Int32; double_dqn::Int32; target_update_freq::Int32
end
"DQNLearner / PrioritizedDQNLearner: `net` is a `kind = :q` or `kind = :dueling` B200Network (FluxApproximator + TargetNetwork, target_network.jl:27-88)."
struct B200DQNLearner <: RLCore.AbstractLearner
    net::B200Network
    cfg::DQNConfigC
end
B200DQNLearner(net::B200Network; γ = 0.99f0, lr = 1f-3, max_grad_norm = 0f0, ρ = 0f0, per_α = 0.6f0, per_β = 0.4f0, per_ϵ = 1f-6,
               huber::Bool = true, double_dqn::Bool = false, target_update_freq::Integer = 100) =
    B200DQNLearner(net, DQNConfigC(γ, lr, 0.9f0, 0.999f0, 1f-8, max_grad_norm, ρ, per_α, per_β, per_ϵ, huber, double_dqn, target_update_freq))
# optimise!(learner, batch): sample + gather, TD loss + backward, clip + Adam, priority write-back, target sync — all on the device
update!(l::B200DQNLearner, t::B200Trajectory) =
    check(ccall((:b200rl_dqn_update, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ref{DQNConfigC}, Ptr{Cfloat}), l.net.h, t.h, Ref(l.cfg), C_NULL))

struct ExplorerC
    eps_stable::Cdouble; eps_init::Cdouble; warmup_steps::Int64; decay_steps::Int64; step::Int64; kind::Int32; is_break_tie::Int32
    beta::Cdouble
end
ExplorerC(s::EpsilonGreedyExplorer{K,B}) where {K,B} =
    ExplorerC(s.ϵ_stable, s.ϵ_init, s.warmup_steps, s.decay_steps, s.step, K === :linear ? 0 : 1, B ? 1 : 0, 0.0)
ExplorerC(::WeightedSoftmaxExplorer) = ExplorerC(0.0, 0.0, 0, 0, 0, 3, 0, 0.0)
ExplorerC(::GumbelSoftmaxExplorer) = ExplorerC(0.0, 0.0, 0, 0, 0, 4, 0, 0.0)
# ReinforcementLearningFarm's EpsilonSpeedyExplorer(β) (its step is a Ref), matched by name so that this package does not depend
# on ReinforcementLearningFarm
is_speedy(s) = nameof(typeof(s)) === :EpsilonSpeedyExplorer
function ExplorerC(s::AbstractExplorer)
    is_speedy(s) || throw(ArgumentError("$(typeof(s)) has no device explorer"))
    ExplorerC(0.0, 0.0, 0, 0, s.step[], 2, 0, s.β)
end
# the explorers b200rl_net_q_explore / b200rl_replay_run plan with (GreedyExplorer: b200rl_net_q_act / a NULL explorer)
device_explorer(s) = s isa Union{EpsilonGreedyExplorer,WeightedSoftmaxExplorer,GumbelSoftmaxExplorer} || is_speedy(s)
# advance the inner explorer's step to where the device call left it (the softmax explorers have no step)
set_step!(s::EpsilonGreedyExplorer, step) = (s.step = step; nothing)
set_step!(s::Union{WeightedSoftmaxExplorer,GumbelSoftmaxExplorer}, step) = nothing
set_step!(s::AbstractExplorer, step) = (s.step[] = step; nothing)      # EpsilonSpeedyExplorer

"""
    B200QBasedPolicy(ctx, learner, explorer, n; explorer_seeds)

`QBasedPolicy(learner, explorer)` (q_based_policy.jl:13-49) for a batched env.  `explorer` is the reference's own
`EpsilonGreedyExplorer{kind, is_break_tie}`, `WeightedSoftmaxExplorer()`, `GumbelSoftmaxExplorer()`, ReinforcementLearningFarm's
`EpsilonSpeedyExplorer(β)` or `GreedyExplorer()`: its fields are read on every `plan!` and its step (if it has one) is advanced
by `n`, the way `BatchExplorer` calls the inner explorer once per column (batch_explorer.jl:15-21); the forward pass, the
per-column schedule, the draws and the selection run in one device call.  On a sharded ctx (rank r of G, `comm_rank_world`) the
`n` envs are global envs r n + 1 … (r + 1) n: the columns are numbered over all ranks and `plan!`, `replay!` and `evaluate` advance
the step by G n per plan, as one `BatchExplorer` over the G n envs would.
"""
mutable struct B200QBasedPolicy{E<:AbstractExplorer} <: AbstractPolicy
    ctx::B200Context
    learner::B200DQNLearner
    explorer::E
    n::Int
    d_rng::Ptr{Cvoid}
    d_action::Ptr{Cvoid}
end
function dmalloc(ctx::B200Context, bytes::Integer)
    out = Ref{Ptr{Cvoid}}(C_NULL)
    check(ccall((:b200rl_malloc, LIB), Cint, (Ptr{Cvoid}, Csize_t, Ref{Ptr{Cvoid}}), ctx.h, bytes, out))
    out[]
end
function B200QBasedPolicy(ctx::B200Context, learner::B200DQNLearner, explorer::AbstractExplorer, n::Integer; explorer_seeds::AbstractVector{Xoshiro})
    length(explorer_seeds) == n || throw(ArgumentError("need one Xoshiro per env"))
    st = raw_states(explorer_seeds)
    d_rng, d_action = dmalloc(ctx, 32n), dmalloc(ctx, 4n)
    GC.@preserve st check(ccall((:b200rl_memcpy_h2d, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Cint), ctx.h, d_rng, st, 32n, 0))
    p = B200QBasedPolicy(ctx, learner, explorer, Int(n), d_rng, d_action)
    finalizer(p) do x
        x.ctx.h == C_NULL && return
        ccall((:b200rl_free, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), x.ctx.h, x.d_rng)
        ccall((:b200rl_free, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), x.ctx.h, x.d_action)
    end
end
"""`(rank, world)` of the ctx's communicator; `(0, 1)` without one (b200rl_comm_rank_world)."""
function comm_rank_world(ctx::B200Context)
    r, w = Ref{Cint}(0), Ref{Cint}(1)
    check(ccall((:b200rl_comm_rank_world, LIB), Cint, (Ptr{Cvoid}, Ref{Cint}, Ref{Cint}), ctx.h, r, w))
    (Int(r[]), Int(w[]))
end
function RLBase.plan!(p::B200QBasedPolicy, env::B200VecEnv)
    ex = ExplorerC(p.explorer)
    check(ccall((:b200rl_net_q_explore, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Ptr{Cvoid}, Ref{ExplorerC}, Ptr{Cvoid}),
                p.learner.net.h, device_ptr(env, OBS_F32), p.n, p.d_rng, Ref(ex), p.d_action))
    set_step!(p.explorer, ex.step + p.n * comm_rank_world(p.ctx)[2])   # BatchExplorer over every rank's columns (DESIGN.md §3)
    DeviceActions(p.d_action)
end
function RLBase.plan!(p::B200QBasedPolicy{GreedyExplorer}, env::B200VecEnv)
    check(ccall((:b200rl_net_q_act, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Ptr{Cvoid}, Cfloat, Ptr{Cvoid}),
                p.learner.net.h, device_ptr(env, OBS_F32), p.n, C_NULL, 0f0, p.d_action))
    DeviceActions(p.d_action)
end

# ---- evaluation -------------------------------------------------------------------------------
"""
    B200GreedyPolicy(net::B200Network, n)

The network's greedy policy on a batch of `n` envs with a discrete action space: `findmax` of the logits / Q-values
(`GreedyExplorer`, explorers/epsilon_greedy_explorer.jl:196-204; no RNG).  `plan!` leaves the actions on the device
(`DeviceActions`), so `run(B200GreedyPolicy(net, n), env, StopAfterNSteps(k), hook)` never copies an action to the host.
For a Gaussian policy use [`evaluate`](@ref), which hands `clamp(μ, lo, hi)` to the env inside the kernel.
"""
mutable struct B200GreedyPolicy <: AbstractPolicy
    net::B200Network
    n::Int
    d_action::Ptr{Cvoid}
end
function B200GreedyPolicy(net::B200Network, n::Integer)
    p = B200GreedyPolicy(net, Int(n), dmalloc(net.ctx, 4n))
    finalizer(x -> (x.net.ctx.h == C_NULL || ccall((:b200rl_free, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), x.net.ctx.h, x.d_action)), p)
end
function RLBase.plan!(p::B200GreedyPolicy, env::B200VecEnv)
    env.continuous && throw(ArgumentError("B200GreedyPolicy plans discrete actions; evaluate a Gaussian policy with `evaluate`"))
    check(ccall((:b200rl_net_act_greedy, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Int64, Ptr{Cvoid}, Cint),
                p.net.h, device_ptr(env, OBS_F32), p.n, p.d_action, 1))
    DeviceActions(p.d_action)
end

struct EvalConfigC
    mode::Int32; n_steps::Int32; max_episodes::Int32
end
"""
    evaluate(net, env; n_steps, max_episodes = 1, mode = :greedy, policy_seeds = nothing)

`run(policy, env, StopAfterNSteps(n_steps))` with the network's greedy (`:greedy`) or sampling (`:sample`, one policy stream per
env from `policy_seeds`) policy, as one fused kernel launch where the network allows it (b200rl_evaluate): every env is reset
first, finished envs auto-reset.  Returns `(; returns, lengths, counts)`: the first `max_episodes` episodes of each env that
end inside the window (`max_episodes × n` matrices; NaN / -1 where no episode ended) and the number of episodes per env.
Average over the envs with `counts .>= max_episodes` to avoid the bias towards short episodes of a fixed window.  The env's
episode statistics advance as under `run`; the network is only read.
"""
function evaluate(net::B200Network, env::B200VecEnv; n_steps::Integer, max_episodes::Integer = 1, mode::Symbol = :greedy,
                  policy_seeds::Union{Nothing,AbstractVector{Xoshiro}} = nothing)
    m = mode === :greedy ? 0 : mode === :sample ? 1 : throw(ArgumentError("mode must be :greedy or :sample"))
    n = env.n
    returns = fill(NaN32, max_episodes, n)
    lengths = fill(Int32(-1), max_episodes, n)
    counts = zeros(Int32, n)
    d_rng = C_NULL
    if policy_seeds !== nothing
        length(policy_seeds) == n || throw(ArgumentError("need one Xoshiro per env"))
        st = raw_states(policy_seeds)
        d_rng = dmalloc(net.ctx, 32n)
        GC.@preserve st check(ccall((:b200rl_memcpy_h2d, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Cint), net.ctx.h, d_rng, st, 32n, 0))
    end
    try
        GC.@preserve returns lengths counts check(ccall((:b200rl_evaluate, LIB), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Ref{EvalConfigC}, Ptr{Cvoid}, Ptr{Float32}, Ptr{Int32}, Ptr{Int32}, Cint),
            net.h, env.h, Ref(EvalConfigC(m, n_steps, max_episodes)), d_rng, returns, lengths, counts, 0))
    finally
        d_rng == C_NULL || ccall((:b200rl_free, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), net.ctx.h, d_rng)
    end
    (; returns, lengths, counts)
end

"""
    evaluate(p::B200QBasedPolicy, env; n_steps, max_episodes = 1)

`run(p, env, StopAfterNSteps(n_steps))` in actor mode (docs/src/How_to_use_hooks.md:96-119): the Q-network planned by the policy's
explorer on the policy's explorer streams, as one fused kernel launch where the network allows it (b200rl_evaluate_explore).  The
same records as `evaluate(net, env; ...)`.  The streams and the explorer's step advance exactly as under `run`; the learner is only
read.  To evaluate without touching a training policy, build a second `B200QBasedPolicy` over the same learner.
"""
function evaluate(p::B200QBasedPolicy, env::B200VecEnv; n_steps::Integer, max_episodes::Integer = 1)
    n = env.n
    returns = fill(NaN32, max_episodes, n)
    lengths = fill(Int32(-1), max_episodes, n)
    counts = zeros(Int32, n)
    if device_explorer(p.explorer)
        ex = Ref(ExplorerC(p.explorer))
        GC.@preserve returns lengths counts check(ccall((:b200rl_evaluate_explore, LIB), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Int32, Ref{ExplorerC}, Ptr{Cvoid}, Ptr{Float32}, Ptr{Int32}, Ptr{Int32}, Cint),
            p.learner.net.h, env.h, n_steps, max_episodes, ex, p.d_rng, returns, lengths, counts, 0))
        set_step!(p.explorer, ex[].step)
    elseif p.explorer isa GreedyExplorer                           # findmax, no draw
        GC.@preserve returns lengths counts check(ccall((:b200rl_evaluate_explore, LIB), Cint,
            (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Float32}, Ptr{Int32}, Ptr{Int32}, Cint),
            p.learner.net.h, env.h, n_steps, max_episodes, C_NULL, p.d_rng, returns, lengths, counts, 0))
    else
        throw(ArgumentError("$(typeof(p.explorer)) has no device explorer"))
    end
    (; returns, lengths, counts)
end

"""
    B200Agent(policy::B200QBasedPolicy, trajectory::B200Trajectory)

`Agent(policy, trajectory)` (agent_base.jl:18-66) with a device-resident replay: transition frames never visit the host.  `_run` announces
every forced reset with a `PreEpisodeStage` push (every lane gets an episode-start frame, so re-entering `run` on a filled trajectory is
fine: the entry straddling the reset is stored and never sampled — EpisodesBuffer's bookkeeping, kept per lane on the device).  Episodes
that end inside the loop start their next frame in the push kernel (in-kernel auto-reset) or at the next `PreActStage` (soft reset).
"""
mutable struct B200Agent <: AbstractPolicy
    policy::B200QBasedPolicy
    trajectory::B200Trajectory
    fused::Bool            # false: `_run` always steps through the stages (the stage protocol)
    replay::Ptr{Cvoid}     # b200rl_replay handle of the device loop (kept across `run` calls: its CUDA graphs stay captured)
    replay_env::Ptr{Cvoid} # the env it was created for
end
function B200Agent(policy::B200QBasedPolicy, trajectory::B200Trajectory)
    a = B200Agent(policy, trajectory, true, C_NULL, C_NULL)
    finalizer(x -> (x.replay == C_NULL || ccall((:b200rl_replay_destroy, LIB), Cint, (Ptr{Cvoid},), x.replay); x.replay = C_NULL), a)
end
RLBase.plan!(a::B200Agent, env::B200VecEnv) = RLBase.plan!(a.policy, env)
Base.push!(a::B200Agent, ::PreEpisodeStage, env::B200VecEnv) = (push_env!(a.trajectory, env; mode = 1); nothing)      # push!(trajectory, (state = s0,)), all lanes
Base.push!(a::B200Agent, ::PreActStage, env::B200VecEnv) = (env.auto_reset || push_env!(a.trajectory, env; mode = 2); nothing)   # lanes soft-reset after their terminal step
function Base.push!(a::B200Agent, ::PostActStage, env::B200VecEnv, action)
    push_env!(a.trajectory, env)
    a.trajectory.controller.n_inserted += 1
    nothing
end
Base.push!(::B200Agent, ::AbstractStage, ::B200VecEnv) = nothing
# optimise!(agent, PostActStage) -> optimise!(policy.learner, stage, trajectory): `for batch in trajectory` samples while the controller allows
function RLBase.optimise!(a::B200Agent, ::PostActStage)
    while on_sample!(a.trajectory.controller)
        update!(a.policy.learner, a.trajectory)
    end
    nothing
end
RLBase.optimise!(::B200Agent, ::AbstractStage) = nothing

struct InsertSampleRatioC
    ratio::Cdouble; threshold::Int64; n_inserted::Int64; n_sampled::Int64
end
"""
    replay!(agent::B200Agent, env, n_steps) -> Bool

`n_steps` × {plan!, act!, push!, optimise!} of the stage protocol on the device (b200rl_replay_run): a stretch of steps without an
update is one collect launch (H = 64 on the tensor cores) and each "1 step + m updates" unit is replayed from a CUDA graph.  The
same transitions, updates, streams and counters as stepping through the stages; the explorer's `step` and the controller's counters
advance.  `false` (nothing done) when the agent / env are outside the device loop: the caller steps through the stages instead.
"""
function replay!(a::B200Agent, env::B200VecEnv, n_steps::Integer)
    p, t, c = a.policy, a.trajectory, a.trajectory.controller
    (a.fused && env isa B200VecEnv{Float32} && env.auto_reset && !env.continuous && t.batch_size > 0 && t.lanes == env.n &&
     (device_explorer(p.explorer) || p.explorer isa GreedyExplorer)) || return false
    if a.replay == C_NULL || a.replay_env != env.h
        a.replay == C_NULL || ccall((:b200rl_replay_destroy, LIB), Cint, (Ptr{Cvoid},), a.replay)
        a.replay = C_NULL
        h = Ref{Ptr{Cvoid}}(C_NULL)
        st = ccall((:b200rl_replay_create, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{DQNConfigC}, Ref{Ptr{Cvoid}}),
                   p.ctx.h, p.learner.net.h, env.h, t.h, Ref(p.learner.cfg), h)
        st in (-1, -3) && return false              # B200RL_ERR_INVALID / _UNSUPPORTED (e.g. a sharded ctx without an exchange): the stage loop runs it
        check(st)
        a.replay, a.replay_env = h[], env.h
    end
    ctl = Ref(InsertSampleRatioC(c.ratio, c.threshold, c.n_inserted, c.n_sampled))
    if device_explorer(p.explorer)
        ex = Ref(ExplorerC(p.explorer))
        check(ccall((:b200rl_replay_run, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ref{ExplorerC}, Ref{InsertSampleRatioC}, Int64, Ptr{Cfloat}),
                    a.replay, p.d_rng, ex, ctl, n_steps, C_NULL))
        set_step!(p.explorer, ex[].step)
    else                                                           # GreedyExplorer: findmax, no draw
        check(ccall((:b200rl_replay_run, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{InsertSampleRatioC}, Int64, Ptr{Cfloat}),
                    a.replay, p.d_rng, C_NULL, ctl, n_steps, C_NULL))
    end
    c.n_inserted, c.n_sampled = Int(ctl[].n_inserted), Int(ctl[].n_sampled)
    true
end

"""
    episodes!(agent, env, max_steps, budget) -> (steps, episodes)

At most `max_steps` env steps of `run(agent, env, stop)` on the device (b200rl_onpolicy_run_episodes / b200rl_replay_run_episodes),
with the stage loop's state.  budget = k - cur for `StopAfterNEpisodes(k)`: the loop stops after the step at which the episodes
counted reach it (refused on a sharded ctx, whose stop would count the episodes of every rank).  budget < 0 for `StopAfterNSteps`:
`max_steps` steps, or fewer when the last rollout they complete ends earlier; no episodes are counted.
"""
function episodes!(a::B200OnPolicyAgent, ::B200VecEnv, max_steps::Integer, budget::Integer)
    steps, eps = Ref{Int64}(0), Ref{Int64}(0)
    GC.@preserve a check(ccall((:b200rl_onpolicy_run_episodes, LIB), Cint, (Ptr{Cvoid}, Int64, Int64, Ptr{Float32}, Ref{Int64}, Ref{Int64}),
                               a.h, max_steps, budget, a.stats, steps, eps))
    t, T = Ref{Cint}(0), Ref{Cint}(0)
    check(ccall((:b200rl_onpolicy_fill, LIB), Cint, (Ptr{Cvoid}, Ref{Cint}, Ref{Cint}), a.h, t, T))
    a.t = Int(t[])                                                  # a stop inside a rollout leaves it part-filled
    steps[], eps[]
end
# The b200rl_eval handle of an evaluation policy for `env` (made on the policy's first fused run on it, destroyed with the policy or
# when it runs on another env); C_NULL where the library refuses the pair (the stage loop then keeps the run).
const EVAL_HANDLES = Dict{UInt,Tuple{Ptr{Cvoid},Ptr{Cvoid}}}()   # objectid(policy) => (env handle, b200rl_eval handle)
function eval_handle!(p, net::B200Network, env::B200VecEnv, mode::Integer)
    id = objectid(p)
    e = get(EVAL_HANDLES, id, nothing)
    e !== nothing && e[1] == env.h && return e[2]
    e === nothing || ccall((:b200rl_eval_destroy, LIB), Cint, (Ptr{Cvoid},), e[2])
    h = Ref{Ptr{Cvoid}}(C_NULL)
    if ccall((:b200rl_eval_create, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Int32, Ref{Ptr{Cvoid}}), net.h, env.h, mode, h) != 0
        delete!(EVAL_HANDLES, id)
        return C_NULL
    end
    e === nothing && finalizer(p) do _
        x = pop!(EVAL_HANDLES, id, nothing)
        x === nothing || net.ctx.h == C_NULL || ccall((:b200rl_eval_destroy, LIB), Cint, (Ptr{Cvoid},), x[2])   # (a closed ctx took its buffers)
    end
    EVAL_HANDLES[id] = (env.h, h[])
    h[]
end
eval_fusable(p::B200GreedyPolicy, env::B200VecEnv) = !env.continuous && eval_handle!(p, p.net, env, 0) != C_NULL
eval_fusable(p::B200QBasedPolicy, env::B200VecEnv) =
    (device_explorer(p.explorer) || p.explorer isa GreedyExplorer) && eval_handle!(p, p.learner.net, env, 2) != C_NULL

# run(policy, env, stop) of a policy that does not train (b200rl_eval_run_episodes, `_run` made the handle): the stage loop's steps,
# episode log, streams and explorer step.  budget < 0: exactly max_steps steps.
function episodes!(p::B200GreedyPolicy, env::B200VecEnv, max_steps::Integer, budget::Integer)
    steps, eps = Ref{Int64}(0), Ref{Int64}(0)
    check(ccall((:b200rl_eval_run_episodes, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Ref{Int64}, Ref{Int64}),
                eval_handle!(p, p.net, env, 0), C_NULL, C_NULL, max_steps, budget, steps, eps))
    steps[], eps[]
end
function episodes!(p::B200QBasedPolicy, env::B200VecEnv, max_steps::Integer, budget::Integer)
    h = eval_handle!(p, p.learner.net, env, 2)
    steps, eps = Ref{Int64}(0), Ref{Int64}(0)
    if device_explorer(p.explorer)
        ex = Ref(ExplorerC(p.explorer))
        check(ccall((:b200rl_eval_run_episodes, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ref{ExplorerC}, Int64, Int64, Ref{Int64}, Ref{Int64}),
                    h, p.d_rng, ex, max_steps, budget, steps, eps))
        set_step!(p.explorer, ex[].step)
    else                                                            # GreedyExplorer: findmax, no draw
        check(ccall((:b200rl_eval_run_episodes, LIB), Cint, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Ref{Int64}, Ref{Int64}),
                    h, C_NULL, C_NULL, max_steps, budget, steps, eps))
    end
    steps[], eps[]
end
function episodes!(a::B200Agent, ::B200VecEnv, max_steps::Integer, budget::Integer)   # (replay!(a, env, 0) made the handle)
    p, c = a.policy, a.trajectory.controller
    ctl = Ref(InsertSampleRatioC(c.ratio, c.threshold, c.n_inserted, c.n_sampled))
    steps, eps = Ref{Int64}(0), Ref{Int64}(0)
    if device_explorer(p.explorer)
        ex = Ref(ExplorerC(p.explorer))
        check(ccall((:b200rl_replay_run_episodes, LIB), Cint,
                    (Ptr{Cvoid}, Ptr{Cvoid}, Ref{ExplorerC}, Ref{InsertSampleRatioC}, Int64, Int64, Ptr{Cfloat}, Ref{Int64}, Ref{Int64}),
                    a.replay, p.d_rng, ex, ctl, max_steps, budget, C_NULL, steps, eps))
        set_step!(p.explorer, ex[].step)
    else                                                            # GreedyExplorer: findmax, no draw
        check(ccall((:b200rl_replay_run_episodes, LIB), Cint,
                    (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{InsertSampleRatioC}, Int64, Int64, Ptr{Cfloat}, Ref{Int64}, Ref{Int64}),
                    a.replay, p.d_rng, C_NULL, ctl, max_steps, budget, C_NULL, steps, eps))
    end
    c.n_inserted, c.n_sampled = Int(ctl[].n_inserted), Int(ctl[].n_sampled)
    steps[], eps[]
end
function ctx_world(env::B200VecEnv)
    rank, world = Ref{Cint}(0), Ref{Cint}(1)
    check(ccall((:b200rl_comm_rank_world, LIB), Cint, (Ptr{Cvoid}, Ref{Cint}, Ref{Cint}), env.ctx.h, rank, world))
    Int(world[])
end

# ---- pure-function drop-ins (utils/basic.jl:138-417) --------------------------------------------
"`generalized_advantage_estimation(rewards, values, γ, λ; dims, terminal)` on the GPU (Float32 / Float64 matrices)."
function generalized_advantage_estimation(ctx::B200Context, rewards::Matrix{T}, values::Matrix{T}, γ::T, λ::T;
                                          dims::Int, terminal::Union{Nothing,Matrix{Bool}} = nothing) where {T<:Union{Float32,Float64}}
    adv = similar(rewards)
    term = terminal === nothing ? C_NULL : convert(Matrix{UInt8}, terminal)
    R, C = size(rewards)
    GC.@preserve adv rewards values term begin
        if T === Float32
            check(ccall((:b200rl_gae_f32, LIB), Cint, (Ptr{Cvoid}, Ptr{T}, Ptr{T}, Ptr{T}, Ptr{UInt8}, T, T, Int64, Int64, Cint, Cint),
                        ctx.h, adv, rewards, values, term, γ, λ, R, C, dims, 0))
        else
            check(ccall((:b200rl_gae_f64, LIB), Cint, (Ptr{Cvoid}, Ptr{T}, Ptr{T}, Ptr{T}, Ptr{UInt8}, T, T, Int64, Int64, Cint, Cint),
                        ctx.h, adv, rewards, values, term, γ, λ, R, C, dims, 0))
        end
    end
    adv
end

"`discount_rewards(rewards, γ; dims, terminal, init)` on the GPU (utils/basic.jl:138-235)."
function discount_rewards(ctx::B200Context, rewards::Matrix{Float32}, γ::Float32; dims::Int, terminal::Union{Nothing,Matrix{Bool}} = nothing,
                          init::Union{Nothing,Vector{Float32}} = nothing)
    out = similar(rewards)
    term = terminal === nothing ? C_NULL : convert(Matrix{UInt8}, terminal)
    ini = init === nothing ? C_NULL : init
    R, C = size(rewards)
    GC.@preserve out rewards term ini check(ccall((:b200rl_discount_rewards_f32, LIB), Cint,
        (Ptr{Cvoid}, Ptr{Float32}, Ptr{Float32}, Ptr{UInt8}, Ptr{Float32}, Float32, Int64, Int64, Cint, Cint),
        ctx.h, out, rewards, term, ini, γ, R, C, dims, 0))
    out
end

# ---- sharded runs: one process per GPU (SURVEY §8e) ------------------------------------------------
"""
    comm_init(ctx, nranks, rank, id128)          # id128 from `comm_unique_id()` on rank 0, shipped by the launcher (MPI, Distributed, a file)
    attach_peer_exchange(ctx, nranks, rank, allgather)

`allgather(bytes::Vector{UInt8})::Vector{Vector{UInt8}}` is any host-side all-gather in rank order; it ships the 64-byte CUDA IPC
handles once.  Afterwards the gradient all-reduce runs inside the optimiser kernel over NVLink peer memory.
"""
function comm_unique_id()
    id = zeros(UInt8, 128)
    GC.@preserve id check(ccall((:b200rl_comm_unique_id, LIB), Cint, (Ptr{UInt8},), id))
    id
end
comm_init(ctx::B200Context, nranks::Integer, rank::Integer, id::Vector{UInt8}) =
    GC.@preserve id check(ccall((:b200rl_comm_init, LIB), Cint, (Ptr{Cvoid}, Cint, Cint, Ptr{UInt8}), ctx.h, nranks, rank, id))
function attach_peer_exchange(ctx::B200Context, nranks::Integer, rank::Integer, allgather)
    handle = zeros(UInt8, 64)
    GC.@preserve handle check(ccall((:b200rl_comm_p2p_export, LIB), Cint, (Ptr{Cvoid}, Ptr{UInt8}, Ptr{Ptr{Cvoid}}), ctx.h, handle, C_NULL))
    handles = allgather(handle)
    regions = fill(C_NULL, nranks)
    for r in 0:nranks-1
        r == rank && continue
        out = Ref{Ptr{Cvoid}}(C_NULL)
        h = handles[r+1]
        GC.@preserve h check(ccall((:b200rl_comm_p2p_open, LIB), Cint, (Ptr{Cvoid}, Ptr{UInt8}, Ref{Ptr{Cvoid}}), ctx.h, h, out))
        regions[r+1] = out[]
    end
    GC.@preserve regions check(ccall((:b200rl_comm_p2p_attach, LIB), Cint, (Ptr{Cvoid}, Ptr{Ptr{Cvoid}}), ctx.h, regions))
    # one rank per physical GPU?  Then the optimiser step (with the gradient exchange) runs in the tail of the loss + backward
    # launch; ranks that share a GPU keep the exchange in its own small kernel (two whole-device kernels cannot be co-resident).
    bus = zeros(UInt8, 32)
    GC.@preserve bus check(ccall((:b200rl_ctx_pci_bus_id, LIB), Cint, (Ptr{Cvoid}, Ptr{UInt8}, Cint), ctx.h, bus, 32))
    ids = allgather(bus)
    check(ccall((:b200rl_comm_p2p_set_exclusive, LIB), Cint, (Ptr{Cvoid}, Cint), ctx.h, length(unique(ids)) == nranks ? 1 : 0))
end
"`set_fused_step(false)` keeps reduce + clip + Adam in a kernel of their own (default: the tail of the loss + backward launch)."
set_fused_step(on::Bool) = check(ccall((:b200rl_set_fused_step, LIB), Cint, (Cint,), on ? 1 : 0))

end # module
