// env_device.cuh — device code of the classic-control envs (state structs, reset!, _step!, observation) and the act! step
// around them, shared by the batched step / reset kernels (env.cu) and the fused rollout, evaluation and DQN collect kernels
// (fwd_tc.cu).  Arithmetic follows the reference line by line with Julia's promotion rules (which sub-expressions are Float64
// for T = Float32) — see DESIGN.md §K1 and
//   RLEnvs/src/environments/examples/CartPoleEnv.jl:98-140, PendulumEnv.jl:84-122, MountainCarEnv.jl:99-135.
// Every translation unit that includes this header MUST be compiled with -fmad=false -prec-div=true -prec-sqrt=true
// -ftz=false (no contraction: Julia never contracts a*b+c); build.py does that for env.cu and fwd_tc.cu.
#pragma once
#include <type_traits>

#include "jl_device.cuh"

namespace envdev {
using jld::Xo;

// b200rl_env_episode_log: a ring of K records per env, (K, N) column-major like the evaluation records, and the number of
// episodes logged so far; count == null: no log.  Record c of env i sits in slot c % K.
struct EpisodeLog {
    float* ret;        // (K, N) the episode's Float32 step-order return (the accumulator of FIELD_EPISODE_RETURN)
    int32_t* len;      // (K, N) env.t at the end of the episode
    uint32_t* count;   // (N)
    int K;
};
__device__ __forceinline__ void log_episode(const EpisodeLog& log, int64_t i, float ret, int len) {
    const uint32_t c = log.count[i];
    const size_t j = (size_t)log.K * (size_t)i + c % (uint32_t)log.K;
    log.ret[j] = ret;
    log.len[j] = len;
    log.count[i] = c + 1;
}

// A flush (env.cu) hands over the records logged since the previous one, env by env in episode order: env i has
// count - cursor of them (the uint32 counters wrap together); more than K means the ring overwrote records nobody read.
struct EpisodeRecord { int64_t env; float ret; int32_t len; };   // b200rl_episode_record
__device__ __forceinline__ uint32_t log_pending(const EpisodeLog& log, const uint32_t* cursor, int64_t i) { return log.count[i] - cursor[i]; }
// env i's n pending records (n <= K) to out[0 .. min(n, room)), tagged with the env's global index
__device__ __forceinline__ void log_emit(const EpisodeLog& log, const uint32_t* cursor, int64_t i, uint32_t n, int64_t global, EpisodeRecord* out,
                                         int64_t room) {
    const uint32_t c0 = cursor[i];
    for (uint32_t e = 0; e < n && (int64_t)e < room; ++e) {
        const size_t j = (size_t)log.K * (size_t)i + (c0 + e) % (uint32_t)log.K;
        out[e] = EpisodeRecord{global, log.ret[j], log.len[j]};
    }
}

struct EnvArrays {
    void* state;      // (NS, N) T
    void* obs;        // (NOBS, N) T   (== state when the observation is the state); a Float64 env's Float32 mirror follows it (obs_f32)
    void* reward;     // (N) T
    uint8_t* flags;   // (N)  bit0 terminal, bit1 already auto-reset
    int32_t* t;       // (N)
    unsigned long long* rng;  // (4, N)
    void* action;     // (N) int32 | T   last action taken
    float* ep_ret;    // (N) running episode return
    double* stats;    // [4] finished episodes, sum return, sum length, env-steps
    int* err;         // device error flag
    // optional fused trajectory push targets (column t of the rollout buffers); may be null
    void* traj_reward;
    uint8_t* traj_terminal;
    int max_timeout;  // MaxTimeoutEnv(env, max_t) (wrappers/MaxTimeoutEnv.jl:17-28); 0 = not wrapped
};
// The kernels that write the episode log take it behind their EnvArrays under a template flag LOG: the instantiations without
// it take EnvArrays alone, the parameters (and so the code) they had before the log existed.
struct EnvArraysLog : EnvArrays {
    EpisodeLog log;
};
template <bool LOG> using EnvArgs = typename std::conditional<LOG, EnvArraysLog, EnvArrays>::type;
__device__ __forceinline__ EpisodeLog episode_log_of(const EnvArrays&) { return EpisodeLog{}; }
__device__ __forceinline__ EpisodeLog episode_log_of(const EnvArraysLog& a) { return a.log; }

__device__ __forceinline__ Xo load_rng(const unsigned long long* rng, int64_t i) {
    const ulonglong2* p = reinterpret_cast<const ulonglong2*>(rng + 4 * i);
    ulonglong2 a = p[0], b = p[1];
    return Xo{a.x, a.y, b.x, b.y};
}
__device__ __forceinline__ void store_rng(unsigned long long* rng, int64_t i, const Xo& g) {
    ulonglong2* p = reinterpret_cast<ulonglong2*>(rng + 4 * i);
    p[0] = make_ulonglong2(g.s0, g.s1);
    p[1] = make_ulonglong2(g.s2, g.s3);
}

// ------------------------------------------------------------------ CartPole ----------
// CONT: CartPoleEnv(continuous = true) — ACT = T, action_space -1.0..1.0 (CartPoleEnv.jl:74-79,96,106-110)
template <class T, bool CONT = false> struct CartPoleD {
    using real = T;
    using act_t = typename std::conditional<CONT, T, int32_t>::type;
    static constexpr int NS = 4, NOBS = 4;
    static constexpr bool kObsIsState = true;
    static constexpr float kActionBound = 1.0f;   // CONT: action_space -1.0..1.0
    struct P { T g, M, m, l, pml, fmag, dt, ththr, xthr; int max_steps; };
    struct S { T x, xd, th, thd; };
    __device__ static S load(const void* st, int64_t i);
    __device__ static void store(void* st, int64_t i, const S& s);
    __device__ static bool valid(const P&, act_t a) {
        if (CONT) return (T)a >= (T)-kActionBound && (T)a <= (T)kActionBound;   // NaN fails
        return a == 1 || a == 2;
    }
    __device__ static unsigned long long n_random(const P&) { return 2; }
    __device__ static act_t from_index(const P&, long long a) { return (act_t)a; }
    // reset!: CartPoleEnv.jl:98-104 — rand(rng, T, 4) then rand(rng, Base.OneTo(2))
    __device__ static void reset(const P&, S& s, Xo& g, act_t& last_action) {
        T u[4];
        jld::rand4(g, u);
        s.x = (T)0.1 * u[0] - (T)0.05;
        s.xd = (T)0.1 * u[1] - (T)0.05;
        s.th = (T)0.1 * u[2] - (T)0.05;
        s.thd = (T)0.1 * u[3] - (T)0.05;
        // discrete: rand(rng, Base.OneTo(2)); continuous: rand(rng, -1.0..1.0) restated as
        // -1 + rand(Float64) * 2 (DomainSets sampler, external/unpinned) — one 64-bit output either way
        if (CONT) last_action = (act_t)(-1.0 + jld::rand_f64(g) * 2.0);
        else last_action = (act_t)jld::rand_oneto(g, 2);
    }
    // _step!: CartPoleEnv.jl:118-140.  `4 / 3` is Float64, so thetaacc, xacc and the two
    // velocity updates are Float64 for T = Float32; x and theta updates stay in T.
    __device__ static void step(const P& p, S& s, int& t, act_t a, bool& done, T& reward) {
        t += 1;
        T force = CONT ? (T)a * p.fmag : (T)(a == 2 ? 1 : -1) * p.fmag;
        T c = jld::jcos(s.th), sn = jld::jsin(s.th);
        T tmp = (force + (p.pml * (s.thd * s.thd)) * sn) / p.M;
        double den = (double)p.l * (4.0 / 3.0 - (double)((p.m * (c * c)) / p.M));
        double thacc = (double)(p.g * sn - c * tmp) / den;
        double xacc = (double)tmp - (((double)p.pml * thacc) * (double)c) / (double)p.M;
        T nx = s.x + p.dt * s.xd;
        T nxd = (T)((double)s.xd + (double)p.dt * xacc);
        T nth = s.th + p.dt * s.thd;
        T nthd = (T)((double)s.thd + (double)p.dt * thacc);
        s.x = nx; s.xd = nxd; s.th = nth; s.thd = nthd;
        done = fabs(nx) > p.xthr || fabs(nth) > p.ththr || t > p.max_steps;
        reward = done ? (T)0 : (T)1;  // CartPoleEnv.jl:84
    }
    __device__ static void write_obs(void*, int64_t, int64_t, const S&) {}
    __device__ static void observe(const S& s, float (&o)[4]) { o[0] = (float)s.x; o[1] = (float)s.xd; o[2] = (float)s.th; o[3] = (float)s.thd; }
};
template <class S> __device__ __forceinline__ S cp_load(const float* st, int64_t i) {
    float4 v = reinterpret_cast<const float4*>(st)[i];
    return S{v.x, v.y, v.z, v.w};
}
template <class S> __device__ __forceinline__ S cp_load(const double* st, int64_t i) {
    const double2* p = reinterpret_cast<const double2*>(st) + 2 * i;
    double2 a = p[0], b = p[1];
    return S{a.x, a.y, b.x, b.y};
}
template <class S> __device__ __forceinline__ void cp_store(float* st, int64_t i, const S& s) {
    reinterpret_cast<float4*>(st)[i] = make_float4(s.x, s.xd, s.th, s.thd);
}
template <class S> __device__ __forceinline__ void cp_store(double* st, int64_t i, const S& s) {
    double2* p = reinterpret_cast<double2*>(st) + 2 * i;
    p[0] = make_double2(s.x, s.xd);
    p[1] = make_double2(s.th, s.thd);
}
template <class T, bool CONT> __device__ __forceinline__ typename CartPoleD<T, CONT>::S CartPoleD<T, CONT>::load(const void* st, int64_t i) {
    return cp_load<S>(reinterpret_cast<const T*>(st), i);
}
template <class T, bool CONT> __device__ __forceinline__ void CartPoleD<T, CONT>::store(void* st, int64_t i, const S& s) {
    cp_store<S>(reinterpret_cast<T*>(st), i, s);
}

// ------------------------------------------------------------------ Pendulum ----------
// T = Float32 | Float64 (the reference constructor's default, PendulumEnv.jl:42): every literal below is written so that the
// Float32 instantiation keeps Julia's promotion points (2*pi, the cost terms and mod() are Float64) and the Float64 one is all-double.
template <class T> struct PendPT { T max_speed, max_torque, g, m, l, dt; int max_steps; int n_actions; };
using PendP = PendPT<float>;
template <class T> struct vec2_of;
template <> struct vec2_of<float> { using type = float2; };
template <> struct vec2_of<double> { using type = double2; };
template <bool CONT, class T = float> struct PendulumD {
    using real = T;
    using act_t = typename std::conditional<CONT, T, int32_t>::type;
    using V2 = typename vec2_of<T>::type;
    static constexpr int NS = 2, NOBS = 3;
    static constexpr bool kObsIsState = false;
    static constexpr float kActionBound = 2.0f;   // CONT: action_space -2.0..2.0 (PendulumEnv.jl:73)
    using P = PendPT<T>;
    struct S { T th, thd; T torque; };
    __device__ static S load(const void* st, int64_t i) {
        V2 v = reinterpret_cast<const V2*>(st)[i];
        return S{v.x, v.y, (T)0};
    }
    __device__ static void store(void* st, int64_t i, const S& s) {
        V2 v; v.x = s.th; v.y = s.thd;
        reinterpret_cast<V2*>(st)[i] = v;
    }
    __device__ static bool valid(const P& p, act_t a) {
        if (CONT) return (T)a >= (T)-kActionBound && (T)a <= (T)kActionBound;   // NaN fails
        return (int)a >= 1 && (int)a <= p.n_actions;
    }
    __device__ static unsigned long long n_random(const P& p) { return (unsigned long long)p.n_actions; }
    __device__ static act_t from_index(const P&, long long a) { return (act_t)a; }
    // reset!: PendulumEnv.jl:84-92 — two scalar rand(rng, T); `2 * pi` is Float64
    __device__ static void reset(const P&, S& s, Xo& g, act_t& last_action) {
        T u1 = jld::rand_real<T>(g);
        s.th = (T)((2 * JLD_PI) * (double)(u1 - (T)1));
        T u2 = jld::rand_real<T>(g);
        s.thd = (T)2 * (u2 - (T)1);
        (void)last_action;  // env.action = zero(T) is the torque field, not the policy action
    }
    // act!/_step!: PendulumEnv.jl:94-122
    __device__ static void step(const P& p, S& s, int& t, act_t a_in, bool& done, T& reward) {
        T a;
        if (CONT) {
            a = (T)a_in;
        } else {  // torque(env, a::Int) is Float64 arithmetic stored into env.action::T
            int n1 = p.n_actions - 1;
            a = (T)((4.0 / (double)n1) * ((double)(int)a_in - (double)n1 / 2 - 1));
        }
        t += 1;
        T th = s.th, thd = s.thd;
        a = jld::jclamp(a, -p.max_torque, p.max_torque);
        T thpi = th + (T)JLD_PI;
        double an = jld::jmod((double)thpi, 2 * JLD_PI) - JLD_PI;   // angle_normalize in Float64
        double costs = (an * an + 0.1 * (double)(thd * thd)) + 0.001 * (double)(a * a);
        T nthd = thd + (((((T)-3 * p.g) / ((T)2 * p.l)) * jld::jsin(thpi)) + (((T)3 * a) / (p.m * (p.l * p.l)))) * p.dt;
        th = th + nthd * p.dt;
        nthd = jld::jclamp(nthd, -p.max_speed, p.max_speed);
        s.th = th; s.thd = nthd; s.torque = a;
        done = t >= p.max_steps;
        reward = (T)(-costs);
    }
    // pendulum_observation: PendulumEnv.jl:70 (the fused Float32 rollout reads it as floats)
    __device__ static void observe(const S& s, float (&o)[4]) { o[0] = (float)jld::jsin(s.th); o[1] = (float)jld::jcos(s.th); o[2] = (float)s.thd; o[3] = 0.f; }
    __device__ static void write_obs(void* obs, int64_t i, int64_t, const S& s) {
        T* o = reinterpret_cast<T*>(obs) + 3 * i;
        o[0] = jld::jsin(s.th); o[1] = jld::jcos(s.th); o[2] = s.thd;
    }
};

// ---------------------------------------------------------------- MountainCar ---------
// CONT: ContinuousMountainCarEnv — force in -1.0..1.0 (MountainCarEnv.jl:73-74,83,93,107-111); T = Float32 | Float64 (the default, :67)
template <class T> struct MountainCarPT { T min_pos, max_pos, max_speed, goal_pos, goal_velocity, power, gravity; int max_steps; };
template <bool CONT = false, class T = float> struct MountainCarD {
    using real = T;
    using act_t = typename std::conditional<CONT, T, int32_t>::type;
    using V2 = typename vec2_of<T>::type;
    static constexpr int NS = 2, NOBS = 2;
    static constexpr bool kObsIsState = true;
    static constexpr float kActionBound = 1.0f;   // CONT: force in -1.0..1.0
    using P = MountainCarPT<T>;
    struct S { T x, v; };
    __device__ static S load(const void* st, int64_t i) {
        V2 v = reinterpret_cast<const V2*>(st)[i];
        return S{v.x, v.y};
    }
    __device__ static void store(void* st, int64_t i, const S& s) {
        V2 v; v.x = s.x; v.y = s.v;
        reinterpret_cast<V2*>(st)[i] = v;
    }
    __device__ static bool valid(const P&, act_t a) {
        if (CONT) return (T)a >= (T)-kActionBound && (T)a <= (T)kActionBound;
        return a >= 1 && a <= 3;
    }
    __device__ static unsigned long long n_random(const P&) { return 3; }
    __device__ static act_t from_index(const P&, long long a) { return (act_t)a; }
    // reset!: MountainCarEnv.jl:99-105 (Float64 literals 0.2, 0.6)
    __device__ static void reset(const P&, S& s, Xo& g, act_t&) {
        T u = jld::rand_real<T>(g);
        s.x = (T)(0.2 * (double)u - 0.6);
        s.v = (T)0;
    }
    // _step!: MountainCarEnv.jl:119-135
    __device__ static void step(const P& p, S& s, int& t, act_t a, bool& done, T& reward) {
        t += 1;
        T x = s.x, v = s.v;
        T force = CONT ? (T)a : (T)((int)a - 2);   // act!(env, a::Int) -> _step!(env, a - 2)
        v = v + (force * p.power + jld::jcos((T)3 * x) * (-p.gravity));
        v = jld::jclamp(v, -p.max_speed, p.max_speed);
        x = x + v;
        x = jld::jclamp(x, p.min_pos, p.max_pos);
        if (x == p.min_pos && v < 0) v = (T)0;
        done = (x >= p.goal_pos && v >= p.goal_velocity) || t >= p.max_steps;
        s.x = x; s.v = v;
        reward = done ? (T)0 : (T)-1;  // MountainCarEnv.jl:95
    }
    __device__ static void observe(const S& s, float (&o)[4]) { o[0] = (float)s.x; o[1] = (float)s.v; o[2] = 0.f; o[3] = 0.f; }
    __device__ static void write_obs(void*, int64_t, int64_t, const S&) {}
};


// ------------------------------------------------------------------- Acrobot ----------
// AcrobotEnv{Float64} (RLEnvs/src/environments/3rd_party/AcrobotEnv.jl:19-225; the constructor's default T).  One thread
// integrates one env.  DEVIATION: the reference calls OrdinaryDiffEq.solve(ode, RK4()) (adaptive step control of an external
// package, not restatable from the tree); this is ONE classical RK4 step over [0, dt] — gym's rk4, which the file cites as the
// source of its equations.  Unpinned; bit-exact against the CPU restatement the tests hold (same expression trees, no contraction).
struct AcrobotP { double l1, l2, m1, m2, lc1, lc2, moi, max_torque_noise, max_vel_a, max_vel_b, g, dt; int max_steps; int book; };
struct AcrobotD {
    using real = double;
    using act_t = int32_t;
    static constexpr int NS = 4, NOBS = 6;
    static constexpr bool kObsIsState = false;
    using P = AcrobotP;
    struct S { double th1, th2, dth1, dth2; };
    __device__ static S load(const void* st, int64_t i) {
        const double2* p = reinterpret_cast<const double2*>(st) + 2 * i;
        double2 a = p[0], b = p[1];
        return S{a.x, a.y, b.x, b.y};
    }
    __device__ static void store(void* st, int64_t i, const S& s) {
        double2* p = reinterpret_cast<double2*>(st) + 2 * i;
        p[0] = make_double2(s.th1, s.th2);
        p[1] = make_double2(s.dth1, s.dth2);
    }
    __device__ static bool valid(const P&, act_t a) { return a >= 1 && a <= 3; }   // Base.OneTo(3)
    __device__ static unsigned long long n_random(const P&) { return 3; }
    __device__ static act_t from_index(const P&, long long a) { return (act_t)a; }
    // reset!: AcrobotEnv.jl:100-107 — T(0.1) * rand(rng, T, 4) .- T(0.05); action = 2
    __device__ static void reset(const P&, S& s, Xo& g, act_t& last_action) {
        double u[4];
        jld::rand4(g, u);
        s.th1 = 0.1 * u[0] - 0.05;
        s.th2 = 0.1 * u[1] - 0.05;
        s.dth1 = 0.1 * u[2] - 0.05;
        s.dth2 = 0.1 * u[3] - 0.05;
        last_action = 2;
    }
    // dsdt: AcrobotEnv.jl:142-196 (expression trees as Julia parses them)
    __device__ static void dsdt(const P& p, const double (&s)[4], double a, double (&du)[4]) {
        const double m1 = p.m1, m2 = p.m2, l1 = p.l1, lc1 = p.lc1, lc2 = p.lc2, I1 = p.moi, I2 = p.moi, g = p.g;
        const double theta1 = s[0], theta2 = s[1], dtheta1 = s[2], dtheta2 = s[3];
        double ddtheta1 = 0.0, ddtheta2 = 0.0;
        const double c2 = jld::jcos(theta2), s2 = jld::jsin(theta2);
        const double d1 = ((m1 * (lc1 * lc1) + m2 * (((l1 * l1) + (lc2 * lc2)) + ((2 * l1) * lc2) * c2)) + I1) + I2;
        const double d2 = m2 * ((lc2 * lc2) + (l1 * lc2) * c2) + I2;
        const double phi2 = ((m2 * lc2) * g) * jld::jcos((theta1 + theta2) - JLD_PI / 2.0);
        const double phi1 = (((((((-m2) * l1) * lc2) * (dtheta2 * dtheta2)) * s2) - ((((((2 * m2) * l1) * lc2) * dtheta2) * dtheta1) * s2)) +
                             ((m1 * lc1 + m2 * l1) * g) * jld::jcos(theta1 - JLD_PI / 2)) + phi2;
        if (!p.book) {
            ddtheta2 = ((a + (d2 / d1) * phi1) - phi2) / (((m2 * (lc2 * lc2)) + I2) - (d2 * d2) / d1);
        } else {
            ddtheta2 = (((a + (d2 / d1) * phi1) - ((((m2 * l1) * lc2) * (dtheta1 * dtheta1)) * s2)) - phi2) / (((m2 * (lc2 * lc2)) + I2) - (d2 * d2) / d1);
            ddtheta1 = (-(d2 * ddtheta2 + phi1)) / d1;
        }
        du[0] = dtheta1; du[1] = dtheta2; du[2] = ddtheta1; du[3] = ddtheta2;
    }
    __device__ static double wrap(double x, double m, double M) {   // AcrobotEnv.jl:201-217
        const double diff = M - m;
        while (x > M) x = x - diff;
        while (x < m) x = x + diff;
        return x;
    }
    // act!: AcrobotEnv.jl:110-140
    __device__ static void step(const P& p, S& s, int& t, act_t a, bool& done, double& reward) {
        t += 1;
        const double torque = (double)((int)a - 2);   // avail_torque = [-1, 0, 1] (max_torque_noise = 0: no draw)
        const double h = p.dt, h2 = p.dt / 2.0;
        const double y0[4] = {s.th1, s.th2, s.dth1, s.dth2};
        double k1[4], k2[4], k3[4], k4[4], y[4];
        dsdt(p, y0, torque, k1);
#pragma unroll
        for (int i = 0; i < 4; ++i) y[i] = y0[i] + h2 * k1[i];
        dsdt(p, y, torque, k2);
#pragma unroll
        for (int i = 0; i < 4; ++i) y[i] = y0[i] + h2 * k2[i];
        dsdt(p, y, torque, k3);
#pragma unroll
        for (int i = 0; i < 4; ++i) y[i] = y0[i] + h * k3[i];
        dsdt(p, y, torque, k4);
        double ns[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) ns[i] = y0[i] + (h / 6.0) * (((k1[i] + 2 * k2[i]) + 2 * k3[i]) + k4[i]);
        ns[0] = wrap(ns[0], -JLD_PI, JLD_PI);
        ns[1] = wrap(ns[1], -JLD_PI, JLD_PI);
        ns[2] = fmin(fmax(ns[2], -p.max_vel_a), p.max_vel_a);
        ns[3] = fmin(fmax(ns[3], -p.max_vel_b), p.max_vel_b);
        s.th1 = ns[0]; s.th2 = ns[1]; s.dth1 = ns[2]; s.dth2 = ns[3];
        const bool succeeded = (-jld::jcos(ns[0]) - jld::jcos(ns[1] + ns[0])) > 1.0;
        done = succeeded || t > p.max_steps;
        reward = succeeded ? 0.0 : -1.0;
    }
    __device__ static void observe(const S&, float (&o)[4]) { o[0] = o[1] = o[2] = o[3] = 0.f; }   // (6 observations: no fused learner path)
    __device__ static void write_obs(void* obs, int64_t i, int64_t, const S& s) {   // acrobot_observation (AcrobotEnv.jl:76)
        double* o = reinterpret_cast<double*>(obs) + 6 * i;
        o[0] = jld::jcos(s.th1); o[1] = jld::jsin(s.th1); o[2] = jld::jcos(s.th2); o[3] = jld::jsin(s.th2); o[4] = s.dth1; o[5] = s.dth2;
    }
};

// StateTransformedEnv(env; state_mapping = s -> Float32.(s)) of a Float64 env: a (NOBS, N) float mirror of the observation, each
// entry the round-to-nearest of the Float64 observation (observe()).  It sits right behind the (NOBS, N) double observation in the
// same allocation, so no kernel takes a new parameter and the Float32 instantiations stay what they were.  Acrobot (6
// observations, no learner reads them) has none.
template <class Env> struct HasObsF32 {
    static constexpr bool value = std::is_same<typename Env::real, double>::value && Env::NOBS <= 4;
};
template <class Env> __device__ __forceinline__ float* obs_f32(const EnvArrays& a, int64_t N) {
    return reinterpret_cast<float*>(reinterpret_cast<double*>(a.obs) + (size_t)N * Env::NOBS);
}
// writes the mirror entry of env i (a no-op for the envs without a mirror)
template <class Env> __device__ __forceinline__ void store_obs_f32(const EnvArrays& a, int64_t i, int64_t N, const typename Env::S& s) {
    if constexpr (HasObsF32<Env>::value) {
        float o[4];
        Env::observe(s, o);
        float* m = obs_f32<Env>(a, N) + (size_t)Env::NOBS * i;
#pragma unroll
        for (int j = 0; j < Env::NOBS; ++j) m[j] = o[j];
    }
}

// What one act! step reports besides the env it updated
template <class T> struct ActStep {
    T rew;
    bool done;      // terminated, the MaxTimeoutEnv cut included
    float ret;      // episode return up to and including this step
    int len;        // env.t after the step: the episode's length when done
};

// act!(env, a) of one env: _step!, the MaxTimeoutEnv cut (terminated also when current_t = t + 1 > max_t, reward untouched,
// wrappers/MaxTimeoutEnv.jl:17-28), the running episode return and the flags byte (bit0 terminal, bit1 auto-reset).  An episode
// that finishes here — done, and not the terminal state of an env that was not reset since — is added to the caller's tally
// (fin_cnt, fin_ret, fin_len).  AUTO: a terminating step is followed by MultiThreadEnv's soft reset (reset!(env; is_force = false)):
// with_rng(f) calls f(Xo&) on the env's stream, which the caller may fetch only then; the reset may redraw `act` (env.action).
// LOG: the same finished episode is also written to env i's episode log `log` (without it the step is the code it was before
// the log existed).
template <class Env, bool AUTO, bool LOG = false, class WithRng>
__device__ __forceinline__ ActStep<typename Env::real> act_step(const typename Env::P& p, int max_timeout, typename Env::S& s, int& t,
                                                                int& flags, float& ep_ret, typename Env::act_t& act, int& fin_cnt,
                                                                float& fin_ret, int& fin_len, WithRng&& with_rng,
                                                                EpisodeLog log = EpisodeLog{}, int64_t i = 0) {
    ActStep<typename Env::real> r;
    Env::step(p, s, t, act, r.done, r.rew);
    if (max_timeout > 0 && t + 1 > max_timeout) r.done = true;
    r.ret = ep_ret + (float)r.rew;
    r.len = t;
    if (r.done && !((flags & 1) && !(flags & 2))) {
        fin_cnt += 1; fin_ret += r.ret; fin_len += t;
        if constexpr (LOG) log_episode(log, i, r.ret, t);
    }
    ep_ret = r.done ? 0.f : r.ret;
    flags = r.done ? 1 : 0;
    if (AUTO && r.done) {
        with_rng([&](Xo& g) { Env::reset(p, s, g, act); });
        t = 0;
        flags = 3;
    }
    return r;
}

#ifdef __CUDACC__
// Episode statistics of one CTA (device-side TotalRewardPerEpisode / BatchStepsPerEpisode, hooks.jl:146-231): each thread's
// finished-episode count, return and length -> warp sums (the returns in float) -> double sums over the warps in warp order -> one
// atomicAdd triple per CTA that saw a finished episode.  `red` is the caller's shared scratch; every thread of the CTA calls this.
// dv / red_dv / dv_out (optional): one more per-thread count, summed the same way and added to *dv_out when non-zero.
template <int NWARPS> struct StatsScratch { float ret[NWARPS]; int cnt[NWARPS], len[NWARPS]; };
template <int NWARPS>
__device__ __forceinline__ void cta_episode_stats(double* stats, int cnt, float ret, int len, StatsScratch<NWARPS>& red, long long dv = 0,
                                                  long long* red_dv = nullptr, unsigned long long* dv_out = nullptr) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        len += __shfl_xor_sync(0xffffffffu, len, o);
        ret += __shfl_xor_sync(0xffffffffu, ret, o);
        if (red_dv) dv += __shfl_xor_sync(0xffffffffu, dv, o);
    }
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
        red.cnt[w] = cnt; red.ret[w] = ret; red.len[w] = len;
        if (red_dv) red_dv[w] = dv;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double cc = 0, rr = 0, ll = 0;
        long long vv = 0;
        for (int k = 0; k < NWARPS; ++k) {
            cc += red.cnt[k]; rr += red.ret[k]; ll += red.len[k];
            if (red_dv) vv += red_dv[k];
        }
        if (cc > 0) { atomicAdd(&stats[0], cc); atomicAdd(&stats[1], rr); atomicAdd(&stats[2], ll); }
        if (vv != 0) atomicAdd(dv_out, (unsigned long long)vv);
    }
}
#endif

// what the fused consumers (fwd_tc.cu) need to know about a b200rl_env handle
struct EnvView {
    int kind, dtype, continuous;
    int64_t N;
    EnvArrays a;
    EpisodeLog log;   // the episode log the env's steps write (count == null: none)
    union {
        CartPoleD<float>::P cp32;
        CartPoleD<double>::P cp64;
        PendP pend;
        MountainCarD<false>::P mc;
        PendPT<double> pend64;
        MountainCarPT<double> mc64;
        AcrobotP acro;
    } p;
};

}  // namespace envdev
