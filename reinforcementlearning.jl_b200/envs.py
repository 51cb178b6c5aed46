"""Host-side mirror of the reference's env interface for the batched env
(RLBase/src/interface.jl:435-597; CartPoleEnv.jl / PendulumEnv.jl / MountainCarEnv.jl).

``B200VecEnv`` plays the role of the absent ``MultiThreadEnv``: ``reset_``/``act_``/``state``/
``reward``/``is_terminated`` have the reference's meaning with one extra leading batch
dimension (arrays are returned in Julia's column-major shape, e.g. state is (NS, N)
Fortran-ordered, so ``state[:, i]`` is env i).  Function names drop Julia's ``!`` for a
trailing underscore.  All arithmetic happens in libb200rl.so; nothing here computes."""
import ctypes as C
import math

import numpy as np

from . import _lib as L

_KINDS = {"CartPole": L.ENV_CARTPOLE, "Pendulum": L.ENV_PENDULUM, "MountainCar": L.ENV_MOUNTAINCAR,
          "ContinuousCartPole": L.ENV_CARTPOLE_CONTINUOUS, "ContinuousMountainCar": L.ENV_MOUNTAINCAR_CONTINUOUS, "Acrobot": L.ENV_ACROBOT}
_BASE = {L.ENV_CARTPOLE_CONTINUOUS: L.ENV_CARTPOLE, L.ENV_MOUNTAINCAR_CONTINUOUS: L.ENV_MOUNTAINCAR}
_NS = {L.ENV_CARTPOLE: 4, L.ENV_PENDULUM: 2, L.ENV_MOUNTAINCAR: 2, L.ENV_ACROBOT: 4}
_NOBS = {L.ENV_CARTPOLE: 4, L.ENV_PENDULUM: 3, L.ENV_MOUNTAINCAR: 2, L.ENV_ACROBOT: 6}


def cartpole_params(T=np.float32, gravity=9.8, masscart=1.0, masspole=0.1, halflength=0.5, forcemag=10.0, max_steps=200,
                    dt=0.02, thetathreshold=12.0, xthreshold=2.4):
    """CartPoleEnvParams{T}(; kwargs...) (CartPoleEnv.jl:22-46): derived fields in Float64, then every field -> T."""
    f = lambda v: float(T(v))
    return L.CartPoleParams(f(gravity), f(masscart), f(masspole), f(masscart + masspole), f(halflength), f(masspole * halflength),
                            f(forcemag), f(dt), f(thetathreshold * math.pi / 180), f(xthreshold), int(max_steps))


def pendulum_params(T=np.float32, max_speed=8, max_torque=2, g=10, m=1, l=1, dt=0.05, max_steps=200, continuous=True, n_actions=3):
    """PendulumEnv(; T, kwargs...) (PendulumEnv.jl:41-66): every field is T(value) (the reference default is T = Float64)."""
    f = lambda v: float(T(v))
    return L.PendulumParams(f(max_speed), f(max_torque), f(g), f(m), f(l), f(dt), int(max_steps), int(n_actions), int(bool(continuous)))


def mountaincar_params(T=np.float32, min_pos=-1.2, max_pos=0.6, max_speed=0.07, goal_pos=0.5, goal_velocity=0.0, power=0.001, gravity=0.0025,
                       max_steps=200):
    """MountainCarEnvParams(; T, kwargs...) (MountainCarEnv.jl:19-40; the reference default is T = Float64)."""
    f = lambda v: float(T(v))
    return L.MountainCarParams(f(min_pos), f(max_pos), f(max_speed), f(goal_pos), f(goal_velocity), f(power), f(gravity), int(max_steps))


def acrobot_params(link_length_a=1.0, link_length_b=1.0, link_mass_a=1.0, link_mass_b=1.0, link_com_pos_a=0.5, link_com_pos_b=0.5, link_moi=1.0,
                   max_vel_a=4 * math.pi, max_vel_b=9 * math.pi, g=9.8, dt=0.2, max_steps=200, book_or_nips="book"):
    """AcrobotEnv(; T = Float64, kwargs...) (3rd_party/AcrobotEnv.jl:19-60); max_torque_noise is fixed at 0."""
    return L.AcrobotParams(link_length_a, link_length_b, link_mass_a, link_mass_b, link_com_pos_a, link_com_pos_b, link_moi, 0.0,
                           max_vel_a, max_vel_b, g, dt, int(max_steps), 1 if book_or_nips == "book" else 0)


class B200VecEnv:
    """N classic-control envs stepped by one sm_90a kernel launch.

    ``rng_state``: (N, 4) uint64 raw Xoshiro256++ states (what Julia's ``Xoshiro(seed_i)`` holds).
    ``auto_reset``: fuse MultiThreadEnv's soft reset of finished sub-envs into ``act_``."""

    def __init__(self, ctx, kind, n_envs, rng_state, T=np.float32, params=None, auto_reset=False, **kwargs):
        self.ctx, self.lib = ctx, ctx.lib
        create_kind = _KINDS[kind] if isinstance(kind, str) else int(kind)
        self.kind = _BASE.get(create_kind, create_kind)     # kind of dynamics; `continuous` carries the action type
        self.n = int(n_envs)
        self.T = np.dtype(T).type
        self.auto_reset = bool(auto_reset)
        self.state_f32 = False
        if params is None:
            if self.kind == L.ENV_CARTPOLE:
                params = cartpole_params(T=self.T, **kwargs)
            elif self.kind == L.ENV_PENDULUM:
                params = pendulum_params(T=self.T, **kwargs)
            elif self.kind == L.ENV_ACROBOT:
                params = acrobot_params(**kwargs)
            elif create_kind == L.ENV_MOUNTAINCAR_CONTINUOUS:  # MountainCarEnv.jl:73-74
                params = mountaincar_params(T=self.T, **{"goal_pos": 0.45, "power": 0.0015, **kwargs})
            else:
                params = mountaincar_params(T=self.T, **kwargs)
        self.params = params
        self.continuous = create_kind in _BASE or (self.kind == L.ENV_PENDULUM and bool(params.continuous))
        # a continuous action is a T (Float64 actions for a Float64 env), a discrete one an Int32 (1-based)
        self.act_dtype = (np.float64 if self.T is np.float64 else np.float32) if self.continuous else np.int32
        rng_state = np.ascontiguousarray(rng_state, dtype=np.uint64).reshape(self.n, 4)
        h = C.c_void_p()
        L.check(self.lib.b200rl_env_create(ctx.h, create_kind, L.F64 if self.T is np.float64 else L.F32, self.n,
                                           C.byref(params), L.ptr(rng_state), C.byref(h)))
        self.h = h

    @classmethod
    def _from_handle(cls, src, h):
        o = cls.__new__(cls)
        o.__dict__.update({k: v for k, v in src.__dict__.items() if k != "h"})
        o.h = h
        return o

    def close(self):
        if getattr(self, "h", None):
            self.lib.b200rl_env_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __len__(self):
        return self.n

    # ---- RLBase verbs -------------------------------------------------------------
    def reset_(self, is_force=True):
        """RLBase.reset!(env) for every env (is_force) or only for finished ones (MultiThreadEnv soft reset)."""
        L.check(self.lib.b200rl_env_reset(self.h, int(is_force)))

    def act_(self, actions):
        """RLBase.act!(env, a): ``actions`` is a host array (N,) or a device pointer (int).
        Discrete actions are 1-based like the reference's ``Base.OneTo(n)``."""
        if isinstance(actions, (int, np.integer)):
            L.check(self.lib.b200rl_env_step(self.h, C.c_void_p(int(actions)), 1, int(self.auto_reset)))
        else:
            a = np.ascontiguousarray(actions, dtype=self.act_dtype)
            if a.shape != (self.n,):
                raise ValueError(f"expected {self.n} actions, got shape {a.shape}")
            # the agent's own pinned action buffer (returned by plan!): stream-ordered copy, no host sync — the next plan!
            # rewrites it with a D2H copy that is ordered behind this H2D copy on the same stream
            pinned = a.ctypes.data == getattr(self, "pinned_action_addr", None)
            L.check(self.lib.b200rl_env_step(self.h, L.ptr(a), 2 if pinned else 0, int(self.auto_reset)))

    def set_max_timeout(self, max_t):
        """MaxTimeoutEnv(env, max_t) (wrappers/MaxTimeoutEnv.jl:17-28); 0 removes the wrapper."""
        L.check(self.lib.b200rl_env_set_max_timeout(self.h, int(max_t)))

    def set_state_float32(self, on=True):
        """StateTransformedEnv(env; state_mapping = s -> Float32.(s)) (wrappers/StateTransformedEnv.jl:15-19) as a flag: state()
        returns Float32 (round to nearest of the Float64 observation) and the learners, trajectories and evaluate() take a Float64
        env.  The dynamics are untouched: every other field stays the unwrapped env's, bit for bit.  ``on=False`` removes the
        wrapper.  The identity on a Float32 env; refused on Acrobot."""
        L.check(self.lib.b200rl_env_set_state_f32(self.h, int(bool(on))))
        self.state_f32 = bool(on)

    def obs_device_ptr(self):
        """device pointer of the Float32 (NOBS, N) observation the networks read (refused for an unwrapped Float64 env)"""
        return self.device_ptr(L.FIELD_OBS_F32)

    def act_random_(self):
        """plan!(RandomPolicy(), env) + act!(env, a) fused: each env draws from its own stream."""
        L.check(self.lib.b200rl_env_step_random(self.h, int(self.auto_reset)))

    def _get(self, field, shape, dtype, order="F"):
        out = np.empty(shape, dtype=dtype, order=order)
        L.check(self.lib.b200rl_env_get(self.h, field, L.ptr(out), out.nbytes))
        return out

    def state(self):
        """state(env): (NOBS, N) observation batch (Float32 behind set_state_float32)."""
        if self.state_f32:
            return self._get(L.FIELD_OBS_F32, (_NOBS[self.kind], self.n), np.float32)
        return self._get(L.FIELD_OBS, (_NOBS[self.kind], self.n), self.T)

    def internal_state(self):
        return self._get(L.FIELD_STATE, (_NS[self.kind], self.n), self.T)

    def reward(self):
        return self._get(L.FIELD_REWARD, (self.n,), self.T)

    def is_terminated(self):
        return self._get(L.FIELD_TERMINAL, (self.n,), np.uint8).astype(bool)

    def flags(self):
        return self._get(L.FIELD_FLAGS, (self.n,), np.uint8)

    def t(self):
        return self._get(L.FIELD_T, (self.n,), np.int32)

    def rng_state(self):
        return self._get(L.FIELD_RNG, (self.n, 4), np.uint64, order="C")

    def last_action(self):
        return self._get(L.FIELD_ACTION, (self.n,), self.act_dtype)

    def set_field(self, field, arr):
        arr = np.asarray(arr)
        arr = np.asfortranarray(arr) if arr.ndim == 2 and field != L.FIELD_RNG else np.ascontiguousarray(arr)
        L.check(self.lib.b200rl_env_set(self.h, field, L.ptr(arr), arr.nbytes))

    def device_ptr(self, field):
        p = C.c_void_p()
        L.check(self.lib.b200rl_env_ptr(self.h, field, C.byref(p)))
        return p.value

    def seed_(self, rng_state):
        """Random.seed!(env, seed) with raw states."""
        rng_state = np.ascontiguousarray(rng_state, dtype=np.uint64).reshape(self.n, 4)
        L.check(self.lib.b200rl_env_seed(self.h, L.ptr(rng_state)))

    def copy(self):
        h = C.c_void_p()
        L.check(self.lib.b200rl_env_copy(self.h, C.byref(h)))
        return B200VecEnv._from_handle(self, h)

    def check(self):
        """Raise if an out-of-space action was seen (the reference's `@assert a in action_space(env)`)."""
        L.check(self.lib.b200rl_env_check(self.h))

    def episode_stats(self, reset=False):
        out = np.zeros(4, dtype=np.float64)
        L.check(self.lib.b200rl_env_episode_stats(self.h, L.ptr(out), int(reset)))
        return {"episodes": int(out[0]), "return_sum": out[1], "length_sum": out[2], "env_steps": int(out[3])}

    # ---- device episode log (b200rl_env_episode_log) -----------------------------------
    EPISODE_RECORD = np.dtype([("env", "<i8"), ("ret", "<f4"), ("len", "<i4")])   # b200rl_episode_record

    def episode_log(self, K):
        """Attach a ring of K {return, length} records per env, written by every step that ends an episode (K = 0 detaches)."""
        L.check(self.lib.b200rl_env_episode_log(self.h, int(K)))

    def episode_log_buffer(self, capacity):
        """Pinned host buffer for flushes of up to ``capacity`` records: (array view, address); free with ctx.host_free."""
        return self.ctx.host_alloc((16 + 16 * int(capacity),), np.uint8)

    def episode_log_flush(self, buf, capacity):
        """Start handing the records logged since the previous flush to the pinned buffer ``buf`` (an address); no sync."""
        L.check(self.lib.b200rl_env_episode_log_flush(self.h, C.c_void_p(buf), int(capacity)))

    def episode_log_read(self, buf_arr, buf):
        """Wait for the last flush into ``buf`` and return its records (EPISODE_RECORD, ordered by env then episode; a copy).
        Raises (ERR_OVERFLOW) when an env finished more than K episodes between two flushes."""
        n = C.c_int64()
        L.check(self.lib.b200rl_env_episode_log_read(self.h, C.c_void_p(buf), C.byref(n)))
        return buf_arr[16:16 + 16 * n.value].view(self.EPISODE_RECORD).copy()

    # ---- spaces (shape information only) ---------------------------------------------
    def action_space(self):
        if self.kind == L.ENV_CARTPOLE:
            return (-1.0, 1.0) if self.continuous else range(1, 3)
        if self.kind == L.ENV_MOUNTAINCAR:
            return (-1.0, 1.0) if self.continuous else range(1, 4)
        if self.kind == L.ENV_ACROBOT:
            return range(1, 4)
        return (-2.0, 2.0) if self.continuous else range(1, int(self.params.n_actions) + 1)

    def state_space(self):
        p = self.params
        inf = float("inf")
        if self.kind == L.ENV_CARTPOLE:  # CartPoleEnv.jl:88-93
            return [(-2 * p.xthreshold, 2 * p.xthreshold), (-inf, inf), (-2 * p.thetathreshold, 2 * p.thetathreshold), (-inf, inf)]
        if self.kind == L.ENV_PENDULUM:  # PendulumEnv.jl:75-79
            return [(-1.0, 1.0), (-1.0, 1.0), (-p.max_speed, p.max_speed)]
        if self.kind == L.ENV_ACROBOT:   # AcrobotEnv.jl:80-90
            return [(-1.0, 1.0)] * 4 + [(-p.max_vel_a, p.max_vel_a), (-p.max_vel_b, p.max_vel_b)]
        return [(p.min_pos, p.max_pos), (-p.max_speed, p.max_speed)]  # MountainCarEnv.jl:87-90
