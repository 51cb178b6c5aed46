"""Host mirror of the learner side: network handle (FluxApproximator + TargetNetwork,
RLCore/src/policies/learners/flux_approximator.jl:11-46, target_network.jl:27-88), the
on-policy agent (Agent + PPOPolicy/A2C, RLCore/src/policies/agent/agent_base.jl:18-66 and the
absent RLZoo learners), the device trajectory (CircularArraySARTSTraces + samplers) and the
DQN learner.  Thin ctypes calls only."""
import ctypes as C

import numpy as np

from . import _lib as L
from .core import AbstractPolicy, FusedAction, PostActStage, PreActStage, PreEpisodeStage, PreExperimentStage
from .envs import _NOBS
from .explorers import (EpsilonGreedyExplorer, EpsilonSpeedyExplorer, GreedyExplorer, GumbelSoftmaxExplorer,
                        WeightedSoftmaxExplorer)

ACT_RELU, ACT_TANH = 0, 1
KIND_CATEGORICAL, KIND_GAUSSIAN, KIND_Q, KIND_DUELING = 0, 1, 2, 3
Q_KINDS = (KIND_Q, KIND_DUELING)     # Q-networks: a target copy, the DQN learner, QBasedPolicy
NET_PARAMS, NET_GRAD, NET_M, NET_V, NET_BETA_T, NET_TARGET = range(6)


def onpolicy_config(gamma=0.99, lambda_=0.95, clip_range=0.1, max_grad_norm=0.5, w_actor=1.0, w_critic=0.5, w_entropy=0.001,
                    lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, min_sigma=0.0, max_sigma=float("inf"), normalize_advantage=True,
                    n_epochs=4, n_microbatches=4, update_freq=32, algo="ppo"):
    """Defaults = the in-tree PPO example (docs/homepage/blog/a_practical_introduction_to_RL.jl/index.html:15238-15286)."""
    return L.OnPolicyConfig(gamma, lambda_, clip_range, max_grad_norm, w_actor, w_critic, w_entropy, lr, beta1, beta2, eps, min_sigma,
                            max_sigma, int(normalize_advantage), n_epochs, n_microbatches, update_freq, {"ppo": 0, "a2c": 1}[algo])


def dqn_config(gamma=0.99, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, max_grad_norm=0.0, rho=0.0, per_alpha=0.6, per_beta=0.4,
               per_eps=1e-6, huber=True, double_dqn=False, target_update_freq=100):
    return L.DQNConfig(gamma, lr, beta1, beta2, eps, max_grad_norm, rho, per_alpha, per_beta, per_eps, int(huber), int(double_dqn),
                       target_update_freq)


class Network:
    """b200rl_net: parameters + Adam state (+ target copy) on the device.

    kind KIND_DUELING: DuelingNetwork(base = trunk, val = Dense(hidden, 1), adv = Dense(hidden, n_out)) with n_out = number of
    actions (1..3); ``params`` is ``Flux.destructure`` of it as it is, and everything that reads Q sees (val + adv) - mean(adv)."""

    def __init__(self, ctx, n_in, hidden, n_out, params, act=ACT_RELU, kind=KIND_CATEGORICAL):
        self.ctx, self.lib = ctx, ctx.lib
        self.desc = L.NetDesc(n_in, hidden, act, n_out, kind)
        n = C.c_int64()
        L.check(self.lib.b200rl_net_nparams(C.byref(self.desc), C.byref(n)))
        self.nparams = n.value
        params = np.ascontiguousarray(params, dtype=np.float32)
        if params.size != self.nparams:
            raise ValueError(f"expected {self.nparams} parameters, got {params.size}")
        h = C.c_void_p()
        L.check(self.lib.b200rl_net_create(ctx.h, C.byref(self.desc), L.ptr(params), C.byref(h)))
        self.h = h
        self.kind, self.n_in, self.n_out = kind, n_in, n_out

    @property
    def is_q(self):
        return self.kind in Q_KINDS

    @staticmethod
    def count_params(ctx, n_in, hidden, n_out, act=ACT_RELU, kind=KIND_CATEGORICAL):
        d = L.NetDesc(n_in, hidden, act, n_out, kind)
        n = C.c_int64()
        L.check(ctx.lib.b200rl_net_nparams(C.byref(d), C.byref(n)))
        return n.value

    def close(self):
        if getattr(self, "h", None):
            self.lib.b200rl_net_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def configure_optimizer(self, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, max_grad_norm=0.5):
        L.check(self.lib.b200rl_net_configure_optimizer(self.h, lr, beta1, beta2, eps, max_grad_norm))

    def get(self, which=NET_PARAMS):
        out = np.empty(2 if which == NET_BETA_T else self.nparams, np.float32)
        L.check(self.lib.b200rl_net_get(self.h, which, L.ptr(out), out.size))
        return out

    def set(self, which, arr):
        arr = np.ascontiguousarray(arr, np.float32)
        L.check(self.lib.b200rl_net_set(self.h, which, L.ptr(arr), arr.size))

    def device_ptr(self, which=NET_PARAMS):
        p = C.c_void_p()
        L.check(self.lib.b200rl_net_ptr(self.h, which, C.byref(p)))
        return p.value

    def step_count(self):
        n = C.c_int64()
        L.check(self.lib.b200rl_net_get_step(self.h, C.byref(n)))
        return n.value

    def set_step_count(self, n):
        L.check(self.lib.b200rl_net_set_step(self.h, int(n)))

    def target_sync(self, rho=0.0):
        L.check(self.lib.b200rl_net_target_sync(self.h, rho))

    def act(self, obs, rng_dev):
        """obs (n_in, N) host array; rng_dev: device pointer to (4, N) policy streams."""
        obs = np.asfortranarray(obs, np.float32)
        n = obs.shape[1]
        action = np.empty(n, np.float32 if self.kind == KIND_GAUSSIAN else np.int32)
        logp = np.empty(n, np.float32); value = np.empty(n, np.float32)
        nh = 2 if self.kind == KIND_GAUSSIAN else self.n_out
        heads = np.empty((nh, n), np.float32, order="F")
        L.check(self.lib.b200rl_net_act(self.h, L.ptr(obs), n, C.c_void_p(rng_dev), L.ptr(action), L.ptr(logp), L.ptr(value), L.ptr(heads), 0))
        return dict(action=action, logp=logp, value=value, heads=heads)

    def values(self, obs, use_target=False):
        obs = np.asfortranarray(obs, np.float32)
        n = obs.shape[1]
        out = np.empty((self.n_out, n), np.float32, order="F") if self.is_q else np.empty(n, np.float32)
        L.check(self.lib.b200rl_net_values(self.h, L.ptr(obs), n, L.ptr(out), int(use_target), 0))
        return out

    def ac_step(self, cfg, states, actions, logp_old, adv, ret, idx=None, adv_mean=0.0, adv_inv_std=1.0, apply_update=True):
        states = np.asfortranarray(states, np.float32)
        total = states.shape[1]
        actions = np.ascontiguousarray(actions)
        assert actions.dtype in (np.int32, np.float32)
        idx = None if idx is None else np.ascontiguousarray(idx, np.int32)
        losses = np.zeros(6, np.float32)
        L.check(self.lib.b200rl_net_ac_step(
            self.h, C.byref(cfg), L.ptr(states), L.ptr(actions), L.ptr(None if logp_old is None else np.ascontiguousarray(logp_old, np.float32)),
            L.ptr(np.ascontiguousarray(adv, np.float32)), L.ptr(np.ascontiguousarray(ret, np.float32)), total, L.ptr(idx),
            0 if idx is None else idx.size, adv_mean, adv_inv_std, int(apply_update), L.ptr(losses)))
        return dict(actor_loss=losses[0], critic_loss=losses[1], entropy=losses[2], loss=losses[3], grad_norm=losses[4])


def _library_budget(budget):
    """the budget argument of b200rl_*_run_episodes: -1 (none) for StopAfterNSteps; an episode budget already spent is 0 (one
    step, as the stage loop checks only after a step), never negative"""
    return -1 if budget is None else max(0, int(budget))


ROLL_STATE, ROLL_ACTION, ROLL_LOGP, ROLL_REWARD, ROLL_TERMINAL, ROLL_VALUE, ROLL_ADV, ROLL_RET, ROLL_RNG, ROLL_NORM = range(10)


class OnPolicyAgent(AbstractPolicy):
    """Agent(policy = PPOPolicy | A2CPolicy, trajectory = PPOTrajectory) on the device.

    Two ways to drive it: the reference's stage protocol (``plan`` returns host actions, the run
    loop calls ``env.act_``, ``push`` / ``optimise`` follow — host buffers every step), or the fused
    path (``collect(n)`` / ``update()``), where actions never leave the device."""

    def __init__(self, ctx, net, env, cfg, policy_rng, host_actions=True):
        self.ctx, self.lib, self.net, self.env, self.cfg = ctx, ctx.lib, net, env, cfg
        self.n, self.T = env.n, cfg.update_freq
        self.host_actions = host_actions
        self.fusable = not host_actions     # run() may hand whole stretches of env steps to run_episodes()
        policy_rng = np.ascontiguousarray(policy_rng, np.uint64).reshape(self.n, 4)
        h = C.c_void_p()
        L.check(self.lib.b200rl_onpolicy_create(ctx.h, net.h, env.h, C.byref(cfg), L.ptr(policy_rng), C.byref(h)))
        self.h = h
        self.continuous = env.continuous
        # pinned host buffer for the per-step action round trip of the stage protocol
        self._act_buf, self._act_buf_addr = ctx.host_alloc((self.n,), np.float32 if self.continuous else np.int32)
        env.pinned_action_addr = self._act_buf.ctypes.data
        self.last_stats = None
        self.n_updates = 0
        self.fetch_stats = False   # read the per-minibatch losses back after every update (a sync)
        self._t = 0                # host mirror of the rollout fill level (no device query per step)

    def close(self):
        if getattr(self, "h", None):
            self.lib.b200rl_onpolicy_destroy(self.h)
            self.h = None
            self._act_buf = None
            self.ctx.host_free(self._act_buf_addr)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def time_kernel(self, which, reps=20):
        ms = C.c_float()
        L.check(self.lib.b200rl_onpolicy_time_kernel(self.h, which, reps, C.byref(ms)))
        return ms.value

    # ---- stage protocol (run.jl:52-68) -------------------------------------------------------
    def plan(self, env):
        if self.host_actions:
            L.check(self.lib.b200rl_onpolicy_plan(self.h, L.ptr(self._act_buf)))
            if self.continuous:
                lo, hi = env.action_space()               # the env asserts a in -2.0..2.0 (Pendulum) | -1.0..1.0
                # a Float64 env receives Float64 of the clamped Float32 sample (exact bounds: the clamp in Float64)
                return np.clip(self._act_buf, np.float32(lo), np.float32(hi)).astype(env.act_dtype)
            return self._act_buf
        L.check(self.lib.b200rl_onpolicy_plan(self.h, None))
        return FusedAction("policy")

    def act_fused(self, env):
        L.check(self.lib.b200rl_onpolicy_act(self.h))

    def push(self, stage, env, action=None):
        if stage == PostActStage:
            L.check(self.lib.b200rl_onpolicy_push(self.h))

    def optimise(self, stage):
        if stage == PostActStage:
            self._t += 1
            if self._t == self.T:
                self._t = 0
                self.update(want_stats=self.fetch_stats)

    # ---- fused path --------------------------------------------------------------------------
    def collect(self, n_steps):
        L.check(self.lib.b200rl_onpolicy_collect(self.h, n_steps))
        self._t = (self._t + n_steps)

    def fill(self):
        t, T = C.c_int(), C.c_int()
        L.check(self.lib.b200rl_onpolicy_fill(self.h, C.byref(t), C.byref(T)))
        return t.value, T.value

    def update(self, perm=None, want_stats=False):
        rows = self.cfg.n_epochs * self.cfg.n_microbatches
        stats = np.zeros((rows, 6), np.float32) if want_stats else None
        if perm is not None:
            perm = np.ascontiguousarray(perm, np.int32)
            assert perm.shape == (self.cfg.n_epochs, self.n * self.T)
        L.check(self.lib.b200rl_onpolicy_update(self.h, L.ptr(perm), L.ptr(stats)))
        self._t = 0
        self.n_updates += 1
        self.last_stats = stats
        return stats

    def iterate(self, n_iters=1, want_stats=False):
        """n_iters x {collect(T); update()} as one CUDA-graph launch per iteration (b200rl_onpolicy_iterate)."""
        rows = self.cfg.n_epochs * self.cfg.n_microbatches
        stats = np.zeros((rows, 6), np.float32) if want_stats else None
        L.check(self.lib.b200rl_onpolicy_iterate(self.h, n_iters, L.ptr(stats)))
        self._t = 0
        self.n_updates += n_iters
        self.last_stats = stats
        return stats

    def run_episodes(self, max_steps, budget):
        """At most max_steps env steps of run(agent, env, stop) on the fused path (b200rl_onpolicy_run_episodes).  budget = k - cur
        for StopAfterNEpisodes(k): stops after the step at which the episodes counted reach it, as the stage loop does (a budget
        <= 0: one step).  budget None for StopAfterNSteps: runs max_steps steps, or stops earlier at the end of the last rollout
        they complete.  Returns (steps run, episodes they ended; 0 without a budget)."""
        rows = self.cfg.n_epochs * self.cfg.n_microbatches
        stats = np.zeros((rows, 6), np.float32) if self.fetch_stats else None
        c0, c1 = np.zeros(3, np.int64), np.zeros(3, np.int64)
        steps, episodes = C.c_int64(), C.c_int64()
        L.check(self.lib.b200rl_onpolicy_export_state(self.h, L.ptr(c0)))
        L.check(self.lib.b200rl_onpolicy_run_episodes(self.h, int(max_steps), _library_budget(budget), L.ptr(stats), C.byref(steps),
                                                      C.byref(episodes)))
        L.check(self.lib.b200rl_onpolicy_export_state(self.h, L.ptr(c1)))
        self._t = int(c1[0])
        if c1[1] != c0[1]:
            self.n_updates += int(c1[1] - c0[1])
            self.last_stats = stats
        return steps.value, episodes.value

    def graph_active(self):
        v = C.c_int()
        L.check(self.lib.b200rl_onpolicy_graph_active(self.h, C.byref(v)))
        return bool(v.value)

    def rollout(self, field):
        n, T, ns = self.n, self.T, self.net.n_in
        spec = {
            ROLL_STATE: ((ns, n, T + 1), np.float32), ROLL_ACTION: ((n, T), np.float32 if self.continuous else np.int32),
            ROLL_LOGP: ((n, T), np.float32), ROLL_REWARD: ((n, T), np.float32), ROLL_TERMINAL: ((n, T), np.uint8),
            ROLL_VALUE: ((n, T + 1), np.float32), ROLL_ADV: ((n, T), np.float32), ROLL_RET: ((n, T), np.float32),
            ROLL_RNG: ((4, n), np.uint64), ROLL_NORM: ((2,), np.float32),
        }[field]
        out = np.empty(spec[0], dtype=spec[1], order="F")
        L.check(self.lib.b200rl_onpolicy_get(self.h, field, L.ptr(out), out.nbytes))
        return out


BATCH_STATE, BATCH_ACTION, BATCH_REWARD, BATCH_TERMINAL, BATCH_NEXT_STATE, BATCH_KEY, BATCH_PRIORITY, BATCH_WEIGHT, BATCH_RNG = range(9)
BATCH_DISCOUNT, BATCH_HORIZON = 9, 10


class Trajectory:
    """Trajectory(container = CircularArraySARTSTraces(capacity) [+ CircularPrioritizedTraces],
    sampler = BatchSampler(batch_size) | NStepBatchSampler(n_step, gamma)) resident on the device.

    n_step > 1: a sampled entry's reward / terminal / next_state come from its n-step window (it ends early at a terminal entry,
    the lane's newest frame or a forced reset), and the batch's ``discount`` (gamma^m) and ``horizon`` (m) say how long the window
    was; the DQN learner's gamma must equal ``gamma``.  n_step = 1 is the BatchSampler, bit for bit."""

    def __init__(self, ctx, ns, capacity, lanes=1, batch_size=0, sampler_rng=None, prioritized=False, default_priority=1.0, n_step=1,
                 gamma=0.99):
        self.ctx, self.lib = ctx, ctx.lib
        self.ns, self.lanes, self.capacity, self.batch_size, self.prioritized = ns, lanes, capacity, batch_size, prioritized
        if batch_size:
            sampler_rng = np.ascontiguousarray(sampler_rng, np.uint64).reshape(batch_size, 4)
        h = C.c_void_p()
        L.check(self.lib.b200rl_traj_create(ctx.h, ns, lanes, capacity, int(prioritized), default_priority, L.ptr(sampler_rng), batch_size, C.byref(h)))
        self.h = h
        self.n_step, self.gamma = 1, 0.99
        if n_step != 1:
            try:
                self.set_nstep(n_step, gamma)
            except Exception:
                self.close()
                raise

    def set_nstep(self, n_step, gamma):
        """NStepBatchSampler(n_step, gamma) from the next sample on (b200rl_traj_set_nstep); n_step = 1 is the BatchSampler."""
        L.check(self.lib.b200rl_traj_set_nstep(self.h, int(n_step), float(gamma)))
        self.n_step, self.gamma = int(n_step), float(np.float32(gamma))

    def close(self):
        if getattr(self, "h", None):
            self.lib.b200rl_traj_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __len__(self):
        n = C.c_int64()
        L.check(self.lib.b200rl_traj_length(self.h, C.byref(n)))
        return n.value

    def push_state(self, obs):
        obs = np.asfortranarray(obs, np.float32)
        L.check(self.lib.b200rl_traj_push_state(self.h, L.ptr(obs), 0))

    def push_episode_start(self, obs, pending_only=False, on_device=False):
        """push!(trajectory, (state = s0,)): every lane, or (pending_only) the lanes whose last transition was terminal."""
        if not on_device:
            obs = np.asfortranarray(obs, np.float32)
        L.check(self.lib.b200rl_traj_push_episode_start(self.h, L.ptr(obs), int(on_device), int(pending_only)))

    def lane_lengths(self):
        out = np.empty(self.lanes, np.int64)
        L.check(self.lib.b200rl_traj_lane_lengths(self.h, L.ptr(out)))
        return out

    def n_sampleable(self):
        n = C.c_int64()
        L.check(self.lib.b200rl_traj_n_sampleable(self.h, C.byref(n)))
        return n.value

    # ---- checkpoint of the ring (fields of b200rl_traj_get) ----------------------------------
    FIELDS = {"state": (0, np.float32), "action": (1, np.int32), "reward": (2, np.float32), "flag": (3, np.uint8), "head": (4, np.int32),
              "count": (5, np.int32), "pending": (6, np.uint8), "n_sampleable": (7, np.int64), "tree": (8, np.float32), "sampler_rng": (9, np.uint64)}

    def export_state(self):
        out = {}
        for name, (f, dt) in self.FIELDS.items():
            if (name == "tree" and not self.prioritized) or (name == "sampler_rng" and not self.batch_size):
                continue
            nb = C.c_size_t()
            L.check(self.lib.b200rl_traj_field_bytes(self.h, f, C.byref(nb)))
            a = np.empty(nb.value // np.dtype(dt).itemsize, dt)
            L.check(self.lib.b200rl_traj_get(self.h, f, L.ptr(a), a.nbytes))
            out[name] = a
        if hasattr(self, "controller"):
            c = self.controller
            out["controller"] = np.array([c.ratio, c.threshold, c.n_inserted, c.n_sampled], np.float64)
        return out

    def import_state(self, st):
        for name, (f, dt) in self.FIELDS.items():
            if name in st:
                a = np.ascontiguousarray(st[name], dt)
                L.check(self.lib.b200rl_traj_set(self.h, f, L.ptr(a), a.nbytes))
        if "controller" in st and hasattr(self, "controller"):
            c = self.controller
            c.ratio, c.threshold, c.n_inserted, c.n_sampled = float(st["controller"][0]), int(st["controller"][1]), int(st["controller"][2]), int(st["controller"][3])

    def push(self, action, reward, terminal, next_obs):
        L.check(self.lib.b200rl_traj_push(self.h, L.ptr(np.ascontiguousarray(action, np.int32)), L.ptr(np.ascontiguousarray(reward, np.float32)),
                                          L.ptr(np.ascontiguousarray(terminal, np.uint8)), L.ptr(np.asfortranarray(next_obs, np.float32)), 0))

    def push_env(self, env, first_state_only=False):
        L.check(self.lib.b200rl_traj_push_env(self.h, env.h, int(first_state_only)))

    def sample(self, beta=0.4, fetch=True):
        L.check(self.lib.b200rl_traj_sample(self.h, beta))
        return self.batch() if fetch else None

    def batch(self):
        B, ns = self.batch_size, self.ns
        spec = {"state": (BATCH_STATE, (ns, B), np.float32), "action": (BATCH_ACTION, (B,), np.int32), "reward": (BATCH_REWARD, (B,), np.float32),
                "terminal": (BATCH_TERMINAL, (B,), np.uint8), "next_state": (BATCH_NEXT_STATE, (ns, B), np.float32),
                "key": (BATCH_KEY, (B,), np.int64), "priority": (BATCH_PRIORITY, (B,), np.float32), "weight": (BATCH_WEIGHT, (B,), np.float32),
                "discount": (BATCH_DISCOUNT, (B,), np.float32), "horizon": (BATCH_HORIZON, (B,), np.int32)}
        out = {}
        for k, (f, shape, dt) in spec.items():
            a = np.empty(shape, dt, order="F")
            L.check(self.lib.b200rl_traj_batch_get(self.h, f, L.ptr(a), a.nbytes))
            out[k] = a
        return out

    def sampler_rng(self):
        a = np.empty((self.batch_size, 4), np.uint64)
        L.check(self.lib.b200rl_traj_batch_get(self.h, BATCH_RNG, L.ptr(a), a.nbytes))
        return a

    def update_priority(self, prio):
        prio = np.ascontiguousarray(prio, np.float32)
        L.check(self.lib.b200rl_traj_update_priority(self.h, L.ptr(prio), 0))

    def total_priority(self):
        v = C.c_float()
        L.check(self.lib.b200rl_traj_total_priority(self.h, C.byref(v)))
        return v.value


class DQNLearner:
    """DQNLearner / PrioritizedDQNLearner update on a device Trajectory."""

    def __init__(self, ctx, net, traj, cfg):
        self.ctx, self.lib, self.net, self.traj, self.cfg = ctx, ctx.lib, net, traj, cfg

    def update(self, want_stats=False):
        stats = np.zeros(4, np.float32) if want_stats else None
        L.check(self.lib.b200rl_dqn_update(self.net.h, self.traj.h, C.byref(self.cfg), L.ptr(stats)))
        return None if stats is None else dict(loss=stats[0], grad_norm=stats[1], mean_abs_td=stats[2], n_updates=int(stats[3]))

    def last_td(self):
        out = np.empty(self.traj.batch_size, np.float32)
        L.check(self.lib.b200rl_dqn_last_td(self.net.h, self.traj.h, L.ptr(out), out.size))
        return out


class InsertSampleRatioController:
    """InsertSampleRatioController(ratio, threshold) (ReinforcementLearningTrajectories 0.4, external; described in
    docs/src/How_to_implement_a_new_algorithm.md:108): counts insertions and sampled batches; a batch may be sampled once
    ``threshold`` insertions happened and while ``n_sampled <= (n_inserted - threshold) * ratio``.  One insertion = one
    push of a frame (all lanes), the batched counterpart of one ``push!``."""

    def __init__(self, ratio=1.0, threshold=1, n_inserted=0, n_sampled=0):
        self.ratio, self.threshold, self.n_inserted, self.n_sampled = float(ratio), int(threshold), int(n_inserted), int(n_sampled)

    def on_insert(self, n=1):
        self.n_inserted += n

    def on_sample(self):
        if self.n_inserted >= self.threshold and self.n_sampled <= (self.n_inserted - self.threshold) * self.ratio:
            self.n_sampled += 1
            return True
        return False


class _FusedEvaluation:
    """run(policy, env, StopAfterNSteps | StopAfterNEpisodes, hook) of a policy that does not train, on the fused evaluation kernel
    (b200rl_eval_run_episodes): the steps, episode log, streams and explorer step of the stage loop.  The library handle is created
    for the env on the first run and kept until the env or network changes or the policy is closed."""
    _eval = _eval_key = None

    def eval_handle(self, env):
        """the handle for runs on env, or None where the library refuses the pair or the policy has no device plan (the stage loop
        then keeps the run and raises its own errors)"""
        net, mode = self._eval_net_mode()
        if net is None:
            return None
        key = (env.h.value, net.h.value, mode)
        if self._eval is not None and self._eval_key == key:
            return self._eval
        self._close_eval()
        h = C.c_void_p()
        st = self.lib.b200rl_eval_create(net.h, env.h, mode, C.byref(h))
        if st in (L.ERR_UNSUPPORTED, L.ERR_INVALID):
            return None
        L.check(st)
        self._eval, self._eval_key = h, key
        return h

    def _close_eval(self):
        if self._eval is not None:
            if self.ctx.h:         # (a closed ctx took the handle's device buffers with it)
                self.lib.b200rl_eval_destroy(self._eval)
            self._eval = None

    def run_episodes(self, env, max_steps, budget):
        """At most max_steps env steps of run(policy, env, stop) on the fused path.  budget = k - cur for StopAfterNEpisodes(k): stops
        after the step at which the episodes counted reach it, as the stage loop does (a budget <= 0: one step); budget None for
        StopAfterNSteps: runs max_steps steps.  Returns (steps run, episodes they ended; 0 without a budget)."""
        h = self.eval_handle(env)
        if h is None:
            raise RuntimeError("the fused evaluation does not take this policy / env pair")
        ex = self._eval_explorer()
        steps, episodes = C.c_int64(), C.c_int64()
        L.check(self.lib.b200rl_eval_run_episodes(h, None if self._d_rng is None else C.c_void_p(self._d_rng), None if ex is None else C.byref(ex),
                                                  int(max_steps), _library_budget(budget), C.byref(steps), C.byref(episodes)))
        if ex is not None and hasattr(self.explorer, "step"):
            self.explorer.step = ex.step
        return steps.value, episodes.value


class QBasedPolicy(_FusedEvaluation, AbstractPolicy):
    """QBasedPolicy(learner = DQNLearner(...), explorer = EpsilonGreedyExplorer(...)) (q_based_policy.jl:13-49) on a batched
    env: ``plan`` = BatchExplorer over Q(state(env), .) — forward pass, schedule, draws and arg-max in one device call.

    ``explorer_rng``: (N, 4) uint64 raw Xoshiro states, one explorer stream per env.

    On a sharded ctx (rank r of G, ``ctx.rank_world()``) the N envs are global envs r N .. r N + N - 1: column i plans at explorer
    step ``step + r N + i`` and every plan advances the explorer by G N, as one BatchExplorer over the G N envs of all ranks would
    (DESIGN.md §3).  Every rank's explorer therefore holds the same step."""

    def __init__(self, ctx, learner, explorer, explorer_rng, n_envs):
        self.ctx, self.lib, self.learner, self.explorer, self.n = ctx, ctx.lib, learner, explorer, int(n_envs)
        rng = np.ascontiguousarray(explorer_rng, np.uint64).reshape(self.n, 4)
        self._d_rng = ctx.malloc(rng.nbytes)
        ctx.h2d(self._d_rng, rng)
        self._d_action = ctx.malloc(self.n * 4)
        # run() on its own (not inside an Agent) may hand whole stretches of env steps to run_episodes() when the explorer plans on
        # the device (eval_handle checks it per run)
        self.fusable = True

    def _eval_net_mode(self):
        return (self.learner.net if type(self.explorer) in DEVICE_EXPLORERS + (GreedyExplorer,) else None), 2

    def _eval_explorer(self):
        return self.explorer.as_struct() if type(self.explorer) in DEVICE_EXPLORERS else None

    def close(self):
        self._close_eval()
        for name in ("_d_rng", "_d_action"):
            p = getattr(self, name, None)
            if p:
                self.ctx.free(p)
                setattr(self, name, None)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def plan_device(self, env):
        """plan!(policy, env) leaving the actions on the device; returns the device pointer of the (N,) int32 actions."""
        net, ex = self.learner.net, self.explorer
        obs = C.c_void_p(env.obs_device_ptr())
        if hasattr(ex, "as_struct"):
            st = ex.as_struct()
            L.check(self.lib.b200rl_net_q_explore(net.h, obs, self.n, C.c_void_p(self._d_rng), C.byref(st), C.c_void_p(self._d_action)))
            ex.advance(self.n * self.ctx.rank_world()[1])
        else:   # GreedyExplorer: findmax, no draw
            L.check(self.lib.b200rl_net_q_act(net.h, obs, self.n, None, 0.0, C.c_void_p(self._d_action)))
        return self._d_action

    def plan(self, env):
        self.plan_device(env)
        return FusedAction("policy")

    def act_fused(self, env):
        env.act_(int(self._d_action))

    def explorer_rng(self):
        out = np.empty((self.n, 4), np.uint64)
        return self.ctx.d2h(out, self._d_rng)

    def set_explorer_rng(self, rng):
        self.ctx.h2d(self._d_rng, np.ascontiguousarray(rng, np.uint64).reshape(self.n, 4))

    def optimise(self, stage, trajectory=None):
        """optimise!(policy, stage, trajectory) = optimise!(policy.learner, stage, trajectory) (q_based_policy.jl:48-49);
        the DQN learner trains at the PostActStage."""
        if stage == PostActStage and trajectory is not None:
            while trajectory.controller.on_sample():
                self.learner.update()


EVAL_MODES = {"greedy": 0, "sample": 1}


class EvaluationPolicy(_FusedEvaluation, AbstractPolicy):
    """The network's policy without training: ``plan`` runs one forward pass on state(env) and leaves the actions on the
    device, ``act_fused`` hands them to ``env.act_``.  ``run(EvaluationPolicy(net, n), env, StopAfterNSteps(k), hook)`` is the
    stage protocol of :func:`evaluate`.

    mode "greedy": findmax of the logits / Q-values, mu of a Gaussian head (b200rl_net_act_greedy; no RNG).
    mode "sample": b200rl_net_act's sampler on one policy stream per env; ``rng``: (N, 4) uint64 raw Xoshiro states.
    A continuous action goes to the env as clamp(a, lo, hi) of its action space (through the host, like OnPolicyAgent's
    host-action path).

    Under run() with a hook that does nothing per step (EmptyHook, DeviceEpisodeStats, DeviceEpisodeLog) and StopAfterNSteps or
    StopAfterNEpisodes, the loop runs on the fused evaluation kernel instead (run_episodes, b200rl_eval_run_episodes) with the
    stage loop's results; ``fusable = False`` keeps the stage loop."""

    def __init__(self, net, n, mode="greedy", rng=None):
        if mode not in EVAL_MODES:
            raise ValueError(f"mode must be one of {sorted(EVAL_MODES)}")
        if mode == "sample" and rng is None:
            raise ValueError('mode "sample" needs rng: (N, 4) uint64 policy streams')
        self.net, self.ctx, self.lib, self.n, self.mode = net, net.ctx, net.ctx.lib, int(n), mode
        self._d_action = self.ctx.malloc(self.n * 4)
        self._d_rng = None
        if mode == "sample":
            rng = np.ascontiguousarray(rng, np.uint64).reshape(self.n, 4)
            self._d_rng = self.ctx.malloc(rng.nbytes)
            self.ctx.h2d(self._d_rng, rng)
        self._host_act = None
        self.fusable = True     # run() may hand whole stretches of env steps to run_episodes()

    def _eval_net_mode(self):
        return self.net, EVAL_MODES[self.mode]

    def _eval_explorer(self):
        return None

    def close(self):
        self._close_eval()
        for name in ("_d_action", "_d_rng"):
            p = getattr(self, name, None)
            if p:
                self.ctx.free(p)
                setattr(self, name, None)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def plan_device(self, env):
        """plan!(policy, env) leaving the raw actions (int32 | float) on the device; returns their device pointer."""
        obs = C.c_void_p(env.obs_device_ptr())
        if self.mode == "greedy":
            L.check(self.lib.b200rl_net_act_greedy(self.net.h, obs, self.n, C.c_void_p(self._d_action), 1))
        else:
            L.check(self.lib.b200rl_net_act(self.net.h, obs, self.n, C.c_void_p(self._d_rng), C.c_void_p(self._d_action),
                                            None, None, None, 1))
        return self._d_action

    def plan(self, env):
        d = self.plan_device(env)
        if env.continuous:
            if self._host_act is None:
                self._host_act = np.empty(self.n, np.float32)
            lo, hi = env.action_space()
            return np.clip(self.ctx.d2h(self._host_act, d), np.float32(lo), np.float32(hi)).astype(env.act_dtype)
        return FusedAction("policy")

    def act_fused(self, env):
        env.act_(int(self._d_action))

    def rng_state(self):
        """the policy streams (N, 4) after the steps so far (mode "sample")"""
        out = np.empty((self.n, 4), np.uint64)
        return self.ctx.d2h(out, self._d_rng)


def evaluate(net, env, n_steps, max_episodes=1, mode="greedy", rng=None):
    """b200rl_evaluate: ``run(policy, env, StopAfterNSteps(n_steps))`` with the network's greedy or sampling policy, in one
    fused launch where the network allows it.  Forces a reset of every env first; the env's episode statistics advance as
    under ``run``.

    ``rng`` (mode "sample"): (N, 4) uint64 policy streams, advanced in place, or a device pointer (int) to them.
    Returns ``returns`` (K, N) float32 and ``lengths`` (K, N) int32 (the first K = max_episodes episodes of each env that
    end inside the window; slots no episode reaches hold NaN / -1) and ``counts`` (N,) int32 (episodes per env, may exceed K).
    Average over the envs with ``counts >= K`` to avoid the bias towards short episodes of a fixed window.

    ``net`` may also be a :class:`QBasedPolicy` (b200rl_evaluate_explore): its Q-network planned by its explorer on its explorer
    streams, exactly as ``run(policy, env, StopAfterNSteps(n_steps))`` would — the streams and the explorer's step advance
    (``explorer.advance(N * n_steps)``, ``N * G * n_steps`` on a sharded ctx of G ranks); ``mode`` and ``rng`` do not apply.  To evaluate without touching a training policy, build a
    second QBasedPolicy over the same learner with its own explorer and streams."""
    if isinstance(net, QBasedPolicy):
        return _evaluate_q_based(net, env, n_steps, max_episodes)
    if mode not in EVAL_MODES:
        raise ValueError(f"mode must be one of {sorted(EVAL_MODES)}")
    ctx, lib, n, K = net.ctx, net.ctx.lib, env.n, int(max_episodes)
    returns = np.full((K, n), np.nan, np.float32, order="F")
    lengths = np.full((K, n), -1, np.int32, order="F")
    counts = np.zeros(n, np.int32)
    d_rng, host_rng = None, None
    if rng is not None and not isinstance(rng, (int, np.integer)):
        host_rng = rng
        arr = np.ascontiguousarray(rng, np.uint64).reshape(n, 4)
        d_rng = ctx.malloc(arr.nbytes)
        ctx.h2d(d_rng, arr)
    elif rng is not None:
        d_rng = int(rng)
    cfg = L.EvalConfig(EVAL_MODES[mode], int(n_steps), K)
    try:
        L.check(lib.b200rl_evaluate(net.h, env.h, C.byref(cfg), None if d_rng is None else C.c_void_p(d_rng), L.ptr(returns),
                                    L.ptr(lengths), L.ptr(counts), 0))
        if host_rng is not None:
            out = np.empty((n, 4), np.uint64)
            ctx.d2h(out, d_rng)
            host_rng[...] = out.reshape(np.shape(host_rng))
    finally:
        if host_rng is not None:
            ctx.free(d_rng)
    return dict(returns=returns, lengths=lengths, counts=counts)


def _evaluate_q_based(policy, env, n_steps, max_episodes):
    ex = policy.explorer
    if type(ex) not in DEVICE_EXPLORERS + (GreedyExplorer,):
        raise TypeError(f"{type(ex).__name__} has no device explorer")
    ctx, lib, n, K = policy.ctx, policy.lib, env.n, int(max_episodes)
    returns = np.full((K, n), np.nan, np.float32, order="F")
    lengths = np.full((K, n), -1, np.int32, order="F")
    counts = np.zeros(n, np.int32)
    st = ex.as_struct() if type(ex) in DEVICE_EXPLORERS else None
    L.check(lib.b200rl_evaluate_explore(policy.learner.net.h, env.h, int(n_steps), K, None if st is None else C.byref(st),
                                        C.c_void_p(policy._d_rng), L.ptr(returns), L.ptr(lengths), L.ptr(counts), 0))
    if st is not None:
        ex.advance(n * policy.ctx.rank_world()[1] * int(n_steps))   # (= st.step - ex.step: BatchExplorer over every rank's columns)
    return dict(returns=returns, lengths=lengths, counts=counts)


# the explorers b200rl_replay_run plans with (b200rl_explorer kinds 0 / 1, 2, 3, 4); GreedyExplorer runs as ex = NULL
DEVICE_EXPLORERS = (EpsilonGreedyExplorer, EpsilonSpeedyExplorer, WeightedSoftmaxExplorer, GumbelSoftmaxExplorer)


class Agent(AbstractPolicy):
    """Agent(policy, trajectory) (agent_base.jl:18-66) for a device-resident replay trajectory: pushes the env's
    transition frames (state / action / reward / terminal never visit the host) and lets the policy's learner train
    whenever the trajectory's controller allows a batch.

    Episode starts (the PreEpisodeStage push of agent_base.jl:45-47): run() announces every forced reset with a PreEpisodeStage
    push -> every lane gets an episode-start frame (so re-entering run() on a filled trajectory is fine: the entry straddling the
    reset exists and is not sampleable, exactly EpisodesBuffer's bookkeeping).  Episodes that end inside the loop: with the env's
    in-kernel auto-reset the trajectory writes the episode-start frame itself (the terminal step's observation already is the new
    episode's first state); with soft resets (auto_reset = False) the lanes whose last transition was terminal get the post-reset
    observation at the next PreActStage."""

    def __init__(self, policy, trajectory, host_actions=False):
        self.policy, self.trajectory, self.host_actions = policy, trajectory, host_actions
        if not hasattr(trajectory, "controller"):
            trajectory.controller = InsertSampleRatioController()
        self._host_act = None
        # run() may hand whole stretches of the loop to run_replay_episodes (b200rl_replay_run_episodes): a DQN learner behind one of
        # the device explorers (epsilon-greedy, speedy, weighted / Gumbel softmax, greedy) whose actions stay on the device.  The env's side is
        # checked per run (replay_supported).
        self.fusable = (not host_actions and isinstance(policy, QBasedPolicy) and isinstance(policy.learner, DQNLearner)
                        and type(policy.explorer) in DEVICE_EXPLORERS + (GreedyExplorer,))
        self._replay, self._replay_key = None, None

    def close(self):
        if getattr(self, "_replay", None):
            self.policy.lib.b200rl_replay_destroy(self._replay)
            self._replay = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- device agent loop ----------------------------------------------------------------------
    def replay_supported(self, env):
        """The env side of the device loop: in-kernel auto-reset, Float32 observations (a Float32 env, or a Float64 one behind
        set_state_float32), a discrete action space, <= 4 observations, and
        the trajectory's controller is an InsertSampleRatioController.  A sharded ctx needs the peer exchange attached or an NCCL
        communicator (refused by create otherwise)."""
        t, lr = self.trajectory, self.policy.learner
        return (self.fusable and env.auto_reset and (env.T is np.float32 or env.state_f32) and not env.continuous and env.kind != L.ENV_ACROBOT
                and type(t.controller) is InsertSampleRatioController and t.batch_size > 0 and t.lanes == env.n and t.ns == lr.net.n_in
                and lr.net.n_in == _NOBS.get(env.kind) and self._handle(env) is not None)

    def _handle(self, env):
        pol, lr = self.policy, self.policy.learner
        key = (env.h.value, lr.net.h.value, self.trajectory.h.value, bytes(lr.cfg))
        if self._replay is not None and self._replay_key == key:
            return self._replay
        self.close()
        h = C.c_void_p()
        st = pol.lib.b200rl_replay_create(pol.ctx.h, lr.net.h, env.h, self.trajectory.h, C.byref(lr.cfg), C.byref(h))
        if st in (L.ERR_UNSUPPORTED, L.ERR_INVALID):
            return None            # e.g. a sharded ctx without an exchange: the stage loop keeps running the agent (and raises its own errors)
        L.check(st)
        self._replay, self._replay_key = h, key
        return h

    def run_replay(self, env, n_steps, want_stats=False):
        """n_steps x {plan!, act!, push!, optimise!} of the stage protocol on the device (b200rl_replay_run): the same
        transitions, updates, streams and counters.  Returns the last update's {loss, grad_norm, mean_abs_td, n_updates}
        (want_stats, synchronises) or None.  On a sharded ctx every rank calls it with the same n_steps, controller and explorer
        (the explorer advances by N * world per step); loss and grad_norm are global, mean_abs_td is the rank's own."""
        pol, c = self.policy, self.trajectory.controller
        h = self._handle(env)
        ex = pol.explorer.as_struct() if type(pol.explorer) in DEVICE_EXPLORERS else None
        ctl = L.InsertSampleRatio(c.ratio, c.threshold, c.n_inserted, c.n_sampled)
        stats = np.full(4, np.nan, np.float32) if want_stats else None
        L.check(pol.lib.b200rl_replay_run(h, C.c_void_p(pol._d_rng), None if ex is None else C.byref(ex), C.byref(ctl), int(n_steps),
                                          L.ptr(stats)))
        if ex is not None and hasattr(pol.explorer, "step"):
            pol.explorer.step = ex.step
        c.n_inserted, c.n_sampled = ctl.n_inserted, ctl.n_sampled
        if stats is None or np.isnan(stats[3]):
            return None
        return dict(loss=stats[0], grad_norm=stats[1], mean_abs_td=stats[2], n_updates=int(stats[3]))

    def run_replay_episodes(self, env, max_steps, budget, want_stats=False):
        """At most max_steps env steps of run(agent, env, stop) on the device (b200rl_replay_run_episodes): the steps, updates,
        streams and counters of the stage loop.  budget = k - cur for StopAfterNEpisodes(k): stops after the step at which the
        episodes counted reach it (a budget <= 0: one step).  budget None for StopAfterNSteps: runs max_steps steps, as run_replay
        does.  Returns (steps run, episodes they ended[, last update's stats or None])."""
        pol, c = self.policy, self.trajectory.controller
        h = self._handle(env)
        ex = pol.explorer.as_struct() if type(pol.explorer) in DEVICE_EXPLORERS else None
        ctl = L.InsertSampleRatio(c.ratio, c.threshold, c.n_inserted, c.n_sampled)
        stats = np.full(4, np.nan, np.float32) if want_stats else None
        steps, episodes = C.c_int64(), C.c_int64()
        L.check(pol.lib.b200rl_replay_run_episodes(h, C.c_void_p(pol._d_rng), None if ex is None else C.byref(ex), C.byref(ctl),
                                                   int(max_steps), _library_budget(budget), L.ptr(stats), C.byref(steps),
                                                   C.byref(episodes)))
        if ex is not None and hasattr(pol.explorer, "step"):
            pol.explorer.step = ex.step
        c.n_inserted, c.n_sampled = ctl.n_inserted, ctl.n_sampled
        if not want_stats:
            return steps.value, episodes.value
        st = None if np.isnan(stats[3]) else dict(loss=stats[0], grad_norm=stats[1], mean_abs_td=stats[2], n_updates=int(stats[3]))
        return steps.value, episodes.value, st

    def graph_active(self):
        v = C.c_int()
        if self._replay is None:
            return False
        L.check(self.policy.lib.b200rl_replay_graph_active(self._replay, C.byref(v)))
        return bool(v.value)

    def push(self, stage, env, action=None):
        if stage == PreEpisodeStage:
            self.trajectory.push_env(env, first_state_only=True)         # push!(trajectory, (state = state(env),)) for every lane
        elif stage == PreActStage:
            if not getattr(env, "auto_reset", True):
                self.trajectory.push_env(env, first_state_only=2)        # lanes that were soft-reset since their terminal transition
        elif stage == PostActStage:
            self.trajectory.push_env(env)                                # (state = s', action, reward, terminal)
            self.trajectory.controller.on_insert(1)

    def plan(self, env):
        if self.host_actions:   # the reference's stage protocol: the action visits the host, the run loop calls act!(env, a)
            d = self.policy.plan_device(env)
            if self._host_act is None:
                self._host_act = np.empty(self.policy.n, np.int32)
            return self.policy.ctx.d2h(self._host_act, d)
        return self.policy.plan(env)

    def act_fused(self, env):
        self.policy.act_fused(env)

    def optimise(self, stage):
        self.policy.optimise(stage, self.trajectory)
