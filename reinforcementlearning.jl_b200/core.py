"""Host mirror of the reference's run loop, stages, hooks and stop conditions for a batched
env (RLCore/src/core/run.jl:22-78, stages.jl:13-37, hooks.jl, stop_conditions.jl,
reset_conditions.jl).  This is the control plane the Julia glue (julia/B200RL.jl) keeps in
Julia; it is restated in Python only so the path can be driven and tested without Julia.

Control flow = the historical ``_run(policy, env::MultiThreadEnv, ...)`` (SURVEY §3.4): no
episode stages, ``is_terminated(env)`` is a vector, finished sub-envs are soft-reset at the
top of every iteration (or inside the step kernel when ``env.auto_reset``)."""
import time

import numpy as np

# ---- debug tracing (TimerOutputs in the reference: `const timer`, ReinforcementLearningCore.jl:17-18; every call of `_run` sits in
#      `@timeit_debug timer "<label>"`, run.jl:46-72; off until `TimerOutputs.enable_debug_timings(RLCore)`, docs/src/tips.md:21-23)
class TimerOutput(dict):
    """label -> [number of calls, total seconds]"""

    def __str__(self):
        rows = sorted(self.items(), key=lambda kv: -kv[1][1])
        return "\n".join(f"{label:36s} {n:8d} calls {1e3 * sec:10.3f} ms" for label, (n, sec) in rows)


timer = TimerOutput()
_debug_timings = False


def enable_debug_timings(on=True):
    """TimerOutputs.enable_debug_timings / disable_debug_timings for run().  Wall-clock around each stage call; kernel time
    proper is measured on the device (Context.timer_start / timer_stop_ms, ncu)."""
    global _debug_timings
    _debug_timings = bool(on)


def _timed(label, fn, *args, **kw):
    if not _debug_timings:
        return fn(*args, **kw)
    t0 = time.perf_counter()
    try:
        return fn(*args, **kw)
    finally:
        rec = timer.setdefault(label, [0, 0.0])
        rec[0] += 1
        rec[1] += time.perf_counter() - t0


# stages (stages.jl:13-28)
PreExperimentStage, PostExperimentStage = "PreExperimentStage", "PostExperimentStage"
PreEpisodeStage, PostEpisodeStage = "PreEpisodeStage", "PostEpisodeStage"
PreActStage, PostActStage = "PreActStage", "PostActStage"


class AbstractHook:
    def push(self, stage, policy, env):  # Base.push!(hook, stage, policy, env) (hooks.jl:32-35)
        pass

    def __add__(self, other):  # ComposedHook via `+`, flattening composed operands (hooks.jl:40-43)
        left = self.hooks if isinstance(self, ComposedHook) else (self,)
        right = other.hooks if isinstance(other, ComposedHook) else (other,)
        return ComposedHook(*left, *right)


class EmptyHook(AbstractHook):
    per_step = False


class ComposedHook(AbstractHook):
    def __init__(self, *hooks):
        self.hooks = tuple(hooks)

    @property
    def per_step(self):  # the composed hook is stage-free only when every member is
        return any(getattr(h, "per_step", True) for h in self.hooks)

    def __getitem__(self, i):  # Base.getindex(hook::ComposedHook, inds...) (hooks.jl:61)
        return self.hooks[i]

    def push(self, stage, policy, env):
        for h in self.hooks:
            h.push(stage, policy, env)


class BatchStepsPerEpisode(AbstractHook):
    """hooks.jl:202-231 — per-env episode lengths from the vector ``is_terminated(env)``."""

    def __init__(self, batchsize):
        self.steps = [[] for _ in range(batchsize)]
        self.step = np.zeros(batchsize, dtype=np.int64)

    def __getitem__(self, _):
        return self.steps

    def push(self, stage, policy, env):
        if stage != PostActStage:
            return
        term = env.is_terminated()
        self.step += 1
        for i in np.nonzero(term)[0]:
            self.steps[i].append(int(self.step[i]))
            self.step[i] = 0


class TotalBatchRewardPerEpisode(AbstractHook):
    """Batched TotalRewardPerEpisode (hooks.jl:146-173): per-env running reward, pushed on termination."""

    def __init__(self, batchsize):
        self.rewards = [[] for _ in range(batchsize)]
        self.reward = np.zeros(batchsize, dtype=np.float64)

    def push(self, stage, policy, env):
        if stage != PostActStage:
            return
        self.reward += env.reward()
        for i in np.nonzero(env.is_terminated())[0]:
            self.rewards[i].append(float(self.reward[i]))
            self.reward[i] = 0.0


class DeviceEpisodeStats(AbstractHook):
    """Device-side reduction of the two hooks above (SURVEY §8f-3): no per-step D2H copy; reads
    four numbers at the end of the experiment."""
    per_step = False   # nothing happens at the Pre/PostAct stages: run() may execute many env steps per launch

    def __init__(self):
        self.stats = None

    def push(self, stage, policy, env):
        if stage == PreExperimentStage:
            env.episode_stats(reset=True)
        elif stage == PostExperimentStage:
            self.stats = env.episode_stats()


class DeviceEpisodeLog(AbstractHook):
    """TotalBatchRewardPerEpisode + BatchStepsPerEpisode kept on the device (b200rl_env_episode_log): ``rewards`` and ``steps`` are
    per-env lists with the meaning of those two hooks' fields, but no step copies anything to the host, so run() keeps its fused
    paths.  Each env logs into a ring of ``capacity`` records; run() splits the fused loop into windows of at most ``capacity``
    env steps and flushes after each (an episode lasts at least one step, so no ring can overflow), the stage loop flushes every
    ``capacity`` PostActStage pushes.  A flush is read one flush later (or at PostExperimentStage), so the host never waits inside
    a window; the records are kept as arrays and turned into the lists when ``rewards`` / ``steps`` are read.  The returns are the
    env's Float32 step-order sums (FIELD_EPISODE_RETURN); evaluate() is not logged.  On a sharded ctx the records carry the
    global env index rank * N + i; the lists are indexed by the local env i.

    The ring stays attached to the env after the run and the two pinned host buffers stay with the hook, so the next run of the
    same hook (or of another DeviceEpisodeLog of the same size on that env, which takes them over) allocates nothing and keeps the
    captured graphs; attaching again empties the ring.  ``close()`` detaches the ring and frees the buffers.  One env is recorded by
    one hook at a time: a second hook that starts while the first is inside a run is refused."""
    per_step = False

    def __init__(self, batchsize, capacity=64):
        if capacity < 1:
            raise ValueError("capacity must be >= 1")
        self._lists = ([[] for _ in range(batchsize)], [[] for _ in range(batchsize)])
        self.capacity = int(capacity)
        self._env = None
        self._bufs = []
        self._chunks = []        # record arrays read from the device, in flush order
        self._pending = None     # index of the buffer whose flush has not been read yet
        self._acts = 0           # PostActStage pushes since the last flush (stage loop)
        self._running = False

    @property
    def rewards(self):
        return self._materialize()[0]

    @property
    def steps(self):
        return self._materialize()[1]

    def __getitem__(self, _):    # getindex of TotalRewardPerEpisode and BatchStepsPerEpisode (hooks.jl:160, 207)
        return self._materialize()

    def push(self, stage, policy, env):
        if stage == PreExperimentStage:
            self._attach(env)
        elif stage == PostActStage:
            self._acts += 1
            if self._acts >= self.capacity:
                self.flush()
        elif stage == PostExperimentStage:
            try:
                self.flush()
                self._read()
            finally:
                self._running = False

    def _attach(self, env):
        owner = getattr(env, "_episode_log_hook", None)
        if owner is not None and owner is not self:
            if owner._running:
                raise RuntimeError("another DeviceEpisodeLog is recording this env")
            owner._hand_over(self, env)
        elif self._env is not None and self._env is not env:
            self.close()
        records = env.n * self.capacity
        if self._bufs and self._records != records:
            self._free_buffers()
        env.episode_log(self.capacity)          # (the same K again: the same ring, emptied)
        env._episode_log_hook = self
        self._env, self._records = env, records
        self._base = env.ctx.rank_world()[0] * env.n
        if not self._bufs:
            self._bufs, self._bufs_ctx = [env.episode_log_buffer(records) for _ in range(2)], env.ctx
        self._next, self._pending, self._acts, self._running = 0, None, 0, True

    def _hand_over(self, other, env):
        """an idle hook lets `other` record `env`: its buffers go along when they have the right size"""
        if self._bufs and self._records == env.n * other.capacity and not other._bufs:
            other._bufs, other._records, other._bufs_ctx, self._bufs = self._bufs, self._records, self._bufs_ctx, []
        self._free_buffers()
        self._env = None

    def _free_buffers(self):
        for _, addr in self._bufs:
            self._bufs_ctx.host_free(addr)
        self._bufs = []

    def close(self):
        """detach the ring from the env and free the pinned buffers"""
        env, self._env, self._running = self._env, None, False
        if env is not None and getattr(env, "_episode_log_hook", None) is self:
            env._episode_log_hook = None
            if env.h:
                env.episode_log(0)
        self._free_buffers()

    def __del__(self):
        try:
            if self._bufs and self._bufs_ctx.h:
                self.close()
        except Exception:
            pass

    def flush(self):
        """Hand the records of the window that just ended to the host buffer not being read, then read the previous flush."""
        if self._env is None:
            return
        try:
            _, addr = self._bufs[self._next]
            self._env.episode_log_flush(addr, self._records)
            self._read()
        except BaseException:
            self._pending, self._running = None, False
            raise
        self._pending, self._next, self._acts = self._next, 1 - self._next, 0

    def _read(self):
        if self._pending is None:
            return
        arr, addr = self._bufs[self._pending]
        self._pending = None
        rec = self._env.episode_log_read(arr, addr)
        if len(rec):
            self._chunks.append(rec)

    def _materialize(self):
        if self._chunks:
            rec = np.concatenate(self._chunks)
            self._chunks = []
            env = rec["env"] - self._base
            rec = rec[np.argsort(env, kind="stable")]   # by env; the flushes are in time order, so episodes stay in order
            ends = np.cumsum(np.bincount(env, minlength=len(self._lists[0])))
            rets, lens = rec["ret"].tolist(), rec["len"].tolist()
            start = 0
            for i, end in enumerate(ends.tolist()):
                if end > start:
                    self._lists[0][i].extend(rets[start:end])
                    self._lists[1][i].extend(lens[start:end])
                start = end
        return self._lists


def _episode_log_window(hook):
    """(the DeviceEpisodeLog hooks of `hook`, the longest window in env steps they allow or None)"""
    hooks = hook.hooks if isinstance(hook, ComposedHook) else (hook,)
    logs = [h for h in hooks if isinstance(h, DeviceEpisodeLog)]
    return logs, (min(h.capacity for h in logs) if logs else None)


def _flush(logs):
    for h in logs:
        h.flush()


def _run_fused(policy, env, stop_condition, hook):
    """StopAfterNSteps or StopAfterNEpisodes on the fused paths: windows of at most the episode log's capacity, each one library call
    (b200rl_*_run_episodes, b200rl_eval_run_episodes) followed by a flush.  The library cuts a window into stretches; a StopAfterNEpisodes window stops at the
    crossing of the remaining budget, a StopAfterNSteps one (no budget) may end early at the end of a rollout.  Returns False
    (nothing run) where the stage loop keeps the run: an episode count on a sharded ctx (the stop would count the episodes of every
    rank), a replay agent the device loop does not take, an evaluation policy / env pair the fused evaluation does not take."""
    episodes = isinstance(stop_condition, StopAfterNEpisodes)
    if episodes and env.ctx.rank_world()[1] > 1:
        return False
    if hasattr(policy, "run_replay"):
        if not policy.replay_supported(env):
            return False
        step = lambda n, budget: policy.run_replay_episodes(env, n, budget)
    elif hasattr(policy, "eval_handle"):       # EvaluationPolicy, a QBasedPolicy on its own
        if policy.eval_handle(env) is None:
            return False
        step = lambda n, budget: policy.run_episodes(env, n, budget)
    else:
        step = policy.run_episodes
    logs, window = _episode_log_window(hook)
    window = window or (1 << 62)
    while True:
        if episodes:
            _, n = step(window, stop_condition.episode - stop_condition.cur)
            stop_condition.cur += n
            is_stop = stop_condition.cur >= stop_condition.episode
        else:
            steps, _ = step(min(window, stop_condition.remaining()), None)
            is_stop = stop_condition.advance(steps)
        _flush(logs)
        if is_stop:
            return True


class TimePerStep(AbstractHook):
    """hooks.jl:243-262 (wall-clock per loop iteration)."""

    def __init__(self, max_steps=100):
        self.times = []
        self.max_steps = max_steps
        self.t = time.perf_counter()

    def push(self, stage, policy, env):
        if stage == PostActStage:
            now = time.perf_counter()
            self.times.append(now - self.t)
            self.times = self.times[-self.max_steps:]
            self.t = now


class DoEveryNSteps(AbstractHook):
    """hooks.jl:270-288."""

    def __init__(self, f, n=1, t=0):
        self.f, self.n, self.t = f, n, t

    def push(self, stage, policy, env):
        if stage == PostActStage:
            self.t += 1
            if self.t % self.n == 0:
                self.f(self.t, policy, env)


class DoOnExit(AbstractHook):
    """hooks.jl DoOnExit: call f(policy, env) at the PostExperimentStage."""

    def __init__(self, f):
        self.f = f

    def push(self, stage, policy, env):
        if stage == PostExperimentStage:
            self.f(policy, env)


# ---- stop conditions (stop_conditions.jl) -------------------------------------------------
class StopIfAny:
    """stop_conditions.jl:13-27: every condition is checked (no short circuit), the results are reduced by any."""

    def __init__(self, *stop_conditions):
        self.stop_conditions = stop_conditions

    def check(self, policy, env):
        return any([s.check(policy, env) for s in self.stop_conditions])


class StopIfAll:
    """stop_conditions.jl:29-38."""

    def __init__(self, *stop_conditions):
        self.stop_conditions = stop_conditions

    def check(self, policy, env):
        return all([s.check(policy, env) for s in self.stop_conditions])


class StopAfterNoImprovement:
    """stop_conditions.jl:120-165: fn() is monitored whenever an episode ended (batched: any sub-env terminated);
    true once it failed to improve by more than delta for `patience` consecutive checks."""

    def __init__(self, fn, patience, delta=0.0):
        self.fn, self.patience, self.delta = fn, int(patience), delta
        self.peak, self.counter = float("-inf"), 1

    def check(self, policy, env):
        if not np.any(env.is_terminated()):
            return False
        val = self.fn()
        if self.delta < val - self.peak:
            self.counter = 1
            self.peak = max(val, self.peak)
            return False
        self.counter += 1
        return self.counter > self.patience


class StopAfterNSteps:
    """stop_conditions.jl:40-76: true on its n-th check (n loop iterations = n*N env-steps)."""

    def __init__(self, step, cur=1):
        self.step, self.cur = step, cur

    def remaining(self):
        """loop iterations left before check() returns true"""
        return max(1, self.step - self.cur + 1)

    def advance(self, n):
        """n loop iterations at once (the fused rollout): true when the n-th of them would have stopped the loop"""
        self.cur += n
        return self.cur > self.step

    def check(self, policy, env):
        res = self.cur >= self.step
        self.cur += 1
        return res


class StopAfterNEpisodes:
    """stop_conditions.jl:82-118, batched: counts every finished sub-env episode."""

    def __init__(self, episode, cur=0):
        self.episode, self.cur = episode, cur

    def check(self, policy, env):
        self.cur += int(np.count_nonzero(env.is_terminated()))
        return self.cur >= self.episode


class StopAfterNSeconds:
    """stop_conditions.jl:203-224."""

    def __init__(self, budget):
        self.deadline = time.time() + budget

    def check(self, policy, env):
        return time.time() > self.deadline


# ---- reset conditions (reset_conditions.jl) ----------------------------------------------------
class ResetIfEnvTerminated:
    """reset_conditions.jl:5-12.  For the batched env it never fires: finished sub-envs are reset individually (soft reset /
    in-kernel auto-reset), never the whole batch."""

    def check(self, policy, env):
        return False


class ResetAfterNSteps:
    """reset_conditions.jl:14-36: true on the (n + 1)-th check, i.e. after n steps; the whole batch is then force-reset."""

    def __init__(self, n):
        self.t, self.n = 0, int(n)

    def check(self, policy, env):
        stop = self.t >= self.n
        self.t += 1
        if stop:
            self.t = 0
        return stop


class StopSignal:
    """stop_conditions.jl:185-200."""

    def __init__(self):
        self.is_stop = False

    def check(self, policy, env):
        return self.is_stop


# ---- policies -----------------------------------------------------------------------------
class AbstractPolicy:
    def plan(self, env):  # RLBase.plan!(policy, env)
        raise NotImplementedError

    def push(self, stage, env, action=None):  # Base.push!(policy, stage, env[, action])
        pass

    def optimise(self, stage):  # RLBase.optimise!(policy, stage)
        pass


class FusedAction:
    """Token returned by a policy whose action selection is fused into the env kernel."""

    def __init__(self, kind):
        self.kind = kind


class RandomPolicy(AbstractPolicy):
    """RandomPolicy() with the reference default of sharing the env's RNG stream
    (random_policy.jl:18-32): the draw happens inside the step kernel (K2)."""

    def plan(self, env):
        return FusedAction("random")


class Experiment:
    """Experiment(policy, env, stop_condition, hook) (run.jl:8-20); ``run(experiment)`` runs it and returns it."""

    def __init__(self, policy, env, stop_condition, hook):
        self.policy, self.env, self.stop_condition, self.hook = policy, env, stop_condition, hook


def run(policy, env=None, stop_condition=None, hook=None, reset_condition=None):
    """Base.run(policy, env, stop_condition, hook[, reset_condition]) for a B200VecEnv (run.jl:22-78 with the
    MultiThreadEnv control flow).  Returns the hook (``run(experiment)`` returns the experiment)."""
    if isinstance(policy, Experiment):
        ex = policy
        run(ex.policy, ex.env, ex.stop_condition, ex.hook)
        return ex
    stop_condition = stop_condition or StopAfterNEpisodes(1)
    hook = hook or EmptyHook()
    reset_condition = reset_condition or ResetIfEnvTerminated()
    hook.push(PreExperimentStage, policy, env)
    policy.push(PreExperimentStage, env)
    env.reset_(is_force=True)  # run.jl:46
    policy.push(PreEpisodeStage, env)   # run.jl:47-49: every lane starts an episode (there is no per-lane episode stage in the batched loop)
    # Fused path: a device-resident agent (actions never visit the host), a hook that does nothing per step and a stop condition
    # that counts steps or episodes let whole stretches of the loop below run on the device, with the transitions, parameters,
    # statistics and stop step of stepping through the stages.
    is_stop = (getattr(policy, "fusable", False) and env.auto_reset and not getattr(hook, "per_step", True)
               and isinstance(stop_condition, (StopAfterNSteps, StopAfterNEpisodes)) and isinstance(reset_condition, ResetIfEnvTerminated)
               and _run_fused(policy, env, stop_condition, hook))

    def act(action):
        if isinstance(action, FusedAction):
            if action.kind == "random":
                env.act_random_()
            else:
                policy.act_fused(env)
        else:
            env.act_(action)

    while not is_stop:   # labels as in run.jl:46-72
        did_reset = False
        while reset_condition.check(policy, env):         # `while !check!(reset_condition, ...)` is evaluated again after the
            _timed("reset!", env.reset_, is_force=True)   # reset (run.jl:46,52): the reference leaves the episode loop and resets
            _timed("push!(policy) PreEpisodeStage", policy.push, PreEpisodeStage, env)
            did_reset = True
        if not did_reset and not env.auto_reset:
            _timed("reset!", env.reset_, is_force=False)  # soft reset of finished sub-envs
        _timed("push!(policy) PreActStage", policy.push, PreActStage, env)
        _timed("optimise! PreActStage", policy.optimise, PreActStage)
        _timed("push!(hook) PreActStage", hook.push, PreActStage, policy, env)
        action = _timed("plan!", policy.plan, env)
        _timed("act!", act, action)
        _timed("push!(policy) PostActStage", policy.push, PostActStage, env, action)
        _timed("optimise! PostActStage", policy.optimise, PostActStage)
        _timed("push!(hook) PostActStage", hook.push, PostActStage, policy, env)
        if stop_condition.check(policy, env):
            is_stop = True
    policy.push(PostExperimentStage, env)
    hook.push(PostExperimentStage, policy, env)
    env.check()
    return hook
