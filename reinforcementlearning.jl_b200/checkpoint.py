"""Checkpoint / resume of a device-resident run (SURVEY §8f-4).  The reference saves `agent` / `env` objects from a hook with
JLD2 (docs/src/How_to_use_hooks.md:124-167: `DoEveryNSteps(n) do t, agent, env; JLD2.@save ...`); here the state lives behind
opaque handles, so the hook copies it out through the C ABI — `b200rl_net_get`, `b200rl_env_get`, `b200rl_onpolicy_get` /
`b200rl_onpolicy_export_state` — into a flat dict of numpy arrays (np.savez-able), and `restore` puts it back into freshly
constructed objects of the same shapes.  A restored run continues bit for bit (tests/test_zz_dqn_agent_gpu.py), at a rollout
boundary or in the middle of a rollout.  Host-side configuration (env kind / params, network shape, hyper-parameters) is the
constructor's business, exactly as `PPOPolicy(...)` is rebuilt before `Flux.loadmodel!` in the reference.

`checkpoint` / `restore` cover on-policy runs (env + actor-critic net + OnPolicyAgent).  Replay runs (`Agent(QBasedPolicy, Trajectory)`)
go through `checkpoint_replay` / `restore_replay`, which add the Q-network's update counter (the target-sync phase), the ring with its
per-lane bookkeeping and sum tree, the sampler / explorer streams, the explorer's step and the controller's counters.  The
trajectory's n-step setting (`Trajectory(..., n_step, gamma)`, the NStepBatchSampler) is configuration, not state: it is not
saved, and the restored trajectory must be constructed with the same one."""
import numpy as np

from . import _lib as L
from . import learners as R
from .core import PostActStage
from .envs import _NOBS, _NS

_ENV_FIELDS = {"state": L.FIELD_STATE, "obs": L.FIELD_OBS, "reward": L.FIELD_REWARD, "flags": L.FIELD_FLAGS, "t": L.FIELD_T,
               "rng": L.FIELD_RNG, "action": L.FIELD_ACTION, "episode_return": L.FIELD_EPISODE_RETURN,
               "episode_stats": L.FIELD_EPISODE_STATS}
_NET_FIELDS = {"params": R.NET_PARAMS, "adam_m": R.NET_M, "adam_v": R.NET_V, "beta_t": R.NET_BETA_T}
_ROLLOUT_FIELDS = {"states": R.ROLL_STATE, "actions": R.ROLL_ACTION, "logp": R.ROLL_LOGP, "rewards": R.ROLL_REWARD,
                   "terminals": R.ROLL_TERMINAL, "values": R.ROLL_VALUE}


def _env_get(env, field):
    n = env.n
    spec = {
        L.FIELD_STATE: ((_NS[env.kind], n), env.T), L.FIELD_OBS: ((_NOBS[env.kind], n), env.T),
        L.FIELD_REWARD: ((n,), env.T), L.FIELD_FLAGS: ((n,), np.uint8), L.FIELD_T: ((n,), np.int32), L.FIELD_RNG: ((n, 4), np.uint64),
        L.FIELD_ACTION: ((n,), env.act_dtype), L.FIELD_EPISODE_RETURN: ((n,), np.float32),
        L.FIELD_EPISODE_STATS: ((4,), np.float64),
    }[field]
    order = "C" if field == L.FIELD_RNG else "F"
    return env._get(field, spec[0], spec[1], order=order)


def checkpoint(env=None, net=None, agent=None):
    """Copy the device state out.  Returns {name: ndarray}; keys are prefixed env/ net/ agent/."""
    out = {}
    if env is not None:
        for name, f in _ENV_FIELDS.items():
            out["env/" + name] = _env_get(env, f)
    if net is not None:
        for name, w in _NET_FIELDS.items():
            out["net/" + name] = net.get(w)
        if net.is_q:
            out["net/target"] = net.get(R.NET_TARGET)
    if agent is not None:
        c3 = np.zeros(3, np.int64)
        L.check(agent.lib.b200rl_onpolicy_export_state(agent.h, L.ptr(c3)))
        out["agent/counters"] = c3
        out["agent/policy_rng"] = agent.rollout(R.ROLL_RNG)
        if c3[0] > 0:   # mid-rollout: the columns filled so far travel too
            for name, f in _ROLLOUT_FIELDS.items():
                out["agent/" + name] = agent.rollout(f)
    return out


def restore(ckpt, env=None, net=None, agent=None):
    """Put a checkpoint back into freshly constructed objects of the same shapes.  Order matters for the optimiser: the agent's
    constructor re-arms beta^t on a net that has not stepped yet, so the net's state goes in after the agent exists."""
    if env is not None:
        for name, f in _ENV_FIELDS.items():
            arr = ckpt["env/" + name]
            if name == "obs" and env.device_ptr(L.FIELD_OBS) == env.device_ptr(L.FIELD_STATE):
                continue                                    # the observation is the state (one buffer)
            a = np.ascontiguousarray(arr) if name == "rng" else np.asfortranarray(arr)
            L.check(env.lib.b200rl_env_set(env.h, f, L.ptr(a), a.nbytes))
    if net is not None:
        for name, w in _NET_FIELDS.items():
            net.set(w, ckpt["net/" + name])
        if net.is_q and "net/target" in ckpt:
            net.set(R.NET_TARGET, ckpt["net/target"])
    if agent is not None:
        c3 = np.ascontiguousarray(ckpt["agent/counters"], np.int64)
        rng = np.asfortranarray(ckpt["agent/policy_rng"], np.uint64)      # (4, N): four words per env, contiguous
        L.check(agent.lib.b200rl_onpolicy_set(agent.h, R.ROLL_RNG, L.ptr(rng), rng.nbytes))
        if c3[0] > 0:
            for name, f in _ROLLOUT_FIELDS.items():
                a = np.asfortranarray(ckpt["agent/" + name])
                L.check(agent.lib.b200rl_onpolicy_set(agent.h, f, L.ptr(a), a.nbytes))
        L.check(agent.lib.b200rl_onpolicy_import_state(agent.h, L.ptr(c3)))
        agent._t = int(c3[0])
        agent.n_updates = int(c3[1])


def checkpoint_replay(env, net, agent):
    """State of a replay run: env, Q-network (+ target, Adam state, update counter), trajectory ring, explorer, controller."""
    out = checkpoint(env=env, net=net)
    out["net/step"] = np.array([net.step_count()], np.int64)
    for k, v in agent.trajectory.export_state().items():
        out["traj/" + k] = v
    pol = agent.policy
    out["policy/explorer_rng"] = pol.explorer_rng()
    out["policy/explorer_step"] = np.array([getattr(pol.explorer, "step", 0)], np.int64)
    return out


def restore_replay(ckpt, env, net, agent):
    restore(ckpt, env=env, net=net)
    net.set_step_count(int(ckpt["net/step"][0]))
    agent.trajectory.import_state({k[5:]: v for k, v in ckpt.items() if k.startswith("traj/")})
    pol = agent.policy
    pol.set_explorer_rng(ckpt["policy/explorer_rng"])
    if hasattr(pol.explorer, "step"):
        pol.explorer.step = int(ckpt["policy/explorer_step"][0])


def save(path, ckpt):
    """np.savez (keys with '/' are legal archive member names)."""
    np.savez(path, **ckpt)


def load(path):
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


class CheckpointEveryNSteps:
    """The hook of docs/src/How_to_use_hooks.md:124-167 (`DoEveryNSteps(n) do t, agent, env ... save`): every `n` env steps
    write `<prefix>_<t>.npz`.  per_step is True, so run() steps through the stages while this hook is attached."""
    per_step = True

    def __init__(self, n, prefix, net=None):
        self.n, self.prefix, self.net, self.t, self.paths = int(n), prefix, net, 0, []

    def push(self, stage, policy, env):
        if stage != PostActStage:
            return
        self.t += 1
        if self.t % self.n == 0:
            path = f"{self.prefix}_{self.t}.npz"
            if hasattr(policy, "trajectory"):      # replay Agent: the ring, explorer and controller travel too
                save(path, checkpoint_replay(env, self.net or policy.policy.learner.net, policy))
            else:
                save(path, checkpoint(env=env, net=self.net or getattr(policy, "net", None), agent=policy if hasattr(policy, "rollout") else None))
            self.paths.append(path)
