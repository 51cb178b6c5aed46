"""Throughput of run(agent, env, StopAfterNEpisodes(k)) on the fused paths (b200rl_onpolicy_run_episodes /
b200rl_replay_run_episodes) against StopAfterNSteps for the same number of env steps, on the H100.

Workloads:
  ppo-c2       bench.py's config c2: PPO on 65 536 CartPole envs, T = 32, 4 epochs x 4 minibatches, 4-64-64-2 actor and critic
  dqn-h64      bench_replay.py's lanes65536 loop: 65 536 CartPole lanes x 16 frames, prioritised, batch 4096, 4-64-64-2 Q-network,
               ratio 1

    python bench_stop_episodes.py [--ppo-episodes 2000000] [--dqn-episodes 3000000] [--reps 3] [--stage-steps 64] [--only NAME]
                                  [--out result.json]

Each workload builds two agents from the same seeds and warms both up (graphs captured).  Then, `reps` times, alternating: agent A
runs StopAfterNEpisodes(k) and reports how many env steps that took; agent B runs StopAfterNSteps for the same number of steps.
Host clock around runs that end in a device synchronise; medians of the env-step rates and their ratio (episodes / steps) are
reported.  The stage-loop rate is what StopAfterNEpisodes ran at before the fused calls existed: a third agent driven through the
stage loop (plan!, act!, push!, optimise! and a host copy of is_terminated per step) for --stage-steps steps, alternated with the
other two; its median is reported.  GPU name, power
limit and max SM clock are read in the same process.  After the timed runs the two agents must hold identical checkpoints.  Prints one JSON line; --out also writes it to a file."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_episode_log import C2, build_ppo, checkpoints_identical   # noqa: E402
from bench_evaluate import gpu_info   # noqa: E402
from bench_replay import WORKLOADS as REPLAY, build as build_replay   # noqa: E402


def env_steps(s):
    return s["env"].episode_stats()["env_steps"] // s["env"].n


def timed(pkg, ctx, s, stop):
    s0 = env_steps(s)
    ctx.sync()
    t0 = time.perf_counter()
    pkg.run(s["agent"], s["env"], stop, pkg.EmptyHook())
    ctx.sync()
    return time.perf_counter() - t0, env_steps(s) - s0


def zeroed_rollout(pkg, s):
    """rollout columns no run has written yet hold whatever the allocation held: zero them so that two agents compare equal there"""
    a = s["agent"]
    for f in range(6):
        z = np.zeros_like(a.rollout(f))
        pkg._lib.check(a.lib.b200rl_onpolicy_set(a.h, f, pkg._lib.ptr(z), z.nbytes))
    return s


def bench(pkg, ctx, name, make, k, warm_steps, reps, stage_steps, replay):
    ep, st = make(), make()
    for s in (ep, st):
        timed(pkg, ctx, s, pkg.StopAfterNSteps(warm_steps))
    timed(pkg, ctx, ep, pkg.StopAfterNEpisodes(max(1, k // 20)))       # (the episode path's first stretches, eagerly)
    timed(pkg, ctx, st, pkg.StopAfterNSteps(env_steps(ep) - env_steps(st)))
    n = ep["env"].n
    # the stage loop StopAfterNEpisodes took before: plan!, act!, push!, optimise! and a host copy of is_terminated per step
    stage = make()
    timed(pkg, ctx, stage, pkg.StopAfterNSteps(warm_steps))
    res = {"episodes": [], "steps": [], "stage": []}
    for _ in range(reps):
        dt, steps = timed(pkg, ctx, ep, pkg.StopAfterNEpisodes(k))
        res["episodes"].append(dict(sec=dt, steps=steps, rate=steps * n / dt))
        dt2, steps2 = timed(pkg, ctx, st, pkg.StopAfterNSteps(steps))
        assert steps2 == steps
        res["steps"].append(dict(sec=dt2, steps=steps2, rate=steps2 * n / dt2))
        dt3, steps3 = timed(pkg, ctx, stage, _Both(pkg.StopAfterNEpisodes(1 << 62), pkg.StopAfterNSteps(stage_steps)))
        res["stage"].append(dict(sec=dt3, steps=steps3, rate=steps3 * n / dt3))
    stage_rate = float(np.median([r["rate"] for r in res["stage"]]))
    # the two agents ran the same steps from the same seeds, one stopped by episodes and one by steps: the same state
    out = {"workload": name, "k": k, "reps": reps, "identical_checkpoints": bool(checkpoints_identical(pkg, ep, st, replay))}
    for key in ("episodes", "steps"):
        out[key] = {"env_steps_per_s": float(np.median([r["rate"] for r in res[key]])),
                    "env_steps_per_s_all": [round(r["rate"]) for r in res[key]], "steps": [r["steps"] for r in res[key]]}
    out["ratio_episodes_over_steps"] = out["episodes"]["env_steps_per_s"] / out["steps"]["env_steps_per_s"]
    out["stage_loop_episodes_env_steps_per_s"] = stage_rate
    out["speedup_over_stage_loop"] = out["episodes"]["env_steps_per_s"] / stage_rate
    for s in (ep, st, stage):
        for v in s.values():
            if hasattr(v, "close"):
                v.close()
    return out


class _Both:
    """StopAfterNEpisodes checked every step (its host copy of is_terminated), the loop bounded by a step count"""

    def __init__(self, episodes, steps):
        self.episodes, self.steps = episodes, steps

    def check(self, policy, env):
        return any([self.episodes.check(policy, env), self.steps.check(policy, env)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ppo-episodes", type=int, default=2_000_000)
    ap.add_argument("--dqn-episodes", type=int, default=3_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--stage-steps", type=int, default=64)
    ap.add_argument("--only", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__ as g
    pkg = g.load_package()
    ctx = pkg.Context(0)
    result = {"bench": "stop_episodes", **gpu_info(), "workloads": []}
    jobs = [("ppo-c2", lambda: zeroed_rollout(pkg, build_ppo(pkg, ctx)), a.ppo_episodes, 4 * C2["T"], False),
            ("dqn-h64", lambda: build_replay(pkg, ctx, REPLAY["lanes65536"]), a.dqn_episodes, 64, True)]
    for name, make, k, warm, replay in jobs:
        if a.only and name != a.only:
            continue
        result["workloads"].append(bench(pkg, ctx, name, make, k, warm, a.reps, a.stage_steps, replay))
    ctx.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
