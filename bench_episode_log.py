"""Cost of the device episode log on the H100: the same training run under DeviceEpisodeStats (four sums for the whole run) and
under DeviceEpisodeLog (every finished episode's return and length, handed to the host in windows of `capacity` env steps).

Workloads:
  ppo-c2       bench.py's config c2: PPO on 65 536 CartPole envs, T = 32, 4 epochs x 4 minibatches, 4-64-64-2 actor and critic,
               run(agent, env, StopAfterNSteps(iters * T), hook) on the fused path (b200rl_onpolicy_iterate; with the log:
               iterate(capacity / T) per window, then a flush)
  dqn-h64      bench_replay.py's c5-h64 loop: 4096 CartPole lanes x 256 frames, prioritised, batch 4096, 4-64-64-2 Q-network
  dqn-h128     the same loop with the config-5 4-128-128-2 Q-network (run_replay in windows of `capacity` steps with the log)

    python bench_episode_log.py [--iters 30] [--dqn-steps 256] [--capacity 64] [--reps 3] [--only NAME] [--out result.json]

Each workload builds one agent per hook from the same seeds, warms both up (graphs captured), then times `reps` runs per hook,
alternating (a new hook per run, as a user writes it; a new DeviceEpisodeLog takes over the previous one's ring and buffers), host clock around runs that end in a device synchronise; the medians are reported with the overhead of the log.
After the timed runs both agents must hold identical checkpoints: the log changes nothing the run computes.  GPU name, power
limit and max SM clock are read in the same process.  Prints one JSON line; --out also writes it to a file."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_evaluate import gpu_info, splitmix   # noqa: E402
from bench_replay import WORKLOADS as REPLAY, build as build_replay   # noqa: E402

C2 = dict(envs=65536, T=32, n_epochs=4, n_micro=4, hidden=64)


def glorot_ac(pkg, seed):
    from b200rl import sharding
    return sharding.glorot_actor_critic(seed, 4, C2["hidden"], 2)


def build_ppo(pkg, ctx):
    n = C2["envs"]
    cfg = pkg.onpolicy_config(update_freq=C2["T"], n_epochs=C2["n_epochs"], n_microbatches=C2["n_micro"])
    env = pkg.B200VecEnv(ctx, "CartPole", n, splitmix(n, 11), auto_reset=True)
    net = pkg.Network(ctx, 4, C2["hidden"], 2, glorot_ac(pkg, 123))
    agent = pkg.OnPolicyAgent(ctx, net, env, cfg, splitmix(n, 12), host_actions=False)
    return dict(env=env, net=net, agent=agent)


def hook_for(pkg, which, n, capacity):
    return pkg.DeviceEpisodeLog(n, capacity=capacity) if which == "log" else pkg.DeviceEpisodeStats()


def timed(pkg, ctx, s, steps, hook):
    ctx.sync()
    t0 = time.perf_counter()
    pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(steps), hook)
    ctx.sync()
    return time.perf_counter() - t0


def checkpoints_identical(pkg, a, b, replay):
    f = pkg.checkpoint.checkpoint_replay if replay else pkg.checkpoint.checkpoint
    x, y = f(a["env"], a["net"], a["agent"]), f(b["env"], b["net"], b["agent"])
    # (env/episode_stats differs by design: DeviceEpisodeStats zeroes the env's counters at the start of every run)
    return sorted(x) == sorted(y) and all(np.array_equal(np.asarray(x[k]), np.asarray(y[k])) for k in x if k != "env/episode_stats")


def bench(pkg, ctx, name, make, n, steps, warmup, reps, capacity, replay):
    s = {"stats": make(), "log": make()}
    for which in ("stats", "log"):
        timed(pkg, ctx, s[which], warmup, hook_for(pkg, which, n, capacity))
    res = {"stats": [], "log": []}
    episodes = 0
    for _ in range(reps):
        for which in ("stats", "log"):
            hook = hook_for(pkg, which, n, capacity)
            dt = timed(pkg, ctx, s[which], steps, hook)
            res[which].append(steps * n / dt)
            if which == "log":
                episodes = sum(map(len, hook.steps))
    out = {"workload": name, "envs": n, "steps": steps, "capacity": capacity, "reps": reps, "episodes_logged_per_run": episodes,
           "identical_checkpoints": bool(checkpoints_identical(pkg, s["stats"], s["log"], replay)),
           "graph_active": bool(s["log"]["agent"].graph_active())}
    for which in ("stats", "log"):
        out[which] = {"env_steps_per_s": float(np.median(res[which])), "env_steps_per_s_all": [round(v) for v in res[which]]}
    out["log_overhead_pct"] = 100.0 * (out["stats"]["env_steps_per_s"] / out["log"]["env_steps_per_s"] - 1.0)
    for x in s.values():
        x["agent"].close()
        for k in ("policy", "traj", "net", "env"):
            if k in x:
                x[k].close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30, help="PPO iterations per timed run")
    ap.add_argument("--dqn-steps", type=int, default=256, help="DQN env steps per timed run")
    ap.add_argument("--capacity", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__ as g
    pkg = g.load_package()
    ctx = pkg.Context(0)
    result = {"bench": "episode_log", **gpu_info(), "workloads": []}
    T = C2["T"]
    jobs = [("ppo-c2", lambda: build_ppo(pkg, ctx), C2["envs"], a.iters * T, 4 * T, False)]
    for name, key in (("dqn-h64", "c5-h64"), ("dqn-h128", "c5-h128")):
        w = REPLAY[key]
        jobs.append((name, lambda w=w: build_replay(pkg, ctx, w), w["lanes"], a.dqn_steps, 64, True))
    for name, make, n, steps, warmup, replay in jobs:
        if a.only and name != a.only:
            continue
        result["workloads"].append(bench(pkg, ctx, name, make, n, steps, warmup, a.reps, a.capacity, replay))
    ctx.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
