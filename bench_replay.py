"""Throughput of the DQN agent loop on the H100: run(Agent(QBasedPolicy(DQNLearner, EpsilonGreedyExplorer), Trajectory), env,
StopAfterNSteps(k), EmptyHook()) on the device path (b200rl_replay_run) against the stage protocol (agent.fusable = False) on
objects built from the same seeds.

Workloads (CartPole, prioritised ring, batch 4096, target sync every 100 updates, exp epsilon decay):
  c5-h128      4096 lanes x 256 frames (1 M transitions), ratio 1 with a threshold, the config-5 Q-net 4-128-128-2
  c5-h64       the same loop with a 4-64-64-2 Q-net
  c5-r025      the config-5 loop with ratio 0.25 (one update every 4 steps: stretches without an update)
  lanes65536   65 536 lanes x 16 frames, 4-64-64-2, ratio 1

    python bench_replay.py [--steps 200] [--warmup 40] [--reps 3] [--only NAME] [--out result.json]

Each workload: a warm-up run on both paths (graphs captured, ring partly filled, learning started), then `reps` timed runs of
`steps` env steps on each path, alternating; host clock around runs that end in a device synchronise.  After the timed runs the
two paths' checkpoints must be identical (every field of checkpoint_replay).  GPU name, power limit and max SM clock are read in
the same process.  Prints one JSON line; --out also writes it to a file."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_evaluate import gpu_info, splitmix   # noqa: E402

WORKLOADS = {
    "c5-h128": dict(lanes=4096, cap=256, hidden=128, ratio=1.0),
    "c5-h64": dict(lanes=4096, cap=256, hidden=64, ratio=1.0),
    "c5-r025": dict(lanes=4096, cap=256, hidden=128, ratio=0.25),
    "lanes65536": dict(lanes=65536, cap=16, hidden=64, ratio=1.0),
}


def q_params(n_in, H, n_out, seed):
    rng = np.random.default_rng(seed)
    parts = []
    for o, i in [(H, n_in), (H, H), (n_out, H)]:
        lim = np.sqrt(6.0 / (i + o))
        parts += [rng.uniform(-lim, lim, (o, i)).astype(np.float32).ravel(order="F"), np.zeros(o, np.float32)]
    return np.concatenate(parts)


def build(pkg, ctx, w, B=4096, threshold=20, seed=5):
    n = w["lanes"]
    env = pkg.B200VecEnv(ctx, "CartPole", n, splitmix(n, seed), auto_reset=True)
    net = pkg.Network(ctx, 4, w["hidden"], 2, q_params(4, w["hidden"], 2, seed + 1), kind=pkg.KIND_Q)
    traj = pkg.Trajectory(ctx, 4, w["cap"], lanes=n, batch_size=B, sampler_rng=splitmix(B, seed + 2), prioritized=True)
    traj.controller = pkg.InsertSampleRatioController(ratio=w["ratio"], threshold=threshold)
    learner = pkg.DQNLearner(ctx, net, traj, pkg.dqn_config(target_update_freq=100))
    ex = pkg.EpsilonGreedyExplorer(0.01, kind="exp", eps_init=1.0, warmup_steps=10 * n, decay_steps=100 * n)
    policy = pkg.QBasedPolicy(ctx, learner, ex, splitmix(n, seed + 3), n)
    return dict(env=env, net=net, traj=traj, policy=policy, agent=pkg.Agent(policy, traj))


def run_steps(pkg, ctx, s, k):
    c = s["traj"].controller
    u0 = c.n_sampled
    ctx.sync()
    t0 = time.perf_counter()
    pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(k), pkg.EmptyHook())
    ctx.sync()
    return time.perf_counter() - t0, c.n_sampled - u0


def bench(pkg, ctx, name, w, steps, warmup, reps):
    fast, stage = build(pkg, ctx, w), build(pkg, ctx, w)
    stage["agent"].fusable = False
    run_steps(pkg, ctx, fast, warmup)
    run_steps(pkg, ctx, stage, warmup)
    res = {"fast": [], "stage": []}
    for _ in range(reps):
        for key, s in (("fast", fast), ("stage", stage)):
            dt, upd = run_steps(pkg, ctx, s, steps)
            res[key].append({"sec": dt, "env_steps_per_s": steps * w["lanes"] / dt, "updates_per_s": upd / dt, "updates": upd})
    a = pkg.checkpoint.checkpoint_replay(fast["env"], fast["net"], fast["agent"])
    b = pkg.checkpoint.checkpoint_replay(stage["env"], stage["net"], stage["agent"])
    identical = sorted(a) == sorted(b) and all(np.array_equal(np.asarray(a[k]), np.asarray(b[k])) for k in a)
    out = {"workload": name, **w, "steps": steps, "reps": reps, "identical_checkpoints": bool(identical),
           "graph_active": fast["agent"].graph_active()}
    for key in ("fast", "stage"):
        out[key] = {m: float(np.median([r[m] for r in res[key]])) for m in ("env_steps_per_s", "updates_per_s")}
        out[key]["env_steps_per_s_all"] = [round(r["env_steps_per_s"]) for r in res[key]]
    out["speedup_env_steps"] = out["fast"]["env_steps_per_s"] / out["stage"]["env_steps_per_s"]
    for s in (fast, stage):
        s["agent"].close()
        for k in ("policy", "traj", "net", "env"):
            s[k].close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__ as g
    pkg = g.load_package()
    ctx = pkg.Context(0)
    result = {"bench": "replay_agent_loop", **gpu_info(), "workloads": []}
    for name, w in WORKLOADS.items():
        if a.only and name != a.only:
            continue
        result["workloads"].append(bench(pkg, ctx, name, w, a.steps, a.warmup, a.reps))
    ctx.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
