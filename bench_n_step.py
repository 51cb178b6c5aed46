"""Cost of n-step returns on the H100: the NStepBatchSampler(n, γ) window walk inside the DQN update and inside the device agent loop.

  update       b200rl_dqn_update on the config-5 shape: 4096 lanes x 256 frames (1 M transitions) prioritised ring filled by
               random CartPole steps, batch 4096, Q-net 4-128-128-2; n = 1, 3, 5 on the same trajectory, alternating in rounds;
               `--updates` back-to-back updates per round timed with CUDA events on the library's stream
  agent_loop   run(Agent(...), env, StopAfterNSteps(k)) on the device path at bench_replay.py's c5-h128 setting, n = 1 vs n = 3
               (two agents built from the same seeds), alternating; host clock around runs that end in a device synchronise

Before any timing, one n = 3 batch at the timed size is checked against the NumPy restatement (tests/nstep_ref.py) over the
exported ring, bit for bit.  GPU name, power limit and max SM clock are read in the same process.  Prints one JSON line.

    python bench_n_step.py [--updates 200] [--rounds 3] [--steps 100] [--warmup 30] [--out result.json]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_evaluate import gpu_info, splitmix      # noqa: E402
from bench_replay import WORKLOADS, build, q_params, run_steps   # noqa: E402

NS = (1, 3, 5)


def bench_update(pkg, ctx, updates, rounds, lanes=4096, cap=256, B=4096, hidden=128, gamma=0.99):
    env = pkg.B200VecEnv(ctx, "CartPole", lanes, splitmix(lanes, 11), auto_reset=True)
    traj = pkg.Trajectory(ctx, 4, cap, lanes=lanes, batch_size=B, sampler_rng=splitmix(B, 12), prioritized=True)
    env.reset_(is_force=True)
    traj.push_env(env, first_state_only=True)
    for _ in range(cap + 20):                        # the ring has wrapped: every lane holds cap entries
        env.act_random_()
        traj.push_env(env)
    net = pkg.Network(ctx, 4, hidden, 2, q_params(4, hidden, 2, 13), kind=pkg.KIND_Q)
    learner = pkg.DQNLearner(ctx, net, traj, pkg.dqn_config(gamma=gamma, target_update_freq=100))
    # correctness at the timed size before timing
    import nstep_ref
    traj.set_nstep(3, gamma)
    b = traj.sample()
    rb = nstep_ref.nstep_batch(traj.export_state(), 4, lanes, cap, b["key"], 3, gamma)
    checked = all(np.array_equal(np.ascontiguousarray(b[f]).view(np.uint8), np.ascontiguousarray(rb[f]).view(np.uint8))
                  for f in ("reward", "terminal", "next_state", "discount", "horizon"))
    mean_h = float(b["horizon"].mean())
    res = {n: [] for n in NS}
    for n in NS:                                     # warm-up (kernel attributes, lazy loading)
        traj.set_nstep(n, gamma)
        for _ in range(5):
            learner.update()
    ctx.sync()
    for _ in range(rounds):
        for n in NS:
            traj.set_nstep(n, gamma)
            ctx.timer_start()
            for _ in range(updates):
                learner.update()
            res[n].append(ctx.timer_stop_ms() / updates)
    out = {"shape": dict(lanes=lanes, cap=cap, batch=B, hidden=hidden, updates_per_round=updates, rounds=rounds),
           "restatement_check_n3": bool(checked), "mean_horizon_n3": mean_h,
           "ms_per_update": {str(n): float(np.median(v)) for n, v in res.items()},
           "ms_per_update_all": {str(n): [round(x, 4) for x in v] for n, v in res.items()}}
    for c in (learner, net, traj, env):
        if hasattr(c, "close"):
            c.close()
    return out


def bench_agent_loop(pkg, ctx, steps, warmup, rounds):
    w = WORKLOADS["c5-h128"]
    agents = {1: build(pkg, ctx, w), 3: build(pkg, ctx, w)}
    agents[3]["traj"].set_nstep(3, 0.99)
    for s in agents.values():
        run_steps(pkg, ctx, s, warmup)
    res = {1: [], 3: []}
    for _ in range(rounds):
        for n, s in agents.items():
            dt, upd = run_steps(pkg, ctx, s, steps)
            res[n].append({"env_steps_per_s": steps * w["lanes"] / dt, "updates_per_s": upd / dt})
    out = {"workload": "c5-h128", **w, "steps": steps, "rounds": rounds,
           "graph_active": {str(n): s["agent"].graph_active() for n, s in agents.items()}}
    for n in res:
        out["n%d" % n] = {m: float(np.median([r[m] for r in res[n]])) for m in ("env_steps_per_s", "updates_per_s")}
    for s in agents.values():
        s["agent"].close()
        for k in ("policy", "traj", "net", "env"):
            s[k].close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__ as g
    pkg = g.load_package()
    ctx = pkg.Context(0)
    result = {"bench": "n_step", **gpu_info(), "update": bench_update(pkg, ctx, a.updates, a.rounds),
              "agent_loop": bench_agent_loop(pkg, ctx, a.steps, a.warmup, a.rounds)}
    ctx.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
