"""Cost of the dueling head (kind 3) against the plain Q-network (kind 2) on the H100, in one process on objects built from the
same seeds, the two kinds alternating.

  loop-h64    bench_replay.py's c5-h64: 4096 lanes x 256 frames, ratio 1, 4-64-64-2 (fused tensor-core collect + graph updates)
  loop-h128   bench_replay.py's c5-h128: the same loop with 4-128-128-2 (staged collect launches)
  update      one b200rl_dqn_update on the config-5 shape (1 M-transition prioritised ring, batch 4096, 4-128-128-2), CUDA events

    python bench_dueling.py [--steps 200] [--warmup 40] [--reps 3] [--updates 200] [--out result.json]

GPU name, power limit and max SM clock are read in the same process.  Prints one JSON line; --out also writes it to a file."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_evaluate import gpu_info, splitmix   # noqa: E402
from bench_replay import q_params, run_steps   # noqa: E402


def dueling_params(n_in, H, n_out, seed):
    """Flux.destructure(DuelingNetwork(Chain(Dense(n_in, H), Dense(H, H)), Dense(H, 1), Dense(H, n_out))) with glorot weights"""
    rng = np.random.default_rng(seed)
    parts = []
    for o, i in [(H, n_in), (H, H), (1, H), (n_out, H)]:
        lim = np.sqrt(6.0 / (i + o))
        parts += [rng.uniform(-lim, lim, (o, i)).astype(np.float32).ravel(order="F"), np.zeros(o, np.float32)]
    return np.concatenate(parts)


def make_net(pkg, ctx, H, kind, seed):
    p = dueling_params(4, H, 2, seed) if kind == pkg.KIND_DUELING else q_params(4, H, 2, seed)
    return pkg.Network(ctx, 4, H, 2, p, kind=kind)


def build_loop(pkg, ctx, H, kind, lanes=4096, cap=256, B=4096, threshold=20, seed=5):
    env = pkg.B200VecEnv(ctx, "CartPole", lanes, splitmix(lanes, seed), auto_reset=True)
    net = make_net(pkg, ctx, H, kind, seed + 1)
    traj = pkg.Trajectory(ctx, 4, cap, lanes=lanes, batch_size=B, sampler_rng=splitmix(B, seed + 2), prioritized=True)
    traj.controller = pkg.InsertSampleRatioController(ratio=1.0, threshold=threshold)
    learner = pkg.DQNLearner(ctx, net, traj, pkg.dqn_config(target_update_freq=100))
    ex = pkg.EpsilonGreedyExplorer(0.01, kind="exp", eps_init=1.0, warmup_steps=10 * lanes, decay_steps=100 * lanes)
    policy = pkg.QBasedPolicy(ctx, learner, ex, splitmix(lanes, seed + 3), lanes)
    return dict(env=env, net=net, traj=traj, policy=policy, agent=pkg.Agent(policy, traj))


def close(s):
    s["agent"].close()
    for k in ("policy", "traj", "net", "env"):
        s[k].close()


def bench_loop(pkg, ctx, H, steps, warmup, reps):
    s = {k: build_loop(pkg, ctx, H, k) for k in (pkg.KIND_Q, pkg.KIND_DUELING)}
    for k in s:
        run_steps(pkg, ctx, s[k], warmup)
    res = {k: [] for k in s}
    for _ in range(reps):
        for k in s:
            dt, _ = run_steps(pkg, ctx, s[k], steps)
            res[k].append(steps * 4096 / dt)
    out = {"workload": f"loop-h{H}", "lanes": 4096, "cap": 256, "hidden": H, "steps": steps, "reps": reps,
           "fused_collect": H == 64}
    for k, name in ((pkg.KIND_Q, "q"), (pkg.KIND_DUELING, "dueling")):
        out[name] = {"env_steps_per_s": float(np.median(res[k])), "env_steps_per_s_all": [round(x) for x in res[k]],
                     "graph_active": s[k]["agent"].graph_active()}
    out["dueling_over_q"] = out["dueling"]["env_steps_per_s"] / out["q"]["env_steps_per_s"]
    for k in s:
        close(s[k])
    return out


def bench_update(pkg, ctx, n_updates, reps, lanes=4096, cap=256, B=4096, seed=7):
    import torch
    trajs, learners, nets = {}, {}, {}
    for kind in (pkg.KIND_Q, pkg.KIND_DUELING):
        tr = pkg.Trajectory(ctx, 4, cap, lanes=lanes, batch_size=B, sampler_rng=splitmix(B, seed), prioritized=True)
        r = np.random.default_rng(seed)
        tr.push_state(r.standard_normal((4, lanes)).astype(np.float32))
        for _ in range(cap):
            tr.push(r.integers(1, 3, lanes).astype(np.int32), r.standard_normal(lanes).astype(np.float32),
                    (r.random(lanes) < 0.05).astype(np.uint8), r.standard_normal((4, lanes)).astype(np.float32))
        nets[kind] = make_net(pkg, ctx, 128, kind, seed + 1)
        trajs[kind] = tr
        learners[kind] = pkg.DQNLearner(ctx, nets[kind], tr, pkg.dqn_config(target_update_freq=100))
    times = {k: [] for k in learners}
    for k in learners:                                           # warm-up
        for _ in range(10):
            learners[k].update()
    ctx.sync()
    for _ in range(reps):
        for k in learners:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ctx.sync()
            e0.record()
            for _ in range(n_updates):
                learners[k].update()
            ctx.sync()
            e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1) / n_updates)
    out = {"workload": "update", "ring": lanes * cap, "batch": B, "hidden": 128, "updates": n_updates, "reps": reps}
    for k, name in ((pkg.KIND_Q, "q"), (pkg.KIND_DUELING, "dueling")):
        out[name] = {"ms_per_update": float(np.median(times[k])), "ms_all": [round(t, 4) for t in times[k]]}
    out["dueling_over_q"] = out["dueling"]["ms_per_update"] / out["q"]["ms_per_update"]
    for k in learners:
        nets[k].close(); trajs[k].close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--updates", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__ as g
    pkg = g.load_package()
    ctx = pkg.Context(0)
    result = {"bench": "dueling_head", **gpu_info(), "workloads": []}
    for H in (64, 128):
        result["workloads"].append(bench_loop(pkg, ctx, H, a.steps, a.warmup, a.reps))
    result["workloads"].append(bench_update(pkg, ctx, a.updates, a.reps))
    ctx.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
