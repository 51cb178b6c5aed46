"""Cost of the speedy and softmax explorers on the H100 against ϵ-greedy, on objects built from the same seeds.

  loop-h64   the device DQN agent loop at bench_replay.py's c5 settings: CartPole, 4096 lanes x 256 frames, prioritised,
             batch 4096, ratio 1, 4-64-64-2 (fused collect)
  loop-h128  the same loop with 4-128-128-2 (staged collect)
  q_explore  one b200rl_net_q_explore on 65 536 columns (4-64-64-2): host clock around `iters` back-to-back calls that end in
             a device synchronise (the calls run on the library's stream)

Explorers: EpsilonGreedyExplorer(:exp), EpsilonSpeedyExplorer(1e-6), WeightedSoftmaxExplorer(), GumbelSoftmaxExplorer(),
alternated rep by rep.  Host clock around runs that end in a device synchronise.  GPU name, power limit and max SM
clock are read in the same process.  Prints one JSON line; --out also writes it to a file.

    python bench_explorers.py [--steps 200] [--warmup 40] [--reps 3] [--iters 200] [--out result.json]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_evaluate import gpu_info, splitmix   # noqa: E402
from bench_replay import q_params, run_steps    # noqa: E402

KINDS = ("eps_greedy", "speedy", "weighted_softmax", "gumbel_softmax")


def explorer(pkg, kind, n):
    if kind == "eps_greedy":
        return pkg.EpsilonGreedyExplorer(0.01, kind="exp", eps_init=1.0, warmup_steps=10 * n, decay_steps=100 * n)
    if kind == "speedy":
        return pkg.EpsilonSpeedyExplorer(1e-6)
    return pkg.WeightedSoftmaxExplorer() if kind == "weighted_softmax" else pkg.GumbelSoftmaxExplorer()


def build(pkg, ctx, kind, hidden, lanes=4096, cap=256, B=4096, threshold=20, seed=5):
    env = pkg.B200VecEnv(ctx, "CartPole", lanes, splitmix(lanes, seed), auto_reset=True)
    net = pkg.Network(ctx, 4, hidden, 2, q_params(4, hidden, 2, seed + 1), kind=pkg.KIND_Q)
    traj = pkg.Trajectory(ctx, 4, cap, lanes=lanes, batch_size=B, sampler_rng=splitmix(B, seed + 2), prioritized=True)
    traj.controller = pkg.InsertSampleRatioController(ratio=1.0, threshold=threshold)
    learner = pkg.DQNLearner(ctx, net, traj, pkg.dqn_config(target_update_freq=100))
    policy = pkg.QBasedPolicy(ctx, learner, explorer(pkg, kind, lanes), splitmix(lanes, seed + 3), lanes)
    return dict(env=env, net=net, traj=traj, policy=policy, agent=pkg.Agent(policy, traj))


def close(s):
    s["agent"].close()
    for k in ("policy", "traj", "net", "env"):
        s[k].close()


def bench_loop(pkg, ctx, hidden, steps, warmup, reps):
    objs = {k: build(pkg, ctx, k, hidden) for k in KINDS}
    for s in objs.values():
        run_steps(pkg, ctx, s, warmup)
    res = {k: [] for k in KINDS}
    for _ in range(reps):
        for k in KINDS:
            dt, _ = run_steps(pkg, ctx, objs[k], steps)
            res[k].append(steps * 4096 / dt)
    out = {k: {"env_steps_per_s": float(np.median(v)), "all": [round(x) for x in v]} for k, v in res.items()}
    for s in objs.values():
        close(s)
    return out


def bench_q_explore(pkg, ctx, iters, reps, N=65536):
    net = pkg.Network(ctx, 4, 64, 2, q_params(4, 64, 2, 6), kind=pkg.KIND_Q)
    obs = np.asfortranarray(np.random.default_rng(1).standard_normal((4, N)).astype(np.float32))
    dobs, dact, drng = ctx.malloc(obs.nbytes), ctx.malloc(N * 4), ctx.malloc(N * 32)
    ctx.h2d(dobs, obs)
    ctx.h2d(drng, splitmix(N, 7))
    res = {k: [] for k in KINDS}
    structs = {k: explorer(pkg, k, N).as_struct() for k in KINDS}

    def call(k):
        assert ctx.lib.b200rl_net_q_explore(net.h, C.c_void_p(dobs), N, C.c_void_p(drng), C.byref(structs[k]), C.c_void_p(dact)) == 0

    for k in KINDS:
        for _ in range(20):
            call(k)
    ctx.sync()
    for _ in range(reps):
        for k in KINDS:
            ctx.sync()
            t0 = time.perf_counter()
            for _ in range(iters):
                call(k)
            ctx.sync()
            res[k].append((time.perf_counter() - t0) / iters * 1e6)
    for d in (dobs, dact, drng):
        ctx.free(d)
    net.close()
    return {k: {"us_per_call": float(np.median(v)), "all": [round(x, 2) for x in v]} for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__ as g
    pkg = g.load_package()
    ctx = pkg.Context(0)
    result = {"bench": "explorers", **gpu_info(),
              "loop-h64": bench_loop(pkg, ctx, 64, a.steps, a.warmup, a.reps),
              "loop-h128": bench_loop(pkg, ctx, 128, a.steps, a.warmup, a.reps),
              "q_explore_65536": bench_q_explore(pkg, ctx, a.iters, a.reps)}
    ctx.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
