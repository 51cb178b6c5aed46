"""What the Float64 dynamics cost: the three device workloads on Float32 CartPole envs and on Float64 ones behind
StateTransformedEnv(env, Float32) (B200VecEnv.set_state_float32), built from the same seeds and run alternately.

  c2        PPO iteration (bench.py's c2): 65 536 CartPole envs, actor / critic 4-64-64, T = 32, 4 epochs x 4 minibatches, one
            CUDA-graph launch per iteration (env-steps/s)
  replay    the DQN agent loop of bench_replay.py's c5-h64 workload (env-steps/s)
  evaluate  bench_evaluate.py's fused greedy evaluation: 65 536 envs, 1 000 steps (env-steps/s)

Each number is the median of --reps timed windows per dtype, Float32 and Float64 windows interleaved.  The GPU name, power limit and
max SM clock are read in the same process.  Prints one JSON line; --out also writes it to a file."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_evaluate import glorot, gpu_info, splitmix   # noqa: E402
from bench_replay import WORKLOADS, build as build_replay, run_steps   # noqa: E402


def _env(pkg, ctx, n, seed, f64):
    env = pkg.B200VecEnv(ctx, "CartPole", n, splitmix(n, seed), T=np.float64 if f64 else np.float32, auto_reset=True)
    if f64:
        env.set_state_float32()
    return env


def _timed(ctx, fn, k):
    ctx.sync()
    t0 = time.perf_counter()
    for _ in range(k):
        fn()
    ctx.sync()
    return time.perf_counter() - t0


def bench_c2(pkg, ctx, reps, iters, n=65536, T=32):
    objs = {}
    for f64 in (False, True):
        env = _env(pkg, ctx, n, 0x9E37, f64)
        net = pkg.Network(ctx, 4, 64, 2, glorot(4, 64, 2, 123))
        agent = pkg.OnPolicyAgent(ctx, net, env, pkg.onpolicy_config(update_freq=T, n_epochs=4, n_microbatches=4), splitmix(n, 0x1234),
                                  host_actions=False)
        env.reset_(is_force=True)
        agent.iterate(2)                                 # eager, then captured
        objs[f64] = (env, net, agent)
    res = {False: [], True: []}
    for _ in range(reps):
        for f64 in (False, True):
            dt = _timed(ctx, lambda: objs[f64][2].iterate(1), iters)
            res[f64].append(iters * T * n / dt)
    for o in objs.values():
        o[2].close(); o[1].close(); o[0].close()
    return res


def bench_replay(pkg, ctx, reps, steps):
    w = WORKLOADS["c5-h64"]
    objs = {}
    for f64 in (False, True):
        s = build_replay(pkg, ctx, w)
        if f64:   # the same seeds, Float64 dynamics
            s["env"].close()
            s["env"] = _env(pkg, ctx, w["lanes"], 5, True)
        run_steps(pkg, ctx, s, 40)
        objs[f64] = s
    res = {False: [], True: []}
    for _ in range(reps):
        for f64 in (False, True):
            dt, _ = run_steps(pkg, ctx, objs[f64], steps)
            res[f64].append(steps * w["lanes"] / dt)
    graphs = all(s["agent"].graph_active() for s in objs.values())
    for s in objs.values():
        s["agent"].close()
        for k in ("policy", "traj", "net", "env"):
            s[k].close()
    return res, graphs


def bench_evaluate(pkg, ctx, reps, n_steps, n=65536):
    L = pkg._lib
    net = pkg.Network(ctx, 4, 64, 2, glorot(4, 64, 2, 123))
    envs = {f64: _env(pkg, ctx, n, 1, f64) for f64 in (False, True)}
    d = [ctx.malloc(n * 4) for _ in range(3)]
    cfg = L.EvalConfig(0, n_steps, 1)
    call = lambda env: L.check(ctx.lib.b200rl_evaluate(net.h, env.h, C.byref(cfg), None, *(C.c_void_p(p) for p in d), 1))
    for env in envs.values():
        call(env)
    res = {False: [], True: []}
    for _ in range(reps):
        for f64 in (False, True):
            res[f64].append(n * n_steps / _timed(ctx, lambda: call(envs[f64]), 1))
    for p in d:
        ctx.free(p)
    for env in envs.values():
        env.close()
    net.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--c2-iters", type=int, default=10)
    ap.add_argument("--replay-steps", type=int, default=200)
    ap.add_argument("--eval-steps", type=int, default=1000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import __graft_entry__ as G
    pkg = G.load_package()
    ctx = pkg.Context(0)
    out = {"metric": "env-steps/s, Float32 env vs Float64 env behind StateTransformedEnv(env, Float32)", "reps": args.reps, **gpu_info()}

    def summary(res):
        f32, f64 = float(np.median(res[False])), float(np.median(res[True]))
        return {"f32": f32, "f64": f64, "f64_over_f32": f64 / f32, "f32_all": [round(x) for x in res[False]], "f64_all": [round(x) for x in res[True]]}
    out["c2"] = summary(bench_c2(pkg, ctx, args.reps, args.c2_iters))
    r, graphs = bench_replay(pkg, ctx, args.reps, args.replay_steps)
    out["replay_c5_h64"] = {**summary(r), "graph_active": graphs}
    out["evaluate"] = summary(bench_evaluate(pkg, ctx, args.reps, args.eval_steps))
    ctx.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
