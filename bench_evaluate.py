"""Throughput of policy evaluation on the H100: greedy b200rl_evaluate (one fused launch per call), the stage protocol
run(EvaluationPolicy, env, StopAfterNSteps(n), DeviceEpisodeStats()) and, for context, the training rollout agent.collect(32),
all at 65 536 CartPole envs with the C2 actor shape (4 -> 64 -> 64 -> 2, relu).

    python bench_evaluate.py [--envs 65536] [--n-steps 1000] [--reps 5] [--stage-steps 200] [--out result.json]

Device time from CUDA events on the library's stream, one warm-up call per measurement, the L2 flushed before every timed call.
The GPU name, power limit and max SM clock are read in the same process.  Prints one JSON line; --out also writes it to a file."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def gpu_info():
    q = "name,power.limit,clocks.max.sm,driver_version"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
        name, power, clk, drv = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clk, "driver": drv}
    except Exception as e:   # the numbers below are then unlabelled: say so in the result
        return {"gpu": None, "error": repr(e)}


def splitmix(n, seed):
    M = (1 << 64) - 1
    out = np.empty((n, 4), np.uint64)
    z = (np.arange(n, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(seed & M)) & np.uint64(M)
    for k in range(4):
        z = (z + np.uint64(0x9E3779B97F4A7C15)) & np.uint64(M)
        x = z.copy()
        x = ((x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & np.uint64(M)
        x = ((x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & np.uint64(M)
        out[:, k] = x ^ (x >> np.uint64(31))
    return out


def glorot(n_in, H, n_out, seed):
    rng = np.random.default_rng(seed)
    parts = []
    for heads in ([n_out], [1]):                                 # actor, critic
        for o, i in [(H, n_in), (H, H)] + [(d, H) for d in heads]:
            lim = np.sqrt(6.0 / (i + o))
            parts += [rng.uniform(-lim, lim, (o, i)).astype(np.float32).ravel(order="F"), np.zeros(o, np.float32)]
    return np.concatenate(parts)


def timed(ctx, fn, reps):
    """device ms of each of `reps` calls (events on the ctx stream), L2 flushed before each"""
    out = []
    for _ in range(reps):
        ctx.flush_l2()
        ctx.timer_record(0)
        fn()
        ctx.timer_record(1)
        out.append(ctx.timer_elapsed_ms(0, 1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=65536)
    ap.add_argument("--n-steps", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--stage-steps", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import __graft_entry__ as g
    pkg = g.load_package()
    L = pkg._lib
    info = gpu_info()
    ctx = pkg.Context(0)
    n, H = args.envs, 64
    params = glorot(4, H, 2, 123)
    net = pkg.Network(ctx, 4, H, 2, params)
    res = {"metric": "evaluation env-steps/s", "envs": n, "actor": "4-64-64-2 relu", **info}

    # ---- fused greedy evaluation: b200rl_evaluate on device outputs (no host copy in the timed call) ---------------------
    env = pkg.B200VecEnv(ctx, "CartPole", n, splitmix(n, 1), auto_reset=True)
    d_ret, d_len, d_cnt = ctx.malloc(n * 4), ctx.malloc(n * 4), ctx.malloc(n * 4)
    cfg = L.EvalConfig(0, args.n_steps, 1)
    call = lambda: L.check(ctx.lib.b200rl_evaluate(net.h, env.h, C.byref(cfg), None, C.c_void_p(d_ret), C.c_void_p(d_len), C.c_void_p(d_cnt), 1))
    call()                                                       # warm-up (module load, shared-memory attribute)
    ms = timed(ctx, call, args.reps)
    cnt = ctx.d2h(np.empty(n, np.int32), d_cnt)
    lens = ctx.d2h(np.empty(n, np.int32), d_len)
    res["fused"] = {"n_steps": args.n_steps, "ms": ms, "value": n * args.n_steps / (np.median(ms) / 1e3), "unit": "env-steps/s",
                    "mean_first_episode_length": float(lens[cnt >= 1].mean()) if (cnt >= 1).any() else None}
    for p in (d_ret, d_len, d_cnt):
        ctx.free(p)

    # ---- stage protocol: run(EvaluationPolicy) with device-side episode statistics -----------------------------------------
    policy = pkg.EvaluationPolicy(net, n)
    policy.fusable = False      # the stage loop itself (run() would take the fused evaluation kernel: bench_evaluate_run.py)
    hook = pkg.DeviceEpisodeStats()
    stage = lambda: pkg.run(policy, env, pkg.StopAfterNSteps(args.stage_steps), hook)
    stage()
    ms = timed(ctx, stage, max(2, args.reps // 2))
    res["stage_protocol"] = {"n_steps": args.stage_steps, "ms": ms, "value": n * args.stage_steps / (np.median(ms) / 1e3), "unit": "env-steps/s",
                             "episodes": hook.stats["episodes"] if hook.stats else None}
    policy.close()
    env.close()

    # ---- context: the training rollout of the same actor (plus its critic), agent.collect(32) ------------------------------
    T = 32
    env = pkg.B200VecEnv(ctx, "CartPole", n, splitmix(n, 1), auto_reset=True)
    agent = pkg.OnPolicyAgent(ctx, net, env, pkg.onpolicy_config(update_freq=T), splitmix(n, 2), host_actions=False)
    env.reset_(is_force=True)
    ms = []
    for k in range(args.reps + 1):
        ctx.flush_l2()
        ctx.timer_record(0)
        agent.collect(T)
        ctx.timer_record(1)
        if k:
            ms.append(ctx.timer_elapsed_ms(0, 1))
        agent.update()                                           # empties the rollout (not timed)
    res["collect32"] = {"n_steps": T, "ms": ms, "value": n * T / (np.median(ms) / 1e3), "unit": "env-steps/s"}
    agent.close(); env.close(); net.close(); ctx.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
