"""Throughput of run(policy, env, stop, hook) for the policies that do not train, at 65 536 CartPole envs with a 4 -> 64 -> 64 -> 2
relu network: the greedy EvaluationPolicy and an epsilon-greedy QBasedPolicy under StopAfterNEpisodes(k) with a DeviceEpisodeLog,
on the fused evaluation kernel (b200rl_eval_run_episodes) against the stage loop (fusable = False) on twins from the same seeds,
alternated; and run(EvaluationPolicy, env, StopAfterNSteps(1000), EmptyHook()) against evaluate(net, env, 1000).

    python bench_evaluate_run.py [--envs 65536] [--episodes-per-env 20] [--capacity 64] [--n-steps 1000] [--reps 5] [--out result.json]

Wall time of each whole run() (it ends with a device synchronisation; the log's flushes and reads are part of it), median of
--reps alternated repetitions after one warm-up of each leg; each leg keeps its env, policy and hook, restored to the same state
before every repetition.  Every pair of twins must stop after the same step with the same episode count.  The GPU name, power limit and max SM
clock are read in the same process.  Prints one JSON line; --out also writes it to a file."""
import argparse
import json
import os
import sys
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_evaluate import glorot, gpu_info, splitmix   # noqa: E402


def q_params(n_in, H, n_out, seed):
    p = glorot(n_in, H, n_out, seed)
    return p[:n_in * H + H + H * H + H + n_out * H + n_out]        # the actor part: one Q-network


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=65536)
    ap.add_argument("--episodes-per-env", type=int, default=20)
    ap.add_argument("--capacity", type=int, default=64)
    ap.add_argument("--n-steps", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import __graft_entry__ as g
    pkg = g.load_package()
    info = gpu_info()
    ctx = pkg.Context(0)
    n, H = args.envs, 64
    k = args.episodes_per_env * n
    res = {"metric": "run() env-steps/s", "envs": n, "network": "4-64-64-2 relu", "episodes": k, "log_capacity": args.capacity, **info}
    ac = pkg.Network(ctx, 4, H, 2, glorot(4, H, 2, 123))
    q = pkg.Network(ctx, 4, H, 2, q_params(4, H, 2, 124), kind=pkg.KIND_Q)

    def make_policy(which):
        if which == "greedy":
            return pkg.EvaluationPolicy(ac, n)
        return pkg.QBasedPolicy(ctx, types.SimpleNamespace(net=q), pkg.EpsilonGreedyExplorer(0.05, warmup_steps=0, decay_steps=0),
                                splitmix(n, 7), n)

    def episodes_leg(which, fused):
        """one leg: its env, policy and hook, kept across the repetitions (the hook's ring, host buffers and the policy's handle are
        allocated once); every repetition starts from the same env state and streams"""
        env = pkg.B200VecEnv(ctx, "CartPole", n, splitmix(n, 1), auto_reset=True)
        env0 = pkg.checkpoint.checkpoint(env=env)
        pol = make_policy(which)
        pol.fusable = fused
        hook = pkg.DeviceEpisodeLog(n, capacity=args.capacity)

        def once():
            pkg.checkpoint.restore(env0, env=env)
            if which != "greedy":
                pol.set_explorer_rng(splitmix(n, 7))
                pol.explorer.step = 1
            hook._chunks = []                      # (the records of the previous repetition: not read here)
            stop = pkg.StopAfterNEpisodes(k)
            steps0 = env.episode_stats()["env_steps"]
            ctx.sync()
            t0 = time.perf_counter()
            pkg.run(pol, env, stop, hook)
            sec = time.perf_counter() - t0
            return dict(sec=sec, steps=round((env.episode_stats()["env_steps"] - steps0) / n), cur=stop.cur)

        def close():
            hook.close(); pol.close(); env.close()
        return once, close

    for which in ("greedy", "epsilon_greedy"):
        out = {"fused": [], "stage": []}
        legs = {leg: episodes_leg(which, leg == "fused") for leg in out}
        for leg in out:
            legs[leg][0]()                         # warm-up
        for _ in range(args.reps):
            for leg in out:
                out[leg].append(legs[leg][0]())
        for leg in out:
            legs[leg][1]()
        steps = {(r["steps"], r["cur"]) for leg in out for r in out[leg]}
        assert len(steps) == 1, steps             # the twins stop after the same step with the same count
        (s, cur), = steps
        entry = {"steps": s, "episodes_counted": cur}
        for leg in out:
            secs = [r["sec"] for r in out[leg]]
            entry[leg] = {"sec": secs, "value": n * s / float(np.median(secs)), "unit": "env-steps/s"}
        entry["speedup"] = entry["fused"]["value"] / entry["stage"]["value"]
        res[f"stop_after_n_episodes_{which}"] = entry

    # ---- StopAfterNSteps(n_steps) fused against evaluate(net, env, n_steps): each includes its forced reset -------------------
    env = pkg.B200VecEnv(ctx, "CartPole", n, splitmix(n, 1), auto_reset=True)
    pol = make_policy("greedy")
    legs = {"run_fused": lambda: pkg.run(pol, env, pkg.StopAfterNSteps(args.n_steps), pkg.EmptyHook()),
            "evaluate": lambda: pkg.evaluate(ac, env, args.n_steps)}
    times = {name: [] for name in legs}
    for name, fn in legs.items():
        fn()
    for _ in range(args.reps):
        for name, fn in legs.items():
            ctx.sync()
            t0 = time.perf_counter()
            fn()
            ctx.sync()
            times[name].append(time.perf_counter() - t0)
    assert pol._eval is not None
    res["stop_after_n_steps"] = {name: {"n_steps": args.n_steps, "sec": t, "value": n * args.n_steps / float(np.median(t)),
                                        "unit": "env-steps/s"} for name, t in times.items()}
    pol.close(); env.close(); ac.close(); q.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
