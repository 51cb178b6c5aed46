"""Throughput of evaluating a QBasedPolicy with its explorer on the H100: b200rl_evaluate_explore (one fused launch per call) with
ϵ-greedy, EpsilonSpeedyExplorer, WeightedSoftmaxExplorer, GumbelSoftmaxExplorer and GreedyExplorer, greedy b200rl_evaluate (mode 0)
on the same Q-network, and, for context, the stage protocol run(QBasedPolicy, env, StopAfterNSteps(n), DeviceEpisodeStats()).
65 536 CartPole envs, a 4 -> 64 -> 64 -> 2 relu Q-network with Glorot-uniform weights and zero biases.

    python bench_evaluate_explore.py [--envs 65536] [--n-steps 1000] [--reps 3] [--stage-steps 200] [--out result.json]

Every variant starts each call from the same env and explorer streams (restored outside the timed region); the variants alternate
within each repetition.  Device time from CUDA events on the library's stream, the L2 flushed before every timed call, the median of
--reps.  The GPU name, power limit and max SM clock are read in the same process.  Prints one JSON line; --out also writes it."""
import argparse
import ctypes as C
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_evaluate import gpu_info, splitmix  # noqa: E402


def glorot_q(n_in, H, n_out, seed):
    rng = np.random.default_rng(seed)
    parts = []
    for o, i in [(H, n_in), (H, H), (n_out, H)]:
        lim = np.sqrt(6.0 / (i + o))
        parts += [rng.uniform(-lim, lim, (o, i)).astype(np.float32).ravel(order="F"), np.zeros(o, np.float32)]
    return np.concatenate(parts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=65536)
    ap.add_argument("--n-steps", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--stage-steps", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import __graft_entry__ as g
    pkg = g.load_package()
    L = pkg._lib
    info = gpu_info()
    ctx = pkg.Context(0)
    n, H, T = args.envs, 64, args.n_steps
    net = pkg.Network(ctx, 4, H, 2, glorot_q(4, H, 2, 123), kind=pkg.KIND_Q)
    res = {"metric": "QBasedPolicy evaluation env-steps/s", "envs": n, "q_network": "4-64-64-2 relu", **info}

    env = pkg.B200VecEnv(ctx, "CartPole", n, splitmix(n, 1), auto_reset=True)
    env0 = pkg.checkpoint.checkpoint(env=env)
    xseeds = splitmix(n, 2)
    d_rng, d_ret, d_len, d_cnt = ctx.malloc(n * 32), ctx.malloc(n * 4), ctx.malloc(n * 4), ctx.malloc(n * 4)
    explorers = {
        "epsilon_greedy": lambda: pkg.EpsilonGreedyExplorer(0.01, eps_init=1.0, warmup_steps=0, decay_steps=n * T // 2),
        "speedy": lambda: pkg.EpsilonSpeedyExplorer(1.0 / (n * T)),
        "weighted_softmax": pkg.WeightedSoftmaxExplorer,
        "gumbel_softmax": pkg.GumbelSoftmaxExplorer,
        "greedy_explorer": pkg.GreedyExplorer,
    }
    cfg = L.EvalConfig(0, T, 1)

    def call(name):
        if name == "greedy_mode0":
            return L.check(ctx.lib.b200rl_evaluate(net.h, env.h, C.byref(cfg), None, C.c_void_p(d_ret), C.c_void_p(d_len), C.c_void_p(d_cnt), 1))
        ex = explorers[name]()
        st = ex.as_struct() if hasattr(ex, "as_struct") else None
        L.check(ctx.lib.b200rl_evaluate_explore(net.h, env.h, T, 1, None if st is None else C.byref(st), C.c_void_p(d_rng),
                                                C.c_void_p(d_ret), C.c_void_p(d_len), C.c_void_p(d_cnt), 1))

    names = ["greedy_mode0"] + list(explorers)
    ms = {k: [] for k in names}
    lens = {}
    for rep in range(args.reps + 1):                             # repetition 0: warm-up (module load, shared-memory attributes)
        for name in names:
            pkg.checkpoint.restore(env0, env=env)                # the same env and explorer streams for every call
            ctx.h2d(d_rng, xseeds)
            ctx.flush_l2()
            ctx.timer_record(0)
            call(name)
            ctx.timer_record(1)
            t = ctx.timer_elapsed_ms(0, 1)
            if rep:
                ms[name].append(t)
            else:
                cnt, ln = ctx.d2h(np.empty(n, np.int32), d_cnt), ctx.d2h(np.empty(n, np.int32), d_len)
                lens[name] = float(ln[cnt >= 1].mean()) if (cnt >= 1).any() else None
    for name in names:
        res[name] = {"n_steps": T, "ms": ms[name], "median_ms": float(np.median(ms[name])),
                     "value": n * T / (np.median(ms[name]) / 1e3), "unit": "env-steps/s", "mean_first_episode_length": lens[name]}

    # ---- context: the stage protocol, q_explore + act! launches per step ------------------------------------------------------
    policy = pkg.QBasedPolicy(ctx, types.SimpleNamespace(net=net), explorers["epsilon_greedy"](), xseeds, n)
    policy.fusable = False      # the stage loop itself (run() would take the fused evaluation kernel: bench_evaluate_run.py)
    hook = pkg.DeviceEpisodeStats()
    stage = []
    for rep in range(args.reps + 1):
        pkg.checkpoint.restore(env0, env=env)
        ctx.flush_l2()
        ctx.timer_record(0)
        pkg.run(policy, env, pkg.StopAfterNSteps(args.stage_steps), hook)
        ctx.timer_record(1)
        if rep:
            stage.append(ctx.timer_elapsed_ms(0, 1))
    res["stage_protocol_epsilon_greedy"] = {"n_steps": args.stage_steps, "ms": stage, "median_ms": float(np.median(stage)),
                                            "value": n * args.stage_steps / (np.median(stage) / 1e3), "unit": "env-steps/s"}
    policy.close()
    for p in (d_rng, d_ret, d_len, d_cnt):
        ctx.free(p)
    env.close(); net.close(); ctx.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
