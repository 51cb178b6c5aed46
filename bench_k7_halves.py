"""A/B timing of two builds of the library on bench.py's config c2 (or c3), in one process on the H100: the tensor-core PPO/A2C
loss + backward kernel alone (agent.time_kernel(0, ...), one minibatch launch) and the full iteration (c2: rollout + GAE + 4 epochs
x 4 minibatches; c3: rollout + GAE + one A2C minibatch; one CUDA graph launch each).

    python bench_k7_halves.py --lib-a OLD/libb200rl.so [--lib-b reinforcementlearning.jl_b200/libb200rl.so] [--rounds 5]
                              [--kernel-reps 20] [--iters 5] [--config c2|c3] [--kernel-only] [--phases] [--out result.json]

Build A from another commit with its own `reinforcementlearning.jl_b200/build.py` (for example in a `git worktree`); B defaults to
the in-tree library.  Both libraries are loaded RTLD_LOCAL, so each one's calls bind to its own kernels.  Each gets its own context
and an agent from the same seeds (c2: bench_episode_log.build_ppo; c3: bench.py's Pendulum A2C setup), warmed up with the graph captured.  Then `rounds` times,
alternating A and B: the kernel time (CUDA events over `kernel-reps` back-to-back launches) and the summed event time of `iters`
iterations, L2 flushed before each, as bench.py times them.  Medians with min and max are reported.  The two agents ran the same
iterations from the same seeds, so their parameters must agree bit for bit at the end.  --phases: the libraries are
B200RL_K7_TIMING builds; the per-phase cycle sums of one worker thread of each 64-sample half, in actor CTA 0 and in the last
(critic) CTA, are read after `kernel-reps` launches.  GPU name, power limit and max SM clock are read in the same process.  Prints
one JSON line; --out also writes it to a file."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_episode_log import build_ppo   # noqa: E402
from bench_evaluate import gpu_info   # noqa: E402

WATCH = (0, 64)   # worker threads of quadrant 0 (half 0) and quadrant 2 (half 1)


def build_c3(pkg, ctx):
    """bench.py --config c3: 32 768 Pendulum envs, A2C, Gaussian head, tanh 3-64-64 trunks, T = 32, one minibatch"""
    from b200rl import sharding as sh
    from bench import _dense
    n, T = 32768, 32
    r = np.random.default_rng(5)
    params = np.concatenate(_dense(r, 64, 3) + _dense(r, 64, 64) + _dense(r, 1, 64) + _dense(r, 1, 64) + _dense(r, 64, 3) + _dense(r, 64, 64) + _dense(r, 1, 64))
    cfg = pkg.onpolicy_config(update_freq=T, n_epochs=1, n_microbatches=1, algo="a2c", w_entropy=0.01, lambda_=0.95)
    env = pkg.B200VecEnv(ctx, "Pendulum", n, sh.splitmix_states(3, 0, n), auto_reset=True)
    net = pkg.Network(ctx, 3, 64, 1, params.copy(), act=pkg.ACT_TANH, kind=pkg.KIND_GAUSSIAN)
    agent = pkg.OnPolicyAgent(ctx, net, env, cfg, sh.splitmix_states(4, 0, n), host_actions=False)
    return dict(env=env, net=net, agent=agent)


def open_side(pkg, path, phases, config):
    L = pkg._lib
    lib = C.CDLL(os.path.abspath(path), mode=os.RTLD_LOCAL)
    for name, (res, args) in L.SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    if phases:
        lib.b200rl_debug_k7_watch.argtypes = [C.c_int]
        lib.b200rl_debug_k7_phases.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    L._LIB = lib                 # Context() binds the library load() returns; every object made from the context uses ctx.lib
    ctx = pkg.Context(0)
    s = (build_ppo if config == "c2" else build_c3)(pkg, ctx)
    s["env"].reset_(is_force=True)
    ctx.flush_l2()
    for _ in range(2):           # the first iteration runs eagerly, the second captures the graph
        s["agent"].iterate(1)
    ctx.sync()
    return dict(path=path, lib=lib, ctx=ctx, **s)


def timed_iters(side, iters):
    ctx, agent = side["ctx"], side["agent"]
    for i in range(iters):
        ctx.flush_l2()
        ctx.timer_record(2 * i)
        agent.iterate(1)
        ctx.timer_record(2 * i + 1)
    ctx.sync()
    return sum(ctx.timer_elapsed_ms(2 * i, 2 * i + 1) for i in range(iters)) / iters


def k7_phases(side, reps):
    """per-phase cycle sums per tile of the watched worker threads (nn_tc.cu K7_T slots 0..9, 16, 17)"""
    lib, agent = side["lib"], side["agent"]
    import torch
    grid = 2 * (torch.cuda.get_device_properties(0).multi_processor_count // 2)   # K7's grid (b200rl_onpolicy_time_kernel)
    out = {}
    buf = (C.c_ulonglong * 40)()
    for role, cta in (("actor_cta0", 0), ("critic_cta_last", grid - 1)):
        for tid in WATCH:
            lib.b200rl_debug_k7_watch(tid | (cta << 16))
            lib.b200rl_debug_k7_phases(buf, 1)
            agent.time_kernel(0, reps)
            lib.b200rl_debug_k7_phases(buf, 1)
            v = list(buf)
            tiles = max(1, v[15])
            out[f"{role}_tid{tid}"] = {"tiles": v[15], **{f"p{i}": round(v[i] / tiles) for i in list(range(10)) + [16, 17]}}
    lib.b200rl_debug_k7_watch(0)
    return out


def stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "all": [round(x, 4) for x in xs]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-a", required=True)
    ap.add_argument("--lib-b", default=os.path.join(ROOT, "reinforcementlearning.jl_b200", "libb200rl.so"))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--kernel-reps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--config", default="c2", choices=["c2", "c3"])
    ap.add_argument("--kernel-only", action="store_true")
    ap.add_argument("--phases", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__ as g
    pkg = g.load_package()
    sides = {"a": open_side(pkg, a.lib_a, a.phases, a.config), "b": open_side(pkg, a.lib_b, a.phases, a.config)}
    res = {k: {"kernel_ms": [], "iteration_ms": []} for k in sides}
    for _ in range(a.rounds):
        for k, s in sides.items():
            res[k]["kernel_ms"].append(s["agent"].time_kernel(0, a.kernel_reps))
        if not a.kernel_only:
            for k, s in sides.items():
                res[k]["iteration_ms"].append(timed_iters(s, a.iters))
    result = {"bench": "k7_halves", "config": a.config, **gpu_info(), "actor_ctas_env": os.environ.get("B200RL_K7_ACTOR_CTAS"), "rounds": a.rounds,
              "kernel_reps": a.kernel_reps, "iters_per_round": a.iters}
    for k, s in sides.items():
        result[k] = {"lib": s["path"], "kernel_ms": stats(res[k]["kernel_ms"])}
        if not a.kernel_only:
            result[k]["iteration_ms"] = stats(res[k]["iteration_ms"])
        if a.phases:
            result[k]["k7_phase_cycles_per_tile"] = k7_phases(s, a.kernel_reps)
    pa, pb = sides["a"]["net"].get(), sides["b"]["net"].get()
    result["params_bit_identical"] = bool(np.array_equal(pa.view(np.uint32), pb.view(np.uint32)))
    result["kernel_b_over_a"] = result["b"]["kernel_ms"]["median"] / result["a"]["kernel_ms"]["median"]
    if not a.kernel_only:
        result["iteration_b_over_a"] = result["b"]["iteration_ms"]["median"] / result["a"]["iteration_ms"]["median"]
    for s in sides.values():
        for key in ("agent", "net", "env", "ctx"):
            s[key].close()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
