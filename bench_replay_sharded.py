"""Throughput of the sharded DQN agent loop (b200rl_replay_run on a communicator of G ranks, one process per GPU, DESIGN.md §3):
run(Agent(QBasedPolicy(DQNLearner, EpsilonGreedyExplorer), Trajectory), env, StopAfterNSteps(k), EmptyHook()) over G x 4096 envs,
each rank stepping its own 4096 (weak scaling) and summing the gradient once per update over the peer exchange (NCCL without it).

Workloads (CartPole, prioritised ring of 256 frames per lane, batch 4096 per rank, ratio 1 with a threshold, target sync every 100
updates, exp epsilon decay) — bench_replay.py's c5-h64 and c5-h128 per rank:
  c5-h64     Q-net 4-64-64-2
  c5-h128    Q-net 4-128-128-2

    python bench_replay_sharded.py [--steps 200] [--warmup 40] [--reps 3]                        # one GPU (G = 1)
    torchrun --nproc_per_node G bench_replay_sharded.py [--steps 200] [--warmup 40] [--reps 3]   # G GPUs

Prints one JSON line (rank 0): per rank and in aggregate env-steps/s and updates/s (medians over the timed runs; an update is one
global optimiser step, so every rank runs the same number), the card name and power limit of every rank's GPU, and
replicas_bit_identical (parameters, Adam state and target equal on every rank after the runs).  With one process the multi-GPU
fields say "not measured".  Writes nothing."""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_replay import q_params   # noqa: E402

WORKLOADS = {
    "c5-h64": dict(lanes=4096, cap=256, hidden=64, ratio=1.0),
    "c5-h128": dict(lanes=4096, cap=256, hidden=128, ratio=1.0),
}


def card(index):
    """name and power limit of GPU `index` (read-only nvidia-smi query)"""
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout
        name, power, clk = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:   # the numbers are then unlabelled: say so in the result
        return {"gpu": None, "error": repr(e)}


def build(pkg, ctx, w, B=4096, threshold=20, seed=5):
    rank, world = ctx.rank_world()
    n = w["lanes"]
    ex = pkg.EpsilonGreedyExplorer(0.01, kind="exp", eps_init=1.0, warmup_steps=10 * n * world, decay_steps=100 * n * world)
    return pkg.sharding.dqn_rank_agent(ctx, "CartPole", n * world, seed, q_params(4, w["hidden"], 2, seed + 1), w["hidden"], 2,
                                       pkg.dqn_config(target_update_freq=100), ex, w["cap"], B, prioritized=True, ratio=w["ratio"],
                                       threshold=threshold)


def run_steps(pkg, job, s, k):
    c = s["traj"].controller
    u0 = c.n_sampled
    job.barrier()
    t0 = time.perf_counter()
    pkg.run(s["agent"], s["env"], pkg.StopAfterNSteps(k), pkg.EmptyHook())
    job.ctx.sync()
    return time.perf_counter() - t0, c.n_sampled - u0


def replica_digest(pkg, s):
    h = hashlib.sha256()
    for which in (pkg.learners.NET_PARAMS, pkg.learners.NET_M, pkg.learners.NET_V, pkg.learners.NET_TARGET):
        h.update(np.ascontiguousarray(s["net"].get(which)).tobytes())
    return h.hexdigest()


def bench(pkg, job, name, w, steps, warmup, reps):
    s = build(pkg, job.ctx, w)
    run_steps(pkg, job, s, warmup)
    runs = []
    for _ in range(reps):
        dt, upd = run_steps(pkg, job, s, steps)
        runs.append({"env_steps_per_s": steps * w["lanes"] / dt, "updates_per_s": upd / dt, "sec": dt})
    mine = {m: float(np.median([r[m] for r in runs])) for m in ("env_steps_per_s", "updates_per_s", "sec")}
    mine["env_steps_per_s_all"] = [round(r["env_steps_per_s"]) for r in runs]
    mine["graph_active"] = s["agent"].graph_active()
    mine["digest"] = replica_digest(pkg, s)
    per_rank = job.gather_objects(mine)
    out = {"workload": name, **w, "lanes_per_rank": w["lanes"], "steps": steps, "reps": reps, "world": job.world,
           "per_rank": [{k: v for k, v in r.items() if k != "digest"} for r in per_rank],
           "replicas_bit_identical": len({r["digest"] for r in per_rank}) == 1}
    if job.world > 1:
        # the slowest rank's wall time bounds the job: aggregate = all envs over the longest median run
        sec = max(r["sec"] for r in per_rank)
        out["aggregate"] = {"env_steps_per_s": steps * w["lanes"] * job.world / sec, "updates_per_s": min(r["updates_per_s"] for r in per_rank)}
    else:
        out["aggregate"] = "not measured (one GPU)"
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
    a = ap.parse_args()
    from bench import Job
    a.gpus = int(os.environ.get("WORLD_SIZE", 1))
    job = Job(a)
    pkg = job.pkg
    info = job.gather_objects(card(job.local_rank))
    result = {"bench": "replay_agent_loop_sharded", "world": job.world, "gpus": info,
              "exchange": ("peer" if job.peer_exchange else "nccl") if job.world > 1 else "not measured (one GPU)", "workloads": []}
    for name, w in WORKLOADS.items():
        if a.only and name != a.only:
            continue
        result["workloads"].append(bench(pkg, job, name, w, a.steps, a.warmup, a.reps))
    if job.rank == 0:
        print(json.dumps(result), flush=True)
    job.close()


if __name__ == "__main__":
    main()
