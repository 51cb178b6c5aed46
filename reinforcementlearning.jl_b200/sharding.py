"""Host-side sharding rules for the multi-GPU path (SURVEY §8e): envs are partitioned by index,
rank r of G owns [r*N/G, (r+1)*N/G); RNG streams are keyed by the GLOBAL env index so a sharded
run owns exactly the streams the single-GPU run would; gradients are local sums scaled by
1/(B_local * G) and summed across ranks (one all-reduce per optimiser step); the advantage
normalisation uses globally reduced sums.  No compute here — index arithmetic, seeding, and the
constructor of one rank's DQN agent (dqn_rank_agent)."""
import numpy as np


def shard_range(n_total, rank, world):
    if n_total % world:
        raise ValueError("the number of envs must be divisible by the number of GPUs")
    n = n_total // world
    return rank * n, (rank + 1) * n


def splitmix_states(seed, lo, hi):
    """Test-harness seeding (SURVEY §8d): env i gets four successive splitmix64 outputs of seed ^ i.
    Returns (hi - lo, 4) uint64 raw Xoshiro256++ states for global env indices lo..hi-1.
    (The Julia glue passes `Xoshiro(hash(seed + i))` states instead.)"""
    M = np.uint64(0xFFFFFFFFFFFFFFFF)
    x = np.uint64(seed) ^ np.arange(lo, hi, dtype=np.uint64)
    out = np.empty((hi - lo, 4), dtype=np.uint64)
    with np.errstate(over="ignore"):
        for k in range(4):
            x = (x + np.uint64(0x9E3779B97F4A7C15)) & M
            z = x.copy()
            z = ((z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & M
            z = ((z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & M
            out[:, k] = z ^ (z >> np.uint64(31))
    return out


def julia_xoshiro_states(seeds):
    """Raw states of Julia's `Xoshiro(seed)` for an iterable of non-negative integer seeds (Julia 1.7–1.10: the SHA-256 digest of the
    seed's little-endian UInt32 words read as four little-endian UInt64; stdlib Random `seed!`).  Lets the Python mirror start the very
    streams the Julia glue passes for `[Xoshiro(s) for s in seeds]`.  Returns (len(seeds), 4) uint64.  Pure host-side seeding — the
    known answers Julia's manual prints for `Xoshiro(1234)` pin it (tests/test_oracle_julia_rng.py, tests/test_host_logic.py)."""
    import hashlib
    out = []
    for seed in seeds:
        seed = int(seed)
        if seed < 0:
            raise ValueError("Xoshiro(seed) needs a non-negative integer")
        words = bytearray()
        while True:
            words += (seed & 0xFFFFFFFF).to_bytes(4, "little")
            seed >>= 32
            if seed == 0:
                break
        out.append(np.frombuffer(hashlib.sha256(bytes(words)).digest(), dtype="<u8"))
    return np.array(out, dtype=np.uint64).reshape(len(out), 4)


def glorot_actor_critic(seed, n_in, hidden, n_out):
    """Flux `glorot_uniform` Dense init (U(+-sqrt(6/(in+out))), zero bias) in Flux.destructure order
    for ActorCritic(actor n_in-H-H-n_out, critic n_in-H-H-1); identical on every rank."""
    r = np.random.default_rng(seed)

    def dense(o, i):
        lim = np.sqrt(6.0 / (i + o))
        return [r.uniform(-lim, lim, (o, i)).astype(np.float32).ravel(order="F"), np.zeros(o, np.float32)]

    parts = dense(hidden, n_in) + dense(hidden, hidden) + dense(n_out, hidden)
    parts += dense(hidden, n_in) + dense(hidden, hidden) + dense(1, hidden)
    return np.concatenate(parts)


def dqn_rank_agent(ctx, env_kind, n_total, seed, q_params, hidden, n_out, cfg, explorer, capacity, batch_size, act=0, kind=None,
                   prioritized=False, n_step=1, ratio=1.0, threshold=1, env_params=None):
    """One rank's share of a sharded DQN replay run (DESIGN.md §3): ``Agent(QBasedPolicy(DQNLearner, explorer), Trajectory)`` over
    the global envs [r N, (r + 1) N) of ``n_total`` (rank and world from ``ctx.rank_world()``).

    Env streams are ``splitmix_states(seed, lo, hi)``, explorer streams ``splitmix_states(seed + 1, lo, hi)`` — keyed by the global
    env index, so the union of the ranks owns exactly the streams of one run over all envs — and the ring's sampler streams
    ``splitmix_states(seed + 2 + r, 0, batch_size)`` (each rank samples its own batch).  ``q_params`` seeds the Q-network and its
    target, identical on every rank; ``explorer`` is this rank's copy of the (identical) explorer, its step the global one.  The
    trajectory holds this rank's N lanes only.  Returns dict(env, net, traj, learner, policy, agent)."""
    from . import envs, learners
    rank, world = ctx.rank_world()
    lo, hi = shard_range(n_total, rank, world)
    n = hi - lo
    kw = {} if env_params is None else dict(params=env_params)
    env = envs.B200VecEnv(ctx, env_kind, n, splitmix_states(seed, lo, hi), auto_reset=True, **kw)
    n_in = envs._NOBS[env.kind]
    q_params = np.ascontiguousarray(q_params, np.float32)
    net = learners.Network(ctx, n_in, hidden, n_out, q_params.copy(), act=act, kind=learners.KIND_Q if kind is None else kind)
    net.set(learners.NET_TARGET, q_params.copy())   # (the target starts as the parameters on every rank)
    traj = learners.Trajectory(ctx, n_in, capacity, lanes=n, batch_size=batch_size,
                               sampler_rng=splitmix_states(seed + 2 + rank, 0, batch_size), prioritized=prioritized,
                               n_step=n_step, gamma=cfg.gamma)
    traj.controller = learners.InsertSampleRatioController(ratio=ratio, threshold=threshold)
    learner = learners.DQNLearner(ctx, net, traj, cfg)
    policy = learners.QBasedPolicy(ctx, learner, explorer, splitmix_states(seed + 1, lo, hi), n)
    return dict(env=env, net=net, traj=traj, learner=learner, policy=policy, agent=learners.Agent(policy, traj))


def attach_peer_exchange(ctx, rank, world, all_gather_bytes):
    """Wire the NVLink peer exchange of a one-process-per-GPU run (include/b200rl.h, b200rl_comm_p2p_*).

    ``all_gather_bytes(b: bytes) -> list[bytes]`` is any host-side all-gather in rank order (torch.distributed,
    MPI, a file system ...): it only ships the 64-byte CUDA IPC handles once.  Returns True when the fused
    exchange is active, False when IPC mapping is refused (the NCCL path stays in use)."""
    import ctypes as C

    from . import _lib as L
    handle = (C.c_char * 64)()
    L.check(ctx.lib.b200rl_comm_p2p_export(ctx.h, handle, None))
    handles = all_gather_bytes(bytes(handle.raw))
    regions = (C.c_void_p * world)()
    ok = True
    for r in range(world):
        if r == rank:
            continue
        p = C.c_void_p()
        if ctx.lib.b200rl_comm_p2p_open(ctx.h, handles[r], C.byref(p)) != L.OK:
            ok = False
            break
        regions[r] = p
    # every rank must take the same decision: one refused mapping disables the exchange everywhere
    flags = all_gather_bytes(b"\x01" if ok else b"\x00")
    if not all(f == b"\x01" for f in flags):
        return False
    L.check(ctx.lib.b200rl_comm_p2p_attach(ctx.h, regions))
    # one rank per physical GPU?  Then the optimiser step (with its gradient exchange) may run in the tail of the whole-device
    # loss + backward launch; ranks sharing a GPU keep the exchange in its own small kernel (they could not both be resident).
    bus = (C.c_char * 32)()
    L.check(ctx.lib.b200rl_ctx_pci_bus_id(ctx.h, bus, 32))
    ids = all_gather_bytes(bytes(bus.value))
    L.check(ctx.lib.b200rl_comm_p2p_set_exclusive(ctx.h, 1 if len(set(ids)) == world else 0))
    return True
