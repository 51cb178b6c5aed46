"""The sharded DQN replay loop on Float64 envs behind StateTransformedEnv(env, Float32), with the two-ranks-in-one-process harness of
test_replay_sharded_gpu.py (two ctx on cuda:0, two threads, peer exchange):

(1) on each rank the device loop equals the stage protocol bit for bit, and the replicas (parameters, Adam state, target, step)
    end bit-identical;
(2) ranks that disagree on the wrapper (one a wrapped Float64 env, the other a Float32 env of the same N) both refuse with
    B200RL_ERR_INVALID and touch nothing."""
import ctypes as C

import numpy as np
import pytest

import test_replay_sharded_gpu as SH

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pairs(pkg):
    p = [SH._two_ranks(pkg), SH._two_ranks(pkg)]
    one = pkg.Context(0)
    yield p, one
    for ctxs in p:
        for c in ctxs:
            c.close()
    one.close()


def _rank(pkg, ctx, n_total, case, f64=True, seed=100, steps=10):
    """SH._agent's rank, its env replaced by the Float64 env over the same global streams (behind the wrapper)"""
    s = SH._agent(pkg, ctx, n_total, case, seed=seed, steps=steps)
    if f64:
        rank, world = ctx.rank_world()
        lo, hi = pkg.sharding.shard_range(n_total, rank, world)
        s["env"].close()
        s["env"] = pkg.B200VecEnv(ctx, case.get("env", "CartPole"), hi - lo, pkg.sharding.splitmix_states(seed, lo, hi), T=np.float64,
                                  auto_reset=True)
        s["env"].set_state_float32()
    return s


def _warm(pkg, one, n_total, case):
    """every kernel of the configuration launched once, unsharded, fused and staged, on Float64 and Float32 envs"""
    for f64 in (True, False):
        for fusable in (True, False):
            w = _rank(pkg, one, n_total, dict(case, threshold=1), f64=f64, seed=5, steps=4)
            w["agent"].fusable = fusable
            pkg.run(w["agent"], w["env"], pkg.StopAfterNSteps(4), pkg.EmptyHook())
            SH._close(w)


CASES = [dict(ratio=1.0, threshold=2, prioritized=True, target_freq=3),
         dict(env="MountainCar", ratio=0.25, threshold=2, prioritized=False, explorer="exp", target_freq=2)]


@pytest.mark.parametrize("case", CASES, ids=["CartPole-per", "MountainCar-uniform"])
def test_sharded_float64_loop_equals_stage_protocol_and_replicas_agree(pkg, pairs, case):
    (fast_ctx, stage_ctx), one = pairs
    n, steps = 127, 14
    _warm(pkg, one, 2 * n, case)
    fast = [_rank(pkg, c, 2 * n, case, steps=steps) for c in fast_ctx]
    stage = [_rank(pkg, c, 2 * n, case, steps=steps) for c in stage_ctx]
    SH._run_pair(pkg, fast, steps)
    SH._run_pair(pkg, stage, steps, fusable=False)
    SH._run_pair(pkg, fast, 5)
    SH._run_pair(pkg, stage, 5, fusable=False)
    assert all(s["agent"]._replay is not None for s in fast) and all(s["agent"]._replay is None for s in stage)
    ck = [[SH._state(pkg, s) for s in p] for p in (fast, stage)]
    for r in range(2):
        SH._assert_same(ck[0][r], ck[1][r])
        assert ck[0][r]["env/state"].dtype == np.float64
    for k in ("net/params", "net/adam_m", "net/adam_v", "net/beta_t", "net/target", "net/step", "policy/explorer_step"):
        assert np.array_equal(ck[0][0][k], ck[0][1][k]), k                   # replicas bit-identical
    assert fast[0]["net"].step_count() > 1
    for s in fast + stage:
        SH._close(s)


def test_ranks_disagreeing_on_the_wrapper_refuse_and_touch_nothing(pkg, pairs):
    (ctxs, _), one = pairs
    L = pkg._lib
    n, case = 64, dict(ratio=1.0, threshold=2)
    _warm(pkg, one, 2 * n, case)
    agreeing = [_rank(pkg, c, 2 * n, case, steps=8) for c in ctxs]
    SH._run_pair(pkg, agreeing, 3)                                            # the pair's exchange warm
    for s in agreeing:
        SH._close(s)
    ranks = [_rank(pkg, ctxs[0], 2 * n, case, f64=True, steps=8), _rank(pkg, ctxs[1], 2 * n, case, f64=False, steps=8)]
    SH._prepare(ranks)
    hs = [s["agent"]._handle(s["env"]) for s in ranks]
    before = [SH._state(pkg, s) for s in ranks]
    codes = [None, None]

    def go(r):
        s = ranks[r]
        c = s["traj"].controller
        ctl = L.InsertSampleRatio(c.ratio, c.threshold, c.n_inserted, c.n_sampled)
        ex = s["policy"].explorer.as_struct()
        codes[r] = ctxs[r].lib.b200rl_replay_run(hs[r], C.c_void_p(s["policy"]._d_rng), C.byref(ex), C.byref(ctl), 4, None)
    SH._in_threads([lambda r=r: go(r) for r in range(2)])
    assert codes == [L.ERR_INVALID, L.ERR_INVALID], codes
    for r in range(2):
        SH._assert_same(before[r], SH._state(pkg, ranks[r]))
    for s in ranks:
        SH._close(s)
