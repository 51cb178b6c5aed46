"""The device episode log's write point (act_step in csrc/env_device.cuh) and its flush helpers, compiled for the host (no GPU),
against a NumPy restatement: ring wrap at K and the per-env counts, the finished-episode rule for a terminal env stepped again
without a reset, the MaxTimeoutEnv cut, and overflow detection in the flush."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))
HD = os.path.join(HERE, "hostdev")
CSRC = os.path.join(os.path.dirname(HERE), "reinforcementlearning.jl_b200", "csrc")
RECORD = np.dtype([("env", "<i8"), ("ret", "<f4"), ("len", "<i4")])


@pytest.fixture(scope="module")
def el(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("episode_log") / "libepisode_log.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-Wno-unknown-pragmas",
                           "-I", HD, "-I", CSRC, "-shared", "-o", so, os.path.join(HD, "episode_log.cpp")])
    L = C.CDLL(so)
    vp, i32, i64 = C.c_void_p, C.c_int, C.c_int64
    L.el_cartpole_run.restype, L.el_cartpole_run.argtypes = i32, [i64, i32, i32, i32, vp, i32, vp, vp, vp, vp, vp, vp, vp]
    L.el_flush.restype, L.el_flush.argtypes = i64, [i32, i64, vp, vp, vp, vp, i64, vp, i64, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Log:
    def __init__(self, K, N):
        self.K, self.N = K, N
        self.ret = np.zeros((N, K), np.float32)      # (K, N) column-major: env i's K slots are contiguous
        self.len = np.zeros((N, K), np.int32)
        self.count = np.zeros(N, np.uint32)
        self.cursor = np.zeros(N, np.uint32)


def _run(el, log, i, actions, seed, max_timeout=0, reset_mode=0):
    n = len(actions)
    rng = O.splitmix_states_fast(1, seed)[0].copy()
    rew, done, fin = np.zeros(n, np.float32), np.zeros(n, np.uint8), np.zeros(n, np.int32)
    a = np.ascontiguousarray(actions, np.int32)
    el.el_cartpole_run(i, log.K, max_timeout, reset_mode, _p(a), n, _p(rng), _p(log.ret), _p(log.len), _p(log.count), _p(rew), _p(done), _p(fin))
    return rew, done.astype(bool), fin


def _restate(rew, done, reset_mode):
    """the episodes a run finishes, in order: (Float32 step-order return, env.t at the end).  reset_mode 2 steps a terminal env
    again without a reset: that step is no new episode and t runs on."""
    eps, ret, t, terminal = [], np.float32(0), 0, False
    for r, d in zip(rew, done):
        if terminal and reset_mode == 1:
            t, terminal = 0, False
        t += 1
        ret = np.float32(ret + r)
        if d and not (terminal and reset_mode == 2):
            eps.append((ret, t))
        if d:
            ret = np.float32(0)
            if reset_mode == 0:
                t = 0
        terminal = bool(d)
    return eps


def _ring(eps, K):
    """what a ring of K slots holds after the episodes eps: slot c % K = episode c"""
    ret, ln = np.zeros(K, np.float32), np.zeros(K, np.int32)
    for c, (r, n) in enumerate(eps):
        ret[c % K], ln[c % K] = r, n
    return ret, ln


@pytest.mark.parametrize("reset_mode", [0, 1, 2])
@pytest.mark.parametrize("max_timeout", [0, 17])
@pytest.mark.parametrize("K", [1, 3, 64])
def test_log_write_matches_restatement(el, reset_mode, max_timeout, K):
    N = 4
    log = Log(K, N)
    rng = np.random.default_rng(K * 100 + max_timeout + reset_mode)
    for i in range(N):
        rew, done, fin = _run(el, log, i, rng.integers(1, 3, 400), seed=i + 7, max_timeout=max_timeout, reset_mode=reset_mode)
        eps = _restate(rew, done, reset_mode)
        assert len(eps) > K or K == 64 or reset_mode == 2
        assert log.count[i] == len(eps) == fin.sum()          # the log counts what the episode tally counts
        ret, ln = _ring(eps, K)
        m = min(len(eps), K)
        filled = np.sort(np.arange(len(eps))[-m:] % K)
        assert np.array_equal(log.ret[i, filled].view(np.uint32), ret[filled].view(np.uint32))
        assert np.array_equal(log.len[i, filled], ln[filled])


def test_terminal_env_stepped_again_is_not_a_new_episode(el):
    log = Log(8, 1)
    actions = np.full(60, 2, np.int32)     # push right until the cart leaves the track, then keep stepping the terminal env
    rew, done, fin = _run(el, log, 0, actions, seed=3, reset_mode=2)
    first = int(np.argmax(done))
    assert done[first:first + 5].all()     # the env stays terminal ...
    assert log.count[0] == 1               # ... and only its first terminal step is an episode
    assert log.len[0, 0] == first + 1 and log.ret[0, 0] == np.float32(first)


def test_max_timeout_cut_ends_the_episode(el):
    log = Log(64, 1)
    M = 12
    rng = np.random.default_rng(5)
    rew, done, fin = _run(el, log, 0, rng.integers(1, 3, 300), seed=11, max_timeout=M, reset_mode=0)
    n = int(log.count[0])
    lens, rets = log.len[0, :n], log.ret[0, :n]
    ends = np.nonzero(done)[0]
    cut = rew[ends] == 1        # the cut keeps the wrapped env's reward: CartPole pays 1 on a step where the pole is still up
    assert n == len(ends) >= 300 // M and cut.sum() > n // 2 and (~cut).any()
    assert (lens[cut] == M).all() and (lens <= M).all()
    assert np.array_equal(rets, (lens - ~cut).astype(np.float32))   # 1 per step, but 0 on the step a pole falls


def _flush(el, log, global0=0, capacity=None):
    cap = log.N * log.K if capacity is None else capacity
    out = np.zeros(max(cap, 1), RECORD)
    over = np.zeros(1, np.int64)
    n = el.el_flush(log.K, log.N, _p(log.ret), _p(log.len), _p(log.count), _p(log.cursor), global0, _p(out), cap, _p(over))
    return out[:min(n, cap)], n, int(over[0])


def test_flush_orders_by_env_then_episode_and_advances_cursors(el):
    K, N = 4, 6
    log = Log(K, N)
    rng = np.random.default_rng(9)
    log.ret[:] = rng.standard_normal((N, K)).astype(np.float32)
    log.len[:] = rng.integers(1, 200, (N, K))
    log.cursor[:] = np.array([0, 5, 2**32 - 2, 7, 3, 0], np.uint32)
    log.count[:] = (log.cursor.astype(np.uint64) + np.array([3, 4, 3, 0, 1, 0])) % 2**32   # env 2's counters wrap past 2^32
    pend = (log.count - log.cursor).astype(np.int64)
    want = [(1000 + i, log.ret[i, c % K], log.len[i, c % K]) for i in range(N) for c in (int(log.cursor[i]) + e for e in range(pend[i]))]
    count0 = log.count.copy()
    got, n, over = _flush(el, log, global0=1000)
    assert over == 0 and n == pend.sum() == len(want)
    assert [tuple(r) for r in got.tolist()] == [(g, float(r), int(ln)) for g, r, ln in want]
    assert np.array_equal(log.cursor, count0)
    got, n, over = _flush(el, log)        # nothing new since: an empty list
    assert n == 0 and over == 0


def test_flush_detects_overflow(el):
    K, N = 3, 4
    log = Log(K, N)
    rng = np.random.default_rng(2)
    for i in range(N):                    # env 1 and 3 run long enough to finish more than K episodes
        _run(el, log, i, rng.integers(1, 3, 250 if i % 2 else 20), seed=40 + i, max_timeout=10)
    assert log.count[1] > K and log.count[3] > K and log.count[0] <= K and log.count[2] <= K
    got, n, over = _flush(el, log)
    assert over == 2
    assert n == log.count[0] + log.count[2] + 2 * K
    assert np.array_equal(log.cursor, log.count)   # the flush still moves on: the next window starts clean
    _run(el, log, 0, rng.integers(1, 3, 20), seed=99, max_timeout=10)
    got, n, over = _flush(el, log)
    assert over == 0 and n > 0 and (got["env"] == 0).all()
