"""NumPy restatement of the n-step sampler (NStepBatchSampler(n, γ); DESIGN.md §3), written from the rules rather than from
csrc/nstep.cuh, plus a host model of the per-lane replay ring to build synthetic rings from push calls.

Ring arrays are those of Trajectory.export_state(): state (ns, lanes, cap+1) f32, reward / flag (lanes, cap+1), all flat with the
lane index fastest; entry key = slot * lanes + lane; flag bit0 terminal, bit1 sampleable."""
import numpy as np

TERMINAL, SAMPLEABLE = 1, 2


def window(flag, reward, lanes, cap, key, n, gamma):
    """(G, terminal, next slot, discount, m) of the entry `key`: the entries of its lane from `key` on, up to n of them, cut after
    a terminal entry and before an entry that is not sampleable."""
    F = cap + 1
    slot, e = divmod(int(key), lanes)
    taken = [slot]
    while len(taken) < n and not flag[taken[-1] * lanes + e] & TERMINAL:
        nxt = (taken[-1] + 1) % F
        if not flag[nxt * lanes + e] & SAMPLEABLE:
            break
        taken.append(nxt)
    g = np.float32(gamma)
    G = np.float32(reward[taken[-1] * lanes + e])
    for s in reversed(taken[:-1]):                    # discount_rewards' order: G = r + γ·G from the back, each op rounded
        G = np.float32(np.float32(reward[s * lanes + e]) + np.float32(g * G))
    d = np.float32(1.0)
    for _ in taken:                                   # γ^m as m left-to-right Float32 products
        d = np.float32(d * g)
    return G, int(flag[taken[-1] * lanes + e] & TERMINAL), (taken[-1] + 1) % F, d, len(taken)


def nstep_batch(st, ns, lanes, cap, keys, n, gamma):
    """reward / terminal / next_state / discount / horizon of the batch with these keys, from exported ring arrays"""
    state, reward, flag = np.asarray(st["state"], np.float32), np.asarray(st["reward"], np.float32), np.asarray(st["flag"], np.uint8)
    B = len(keys)
    out = dict(reward=np.empty(B, np.float32), terminal=np.empty(B, np.uint8), next_state=np.empty((ns, B), np.float32, order="F"),
               discount=np.empty(B, np.float32), horizon=np.empty(B, np.int32))
    for k, key in enumerate(keys):
        G, t, nslot, d, m = window(flag, reward, lanes, cap, key, n, gamma)
        e = int(key) % lanes
        out["reward"][k], out["terminal"][k], out["discount"][k], out["horizon"][k] = G, t, d, m
        out["next_state"][:, k] = state[ns * (nslot * lanes + e): ns * (nslot * lanes + e) + ns]
    return out


class HostRing:
    """The per-lane ring's push semantics (EpisodesBuffer bookkeeping per lane) on the host, for synthetic rings."""

    def __init__(self, ns, lanes, cap):
        self.ns, self.lanes, self.cap, F = ns, lanes, cap, cap + 1
        self.state = np.zeros(ns * lanes * F, np.float32)
        self.reward = np.zeros(lanes * F, np.float32)
        self.action = np.zeros(lanes * F, np.int32)
        self.flag = np.zeros(lanes * F, np.uint8)
        self.head = np.zeros(lanes, np.int64)
        self.count = np.zeros(lanes, np.int64)
        self.pending = np.zeros(lanes, np.uint8)

    def _write(self, slot, e, obs):
        k = slot * self.lanes + e
        self.flag[k] = 0                                   # the entry that started at this frame is gone
        self.state[self.ns * k: self.ns * k + self.ns] = obs

    def push_episode_start(self, obs, pending_only=False):
        F = self.cap + 1
        for e in range(self.lanes):
            if pending_only and not self.pending[e]:
                continue
            self._write(self.head[e], e, obs[:, e])
            self.head[e] = (self.head[e] + 1) % F
            self.count[e] = min(self.count[e] + 1, F)
            self.pending[e] = 0

    def push(self, a, r, t, next_obs):
        """t: bit0 terminal, bit1 the env auto-reset (next_obs is also the next episode's first frame)"""
        F = self.cap + 1
        for e in range(self.lanes):
            h = self.head[e]
            p = (h + F - 1) % F
            self.action[p * self.lanes + e] = a[e]
            self.reward[p * self.lanes + e] = r[e]
            self.flag[p * self.lanes + e] = (t[e] & TERMINAL) | SAMPLEABLE
            self._write(h, e, next_obs[:, e])
            nh, cnt, pend = (h + 1) % F, min(self.count[e] + 1, F), 0
            if t[e] & TERMINAL:
                if t[e] & 2:
                    self._write(nh, e, next_obs[:, e])
                    nh, cnt = (nh + 1) % F, min(cnt + 1, F)
                else:
                    pend = 1
            self.head[e], self.count[e], self.pending[e] = nh, cnt, pend

    def export(self):
        return dict(state=self.state, reward=self.reward, flag=self.flag, action=self.action)

    def sampleable_keys(self):
        return np.flatnonzero(self.flag & SAMPLEABLE)
