// ORACLE — TEST INFRASTRUCTURE ONLY (see jl_math.hpp header).
//
// CPU restatement of the trajectory container + samplers on the hot path (SURVEY §8 row a11).
// The upstream code lives in the registered package ReinforcementLearningTrajectories
// (compat "0.4", RLCore/Project.toml:20,40) + CircularArrayBuffers ("0.1.12"), which is NOT
// vendored under /root/reference and has no Manifest pin -> PARITY UNPINNED.  What is
// restated is the published behaviour recorded in SURVEY Appendix B, anchored on the
// reference's own call sites and boundary tests:
//   push order / trace layout   RLCore/src/policies/agent/agent_base.jl:45-59,
//                               agent_srt_cache.jl:30-50, docs/src/How_to_implement_a_new_algorithm.md:84-112
//   length semantics            RLCore/test/policies/agent.jl:27-34 (0 after the first state, 1 after the first transition)
//   iteration tuple             RLCore/test/policies/q_based_policy.jl:40-58 (state,next_state,action,reward,terminal)
//   EpisodesBuffer length       RLCore/test/core/base.jl:20 (length(container) == steps + episodes - 1: the first state of every episode
//                               is a frame of its own; the entry straddling two episodes exists but is not sampleable)
// Layout: `lanes` independent rings of cap+1 slots (lanes = 1 is exactly the reference's single-stream CircularArraySARTSTraces wrapped
// in an EpisodesBuffer).  Entry p of a lane is the transition state[p] -> state[p+1] (MultiplexTraces).  Samplers draw WITH
// replacement (BatchSampler) from one Xoshiro stream per batch slot (a definition of this project: the reference draws the whole batch from
// a single stream).  A terminal bit 1 in push() means "next_obs already is the next episode's first state" (the batched env's in-kernel
// auto-reset): it is stored twice, as the masked :next_state and as the episode-start frame.
#pragma once
#include <cmath>
#include <cstdint>
#include <vector>

#include "jl_rng.hpp"

namespace oracle {

struct SumTree {  // leaves [L, 2L), node k = node 2k + node 2k+1, float32 sums
    int64_t L = 1;
    std::vector<float> tree;
    void init(int64_t n_slots) {
        L = 1;
        while (L < n_slots) L <<= 1;
        tree.assign(2 * L, 0.f);
    }
    float total() const { return tree[1]; }
    void set(int64_t slot, float p) {
        int64_t k = L + slot;
        tree[k] = p;
        for (k >>= 1; k >= 1; k >>= 1) tree[k] = tree[2 * k] + tree[2 * k + 1];
    }
    int64_t find(float v) const {   // never steps into an empty subtree: rounding cannot land on a zero-priority leaf
        int64_t k = 1;
        while (k < L) {
            int64_t l = 2 * k;
            float tl = tree[l], tr = tree[l + 1];
            if (tl > 0.f && (v < tl || !(tr > 0.f))) k = l;
            else { v -= tl; k = l + 1; }
        }
        return k - L;
    }
};

struct Traj {
    int ns;
    int64_t lanes, cap;       // cap sampleable transitions per lane at most; cap+1 slots
    std::vector<float> state;     // (ns, lanes, cap+1)
    std::vector<int32_t> action;  // (lanes, cap+1)
    std::vector<float> reward;    // (lanes, cap+1)
    std::vector<uint8_t> flag;    // bit0 terminal, bit1 sampleable
    std::vector<int32_t> head, count;
    std::vector<uint8_t> pending;
    int64_t n_valid = 0;
    bool prioritized = false;
    float default_priority = 1.f;
    SumTree st;

    Traj(int ns_, int64_t lanes_, int64_t cap_, bool prio, float defp)
        : ns(ns_), lanes(lanes_), cap(cap_), state((size_t)ns_ * lanes_ * (cap_ + 1)), action(lanes_ * (cap_ + 1)),
          reward(lanes_ * (cap_ + 1)), flag(lanes_ * (cap_ + 1), 0), head(lanes_, 0), count(lanes_, 0), pending(lanes_, 0), prioritized(prio),
          default_priority(defp) {
        if (prio) st.init(lanes * (cap + 1));
    }
    int64_t frames() const { return cap + 1; }
    int64_t length(int64_t lane = 0) const { return count[lane] > 0 ? count[lane] - 1 : 0; }  // entries, sampleable or not
    void write_state(int64_t slot, int64_t e, const float* obs) {
        for (int k = 0; k < ns; ++k) state[(size_t)ns * (slot * lanes + e) + k] = obs[(size_t)ns * e + k];
    }
    void destroy(int64_t slot, int64_t e) {   // the state at `slot` is overwritten: the entry starting there is gone
        int64_t k = slot * lanes + e;
        if (flag[k] & 2) n_valid -= 1;
        flag[k] = 0;
        if (prioritized) st.set(k, 0.f);
    }
    // push!(trajectory, (state = s0,)) — agent_base.jl:45-47.  mode 0: every lane; 1: lanes whose last transition was terminal
    void push_episode_start(const float* obs, int mode) {
        int64_t F = frames();
        for (int64_t e = 0; e < lanes; ++e) {
            if (mode == 1 && !pending[e]) continue;
            int64_t h = head[e];
            destroy(h, e);
            write_state(h, e, obs);
            head[e] = (int32_t)((h + 1) % F);
            count[e] = (int32_t)std::min<int64_t>(count[e] + 1, F);
            pending[e] = 0;
        }
    }
    void push_state(const float* obs) { push_episode_start(obs, 0); }
    // push!(trajectory, (state = s', action, reward, terminal)) — agent_base.jl:56-59
    void push(const int32_t* a, const float* r, const uint8_t* t, const float* next_obs) {
        int64_t F = frames();
        for (int64_t e = 0; e < lanes; ++e) {
            int64_t h = head[e], p = (h + F - 1) % F;
            action[p * lanes + e] = a[e];
            reward[p * lanes + e] = r[e];
            flag[p * lanes + e] = (uint8_t)((t[e] & 1) | 2);
            n_valid += 1;
            if (prioritized) st.set(p * lanes + e, default_priority);
            destroy(h, e);
            write_state(h, e, next_obs);
            int64_t nh = (h + 1) % F;
            int64_t cnt = std::min<int64_t>(count[e] + 1, F);
            uint8_t pend = 0;
            if (t[e] & 1) {
                if (t[e] & 2) {
                    destroy(nh, e);
                    write_state(nh, e, next_obs);
                    nh = (nh + 1) % F;
                    cnt = std::min<int64_t>(cnt + 1, F);
                } else {
                    pend = 1;
                }
            }
            head[e] = (int32_t)nh; count[e] = (int32_t)cnt; pending[e] = pend;
        }
    }
    // gather one transition by key = slot * lanes + lane
    void gather(int64_t key, float* s, int32_t* a, float* r, uint8_t* t, float* s2) const {
        int64_t slot = key / lanes, e = key % lanes, nslot = (slot + 1) % frames();
        for (int k = 0; k < ns; ++k) {
            s[k] = state[(size_t)ns * (slot * lanes + e) + k];
            s2[k] = state[(size_t)ns * (nslot * lanes + e) + k];
        }
        *a = action[key];
        *r = reward[key];
        *t = flag[key] & 1;
    }
};

// BatchSampler: slot k draws rand(rng_k, 1:lanes*cap) until it hits a sampleable entry (uniform over the sampleable entries, with replacement)
static inline void sample_uniform(const Traj& tr, jl::Xoshiro* slots, int64_t B, int64_t* key_out) {
    uint64_t n = (uint64_t)(tr.lanes * tr.cap);
    int64_t F = tr.frames();
    for (int64_t k = 0; k < B; ++k) {
        key_out[k] = -1;
        for (int tries = 0; tries < 4096; ++tries) {
            int64_t q = jl::rand_oneto(slots[k], n) - 1;
            int64_t e = q % tr.lanes, j = q / tr.lanes, cnt = tr.count[e];
            if (j >= cnt - 1) continue;
            int64_t slot = ((int64_t)tr.head[e] - cnt + j + 2 * F) % F;
            if (tr.flag[slot * tr.lanes + e] & 2) { key_out[k] = slot * tr.lanes + e; break; }
        }
    }
}
// prioritised: slot k draws v = rand(rng_k, Float32) * total and descends the sum tree;
// weights w = (n * p / total)^(-beta) / max_k w, n = number of sampleable entries   (SURVEY Appendix B, PrioritizedDQN)
static inline void sample_prioritized(const Traj& tr, jl::Xoshiro* slots, int64_t B, float beta, int64_t* key_out, float* prio_out, float* w_out) {
    float total = tr.st.total();
    float wmax = 0.f;
    for (int64_t k = 0; k < B; ++k) {
        float v = jl::rand_f32(slots[k]) * total;
        int64_t key = tr.st.find(v);
        float p = tr.st.tree[tr.st.L + key];
        key_out[k] = key;
        prio_out[k] = p;
        float w = std::pow((float)tr.n_valid * (p / total), -beta);
        w_out[k] = w;
        wmax = std::max(wmax, w);
    }
    for (int64_t k = 0; k < B; ++k) w_out[k] = w_out[k] / wmax;
}

}  // namespace oracle
