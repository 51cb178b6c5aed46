// ring.cuh — the per-lane push! of the device replay ring (CircularArraySARTSTraces with EpisodesBuffer bookkeeping per lane;
// layout and semantics: traj.cu's header comment).  push_sart_kernel / push_episode_start_kernel (traj.cu) and the fused DQN
// collect kernel (fwd_tc.cu) run these functions, so a push writes the same slots, flags, counters and leaf values everywhere.
#pragma once
#include <cstdint>

struct Ring {
    int ns;
    int64_t lanes, cap;
    float* state; int32_t* action; float* reward; uint8_t* flag;
    int32_t* head;       // (lanes) next slot to write
    int32_t* count;      // (lanes) state frames stored, <= cap + 1
    uint8_t* pending;    // (lanes) the last stored transition was terminal and its episode-start frame has not been pushed yet
    long long* n_valid;  // (1) sampleable entries over all lanes
    float* tree; int64_t L;
    __host__ __device__ int64_t frames() const { return cap + 1; }
};
constexpr uint8_t kRingTerminal = 1, kRingSampleable = 2;

// sum-tree leaves a push rewrites (key -1 = none): the caller applies them (key lists for tree_update_keys_kernel, or directly)
struct RingLeaves { int64_t key[3]; float val[3]; };

#ifdef __CUDACC__
namespace ring {

__device__ __forceinline__ void write_state(const Ring& r, int64_t slot, int64_t e, const float* src) {
    float* dst = r.state + (int64_t)r.ns * (slot * r.lanes + e);
    for (int c = 0; c < r.ns; ++c) dst[c] = src[c];
}
// the state frame at `slot` is about to be overwritten: the entry that started there is gone
__device__ __forceinline__ int destroy_entry(const Ring& r, int64_t slot, int64_t e) {
    const int64_t k = slot * r.lanes + e;
    const int was = (r.flag[k] & kRingSampleable) ? 1 : 0;
    r.flag[k] = 0;
    return was;
}
// push!(trajectory, (state = s0,)) of lane e; obs = its ns state values.  Returns the change of the sampleable count.
__device__ __forceinline__ long long push_episode_start(const Ring& r, int64_t e, const float* obs, RingLeaves& lv) {
    lv.key[0] = -1; lv.key[1] = -1; lv.key[2] = -1;
    const int64_t F = r.frames();
    const int64_t h = r.head[e];
    const int lost = destroy_entry(r, h, e);
    write_state(r, h, e, obs);
    lv.key[0] = h * r.lanes + e; lv.val[0] = 0.f;
    r.head[e] = (int32_t)((h + 1) % F);
    r.count[e] = (int32_t)min((int64_t)r.count[e] + 1, F);
    r.pending[e] = 0;
    return lost ? -1 : 0;
}
// push!(trajectory, (state = s', action, reward, terminal)) of lane e.  t: bit0 terminal, bit1 "the env has already
// auto-reset: next_obs is the first state of the next episode" (the env's FLAGS byte) -> the episode-start frame is written
// too.  next_obs = the lane's ns state values.  Returns the change of the sampleable count; *advanced = frames written.
__device__ __forceinline__ long long push_sart(const Ring& r, int64_t e, int32_t a, float rew, uint8_t t, const float* next_obs,
                                               float default_priority, RingLeaves& lv, int* advanced) {
    const int64_t F = r.frames();
    const int64_t h = r.head[e];
    const int64_t p = (h + F - 1) % F;                 // slot of the state the action was taken in
    r.action[p * r.lanes + e] = a;
    r.reward[p * r.lanes + e] = rew;
    r.flag[p * r.lanes + e] = (uint8_t)((t & kRingTerminal) | kRingSampleable);
    long long dv = 1;
    dv -= destroy_entry(r, h, e);
    write_state(r, h, e, next_obs);
    int64_t nh = (h + 1) % F;
    int cnt = (int)min((int64_t)r.count[e] + 1, F);
    lv.key[0] = p * r.lanes + e; lv.val[0] = default_priority;
    lv.key[1] = h * r.lanes + e; lv.val[1] = 0.f;
    lv.key[2] = -1;
    int adv = 1;
    uint8_t pend = 0;
    if (t & kRingTerminal) {
        if (t & 2) {                                   // auto-reset: next_obs doubles as the episode-start frame
            dv -= destroy_entry(r, nh, e);
            write_state(r, nh, e, next_obs);
            lv.key[2] = nh * r.lanes + e; lv.val[2] = 0.f;
            nh = (nh + 1) % F;
            cnt = (int)min((int64_t)cnt + 1, F);
            adv = 2;
        } else {
            pend = 1;                                  // the caller pushes the episode start once the env has been reset
        }
    }
    r.head[e] = (int32_t)nh;
    r.count[e] = cnt;
    r.pending[e] = pend;
    if (advanced) *advanced = adv;
    return dv;
}

}  // namespace ring
#endif
