// replay_schedule.h — the InsertSampleRatioController schedule of the DQN agent loop (b200rl_replay_run), computed on the host
// ahead of the launches.  Plain C++; the CPU suite compiles it and checks it against learners.InsertSampleRatioController.
#pragma once
#include <cmath>
#include <cstdint>

#include "../../include/b200rl.h"

namespace replay {

// controller values the schedule accepts: a finite ratio in [0, 1e6] and non-negative counters (a non-finite ratio would
// never stop sampling)
inline bool controller_ok(const b200rl_insert_sample_ratio& c) {
    return c.ratio >= 0.0 && c.ratio <= 1e6 && std::isfinite(c.ratio) && c.n_inserted >= 0 && c.n_sampled >= 0 &&
           c.n_inserted < (1ll << 52) && c.n_sampled < (1ll << 52);
}

// push!(trajectory) of one frame followed by optimise!: on_insert(1), then `while on_sample()` — returns the number of
// updates (batches sampled) after this insertion and advances the counters.  n_sampled <= (n_inserted - threshold) * ratio
// is compared as Float64 (exact for counters below 2^52).
inline int64_t insert_then_sample(b200rl_insert_sample_ratio& c) {
    c.n_inserted += 1;
    int64_t m = 0;
    while (c.n_inserted >= c.threshold && (double)c.n_sampled <= (double)(c.n_inserted - c.threshold) * c.ratio) {
        c.n_sampled += 1;
        m += 1;
    }
    return m;
}

}  // namespace replay
