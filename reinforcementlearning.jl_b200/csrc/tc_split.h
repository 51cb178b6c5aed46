// tc_split.h — how the tensor-core loss + backward kernel (nn_tc.cu) divides its persistent CTAs between the actor and the critic.
// Plain C++ (also compiled for the host by the CPU test suite).
#pragma once
#include <cstdint>

// CTAs given to the actor out of `grid` (the rest work on the critic).  Cost model: a critic tile costs ~0.87 of an actor tile
// with the categorical PPO / A2C loss and ~0.85 with the Gaussian head (the critic skips the softmax / log-density, entropy and
// PPO ratio); the split minimises the longer of the two roles' whole-tile counts.  The two ratios were swept on an earlier
// version of this kernel for another GPU.  On an H100 SXM (132 CTAs, 700 W) a sweep of B200RL_K7_ACTOR_CTAS over 66 .. 74 puts
// the optimum of the whole-tile hand-over kernel at 67-68 actor CTAs for bench.py c2 (the rule: 70, 3 % slower) and at 69 for c3
// (the rule: 71, 2 % slower), and that of the per-half hand-over kernel at 66 for both (the rule: 6 % / 7 % slower): critic and
// actor tiles cost about the same there.  The ratios and the splits they give are pinned by the host test of this rule.
// At most grid / 2 + 8 (the fused optimiser step stages <= 82 partial rows), at least grid / 2.
static inline int b200rl_tc_actor_ctas(int grid, bool gaussian_head, int64_t ntiles) {
    const double r = gaussian_head ? 0.85 : 0.87;
    int best = grid / 2;
    double best_cost = 1e300;
    for (int na = grid / 2; na <= grid / 2 + 8 && na < grid; ++na) {
        const double ca = (double)((ntiles + na - 1) / na), cc = r * (double)((ntiles + (grid - na) - 1) / (grid - na));
        const double cost = ca > cc ? ca : cc;
        if (cost < best_cost - 1e-9) { best_cost = cost; best = na; }
    }
    return best;
}
