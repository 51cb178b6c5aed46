// ORACLE — TEST INFRASTRUCTURE ONLY (see jl_math.hpp header).
// Minibatch permutation used when the host does not supply `shuffle!(rng, 1:N*T)` itself
// (SURVEY Appendix B, PPO _update!): a keyed 4-round alternating Feistel bijection on the
// smallest power-of-two domain 2^bits >= n (bits >= 2; left half floor(bits/2) bits, the halves
// swap widths every round) with cycle walking.  A definition of this project (the reference's shuffle!
// is a sequential Fisher-Yates on one stream); DESIGN.md §K7.
#pragma once
#include <cstdint>
namespace oracle {
static inline uint32_t mix32(uint32_t h) {
    h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
    return h;
}
static inline uint32_t perm_index(uint32_t q, uint32_t n, uint32_t key) {
    int bits = 2;
    while (bits < 32 && (1u << bits) < n) ++bits;
    const int wl = bits / 2, wr = bits - wl;          // widths of the left / right half
    const uint32_t ml = (1u << wl) - 1, mr = (1u << wr) - 1;
    uint32_t x = q;
    do {
        uint32_t l = x >> wr, r = x & mr;
        for (uint32_t round = 0; round < 4; ++round) {
            // the half being rewritten has wl bits on even rounds and wr bits on odd rounds
            uint32_t t = l ^ (mix32(r + key + round * 0x9E3779B9u) & ((round & 1) ? mr : ml));
            l = r; r = t;
        }
        x = (l << wr) | r;
    } while (x >= n);
    return x;
}
}  // namespace oracle
