// common.cuh — shared host-side plumbing of libb200rl.so (ctx, error convention, handles).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/b200rl.h"

#define B200RL_ABI_VERSION 2

void b200rl_set_error(const char* fmt, ...);

#define CUDA_TRY(expr)                                                                      \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) {                                                            \
            b200rl_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return _e == cudaErrorMemoryAllocation ? B200RL_ERR_OOM : B200RL_ERR_CUDA;      \
        }                                                                                   \
    } while (0)
// CUDA_TRY inside a create: `cleanup` (the destroy of the half-built handle) runs before the error is returned
#define CUDA_TRY_OR(expr, cleanup)                                                          \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) {                                                            \
            b200rl_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            cleanup;                                                                        \
            return _e == cudaErrorMemoryAllocation ? B200RL_ERR_OOM : B200RL_ERR_CUDA;      \
        }                                                                                   \
    } while (0)

#define REQUIRE(cond, code, msg)                 \
    do {                                         \
        if (!(cond)) {                           \
            b200rl_set_error("%s: %s", __func__, msg); \
            return code;                         \
        }                                        \
    } while (0)

#define TRY(expr)                \
    do {                         \
        int _s = (expr);         \
        if (_s != B200RL_OK) return _s; \
    } while (0)

struct b200rl_comm_state;  // comm.cu

struct b200rl_ctx {
    int device = 0;
    int sm_count = 0;
    size_t l2_bytes = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    static constexpr int kTimerSlots = 512;
    cudaEvent_t slots[kTimerSlots] = {};   // b200rl_timer_record / _elapsed_ms: created on first use
    int phase_base = -1;                   // >= 0: b200rl_onpolicy_update records its phases into slots[phase_base ...] (eager path only)
    void* flush_buf = nullptr;
    size_t flush_bytes = 0;
    void* scratch = nullptr;  // general device scratch (grown on demand)
    size_t scratch_bytes = 0;
    std::vector<void*> retired;  // outgrown scratch buffers, freed with the ctx
    b200rl_comm_state* comm = nullptr;
    uint64_t launches = 0;    // kernels launched through this ctx (bench "gpu_launches")
};

int ctx_scratch(b200rl_ctx* ctx, size_t bytes, void** out);
static inline int ctx_bind(b200rl_ctx* ctx) {
    if (!ctx) { b200rl_set_error("null ctx"); return B200RL_ERR_INVALID; }
    CUDA_TRY(cudaSetDevice(ctx->device));
    return B200RL_OK;
}
#define LAUNCH_CHECK(ctx)                 \
    do {                                  \
        (ctx)->launches++;                \
        CUDA_TRY(cudaGetLastError());     \
    } while (0)

static inline unsigned grid_for(int64_t n, int block) { return (unsigned)((n + block - 1) / block); }
// Function attributes (cudaFuncAttributeMaxDynamicSharedMemorySize) are per DEVICE: a process that drives several devices
// must set them once on each.  `mask` is the call site's static bit set; true the first time `device` is seen.
static inline bool first_use_on_device(unsigned long long& mask, int device) {
    const unsigned long long bit = 1ull << (device & 63);
    if (mask & bit) return false;
    mask |= bit;
    return true;
}

// ---- NVLink peer exchange (comm.cu): low-latency PUSH protocol --------------------------------------------------
// Every rank owns an inbox region mapped into all ranks of the node.  A sender writes 8-byte packets {32 data bits,
// sequence number} straight into the receivers' inboxes (remote NVLink stores: one-way latency, no round trip); a receiver
// polls its OWN memory until the packet carries the current sequence number — the packet validates itself, so there are no
// separate flags and no fences.  Two slots (sequence & 1): a slot is rewritten two exchanges later, by which time the
// receiver has long consumed it (it had to push its own packets of the exchange in between, after finishing this one).
//   inbox_x[2][kP2PMaxRanks][kP2PXCap]   gradient words (+ 4 loss sums)     — fused reduce / exchange / clip / Adam kernel
//   inbox_y[2][kP2PMaxRanks][kP2PYCap]   small all-reduces (one word per float, two per double)
constexpr size_t kP2PXCap = 32768;
constexpr size_t kP2PYCap = 2048;
constexpr int kP2PMaxRanks = 8;
constexpr size_t kP2POffY = 2 * (size_t)kP2PMaxRanks * kP2PXCap * 8;
constexpr size_t kP2PRegionBytes = kP2POffY + 2 * (size_t)kP2PMaxRanks * kP2PYCap * 8;
struct P2PTable {   // nranks == 0: not attached
    int nranks, rank;
    unsigned char* base[kP2PMaxRanks];
    int exclusive;      // 1: every peer region lives on another device than ours (one rank per GPU).  Only then may a kernel that
                        // occupies the whole device wait for a peer inside itself (the fused K7 + optimiser step): two ranks
                        // sharing one device would deadlock, each waiting for packets of a kernel that cannot be scheduled.
};
bool b200rl_comm_p2p_table(b200rl_ctx* ctx, P2PTable* out);   // false when no peer exchange is attached
int b200rl_comm_world(b200rl_ctx* ctx);                        // ranks of the communicator (1 without one)
int b200rl_comm_rank(b200rl_ctx* ctx);                         // this ctx's rank (0 without a communicator)
bool b200rl_comm_has_nccl(b200rl_ctx* ctx);                    // the communicator has an NCCL communicator (not peer exchange only)
// device-resident sequence numbers of the peer exchanges {gradient exchange, small all-reduce}: every exchange kernel reads
// its counter, uses value + 1 and stores it back when it is done — no host-side state, so a captured CUDA graph can be replayed
unsigned int* b200rl_comm_p2p_seq_dev(b200rl_ctx* ctx);

#ifdef __CUDACC__
// packet address: inbox of rank `dst`, area (0 = x, 1 = y), slot, written by rank `src`, word index idx
__device__ __forceinline__ uint2* p2p_packet(const P2PTable& t, int dst, int area, unsigned slot, int src, size_t idx) {
    const size_t cap = area ? kP2PYCap : kP2PXCap;
    return reinterpret_cast<uint2*>(t.base[dst] + (area ? kP2POffY : 0)) + ((size_t)slot * kP2PMaxRanks + src) * cap + idx;
}
__device__ __forceinline__ void p2p_push(const P2PTable& t, int area, unsigned slot, size_t idx, unsigned bits, unsigned seq) {
    for (int r = 0; r < t.nranks; ++r) {
        if (r == t.rank) continue;
        uint2* q = p2p_packet(t, r, area, slot, t.rank, idx);
        asm volatile("st.relaxed.sys.global.v2.u32 [%0], {%1, %2};" ::"l"(q), "r"(bits), "r"(seq) : "memory");
    }
}
// spin on the own inbox until rank `src`'s packet of this exchange has landed; a peer that never arrives (crashed rank)
// traps after ~10 s instead of hanging the GPU
__device__ __forceinline__ unsigned p2p_recv(const P2PTable& t, int area, unsigned slot, int src, size_t idx, unsigned seq) {
    const uint2* q = p2p_packet(t, t.rank, area, slot, src, idx);
    unsigned long long t0 = 0;
    unsigned spins = 0;
    for (;;) {
        unsigned a, b;
        asm volatile("ld.relaxed.sys.global.v2.u32 {%0, %1}, [%2];" : "=r"(a), "=r"(b) : "l"(q) : "memory");
        if (b == seq) return a;
        if ((++spins & 1023u) == 0) {
            unsigned long long now;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (t0 == 0) t0 = now;
            else if (now - t0 > 10000000000ull) __trap();
        }
    }
}
// the exchange's sum of one element over the ranks, in rank order (bit-identical on every rank): `mine` for the own rank, the packets
// of word_idx (sizeof(T) / 4 consecutive words) from the peers.  The caller pushes its own packets first.
template <class T>
__device__ __forceinline__ T p2p_sum_ranks(const P2PTable& t, int area, unsigned slot, size_t word_idx, T mine, unsigned seq) {
    constexpr int W = sizeof(T) / 4;
    T acc = 0;
    for (int r = 0; r < t.nranks; ++r) {
        T val = mine;
        if (r != t.rank) {
            unsigned u[W];
            for (int h = 0; h < W; ++h) u[h] = p2p_recv(t, area, slot, r, word_idx + h, seq);
            memcpy(&val, u, sizeof(T));
        }
        acc += val;
    }
    return acc;
}
#endif
