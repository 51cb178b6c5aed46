// nn_tc.cu — K7 on tensor cores (Hopper wgmma): PPO / A2C loss + backward for H = 64.
//
// The 64 x 64 layers are [128 samples x 64] x [64 x 64] GEMMs per tile, run by one MMA warpgroup with wgmma (both operands in
// shared memory, SWIZZLE_NONE canonical layout, see wgmma.cuh) into FP32 registers; it hands the results to the worker warps
// through shared memory.  Parity needs ~FP32 accuracy (1e-5 relative on losses), which no single tensor-core input format
// gives, so every product is a 3-term split
//     A*B ~= A_hi*B_hi + A_hi*B_lo + A_lo*B_hi,   x_hi = fp16(x * S), x_lo = fp16(x * S - x_hi)      (22 mantissa bits)
// with a power-of-two scale S per operand (exact; undone on the FP32 accumulator), accumulated in FP32.  fp16 covers K = 16 per
// instruction at the same 2^-22 product accuracy as a tf32 split at K = 8.  fp16 has 5 exponent bits: activations
// must stay below 65504 in magnitude (scale 1), weights below 1023 (scale 64); gradients are scaled by ~1/(4 inv_B) at launch.
// The forward's relu H1 is an operand at scale 64: from H1 = 1023.75 on it rounds to inf, and every head output of that sample
// comes out NaN (tc_fwd.cuh act2_f), not finite and wrong.
// Below 6e-5 the lo part is subnormal: absolute error <= 2^-25 per element, far inside the 1e-5 bar.  Layer 1 (K <= 4) and the
// heads (N <= 2) stay on FFMA.  The forward-only kernels (policy inference, fused rollout) live in fwd_tc.cu (same split).
#include "nn.cuh"
#include "perm.cuh"
#include "policy.cuh"
#include "tc_fwd.cuh"
#include "tc_split.h"
#include "wgmma.cuh"

namespace {

// the W2 operand image and the fp16 split of the tensor-core forward (tc_fwd.cuh)
using tcfwd::G_F;
using tcfwd::GW_S;
using tcfwd::WIMG_BYTES;
using tcfwd::split2;
using tcfwd::wimg_off;
constexpr int TM = tcfwd::TM;        // samples per tile = two wgmma M = 64 blocks
constexpr int H = tcfwd::H;
constexpr float kScaleW = tcfwd::kScale;   // power-of-two operand scales (see the header comment)

// =====================================================================================================
// K7 on tensor cores: PPO / A2C loss + backward for one minibatch, all four tile GEMMs on wgmma.
//   GEMM1  H2pre[s][o] = sum_i H1[s][i]  W2[o][i]     A = H1 image (K-major), B = W2 image (K-major)
//   GEMM2  dH1[s][i]   = sum_j dP2[s][j] W2[j][i]     A = dP2 image (K-major view of dP2^T), B = the W2 image read MN-major
//   GEMM3  dW2[j][i]  += sum_s dP2[s][j] H1[s][i]     A = dP2^T, B = H1^T (and the 1.0 column of x^T for db2): feature-major images (MN-major)
//   GEMM4  dW1 | db1  += sum_s dP1[s][f] [x | 1][s]   A = dP1^T, B = [x | 1]^T (MN-major)
// every product the 3-term fp16 split (hi*hi + hi*lo + lo*hi), FP32 accumulate.  GEMM3 / GEMM4 reduce over the tile's samples;
// the MMA warpgroup adds their results into FP32 shared-memory accumulators (round-to-nearest adds, fixed owner per entry).
// One CTA per SM (640 threads, actor or critic), persistent, software-pipelined across tiles (see the loop).
// Thread <-> data (workers): warp w: sample quadrant q = w % 4, feature block c = w / 4; thread = sample s = 32q + lane.
constexpr int NT7 = 512;
// the fused optimiser step stages the CTA's slice of every partial row through registers: at most kMaxStage floats per worker thread
// (10 * 512 >= 64 * 74 with the BASELINE network; nn_tc_step_fits)
constexpr int kMaxStage = 10;
// The activation images: element (feature f, sample s) at
//     (f / 8) * GS_T + (s / 8) * GF_T + (s % 8) * 16 + (f % 8) * 2
// i.e. [feature block of 8][sample][8 features]: thread = sample writes 8 features as ONE 16-byte vector, and the 32 lanes of a
// warp cover 512 contiguous bytes (no bank conflicts).  Read MN-major (MN = feature, K = sample: LBO = GF_T, SBO = GS_T) they
// are the operands of GEMM3 / GEMM4; read K-major (M = sample, K = feature: LBO = GS_T, SBO = GF_T) those of GEMM1 / GEMM2.
constexpr int GF_T = 128;                 // stride between 8-sample groups
constexpr int GS_T = 16 * GF_T;           // stride between 8-feature blocks (128 samples)
constexpr int FIMG = 8 * GS_T;            // [64 features x 128 samples] fp16 = 16 KB
constexpr float kScaleH = 64.0f, kScaleX = 64.0f;   // power-of-two scales of the H1 / observation operands (weights: kScaleW)
// Row stride of the GEMM3 accumulators in shared memory: 72 = 8 (mod 32), so the fragment's owner threads, reading and writing
// 8-byte column pairs, hit 16 different bank pairs per half-warp (a stride of 65 put up to 4 lanes on one bank)
constexpr int kAccW2S = 72;
constexpr int kNo = 2;   // head outputs this kernel handles (nn_tc_bwd_supported: actor n_out <= 2, critic n_out = 1)

struct SmemBwd {
    static_assert(FIMG % 128 == 0 && WIMG_BYTES % 128 == 0 && (2 * GS_T) % 16 == 0, "operand images must stay 128-byte aligned");
    alignas(128) uint8_t FP_full[FIMG];    // dP2^T hi (rows = feature j, K = sample), fp16
    alignas(128) uint8_t FP_lo[FIMG];
    // H1 hi | lo by CTA-local tile parity, written by layer1(): the A operand of GEMM1 read K-major, the B operand of GEMM3 read
    // MN-major (the same bytes), and H1 for the tanh branch of the GEMM2 epilogue
    alignas(128) uint8_t AH[2][2][FIMG];
    alignas(128) uint8_t FQ_full[FIMG];    // dP1^T hi | lo: A operand of GEMM4, written by the MMA warpgroup from GEMM2's accumulators
    alignas(128) uint8_t FQ_lo[FIMG];
    alignas(128) uint8_t B1[WIMG_BYTES];   // rows 0..63: hi, 64..127: lo of (n = out o, k = in i)  = 64 W2[o + 64 i]
    // B operand of GEMM4, double-buffered by tile parity (written at publish time, read by the GEMM3 / GEMM4 of the same tile):
    // features 0..3 = x_i hi, 4 = 1.0 (-> db1, and db2 in GEMM3), 8..11 = x_i lo, the rest 0;  K = sample
    alignas(128) uint8_t XT[2][2 * GS_T];
    alignas(16) float D[TM * H];           // FP32 result of GEMM1 for the workers (d_off layout)
    // relu trunks: bit f = (H1[s][f] > 0) of sample s, by tile parity (written by layer1(), read by the GEMM2 epilogue: act'(H1));
    // the sign is not recoverable from the fp16 image (hi > 0 and H1 > 0 differ for tiny positive H1)
    uint64_t H1pos[2][TM];
    float W1[kInMax * H];
    float b1[H], b2[H];
    float W3[H * kNo];                     // [feature][head output]
    float b3[kNo];
    float Zp[4 * kNo * TM];                // head partials [c][o][s]
    float Red[32];
    double RedD[16];
    float step_scale;
    alignas(8) uint64_t bar1[2];           // per 64-sample half
    alignas(8) uint64_t bar3;
    alignas(8) uint64_t bar4;
    alignas(8) float AccW2[64 * kAccW2S + 64];        // FP32 accumulators of GEMM3: dW2[j][i] at j * kAccW2S + i, then db2[j] (all still operand-scaled)
    float AccD4[64 * 9];                   // ... of GEMM4: dW1[f][i] at f * 9 + i, db1[f] at f * 9 + 4
};
// D[s][col] (floats): 16-byte units XOR-swizzled by the sample, so that 8 consecutive samples read at the same column hit 8
// different bank groups
__device__ __forceinline__ int d_off(int s, int col) { return s * H + ((((col >> 2) ^ (s & 15))) << 2) + (col & 3); }
__device__ __forceinline__ void d_ld16(const float* D, int s, int f0, float (&v)[16]) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const float4 q4 = *reinterpret_cast<const float4*>(D + d_off(s, f0 + 4 * u));
        v[4 * u] = q4.x; v[4 * u + 1] = q4.y; v[4 * u + 2] = q4.z; v[4 * u + 3] = q4.w;
    }
}
// MMA warpgroup: samples 64h .. 64h+63 of a [128 samples x 64] A image pair (hi, lo; K-major view of an F image) times the W2
// image (TB = 0: K-major, GEMM1; TB = 1: MN-major, GEMM2; b_step = bytes its descriptor advances per K = 16 step), the three
// split terms accumulated into the same registers
template <int TB>
__device__ __forceinline__ void gemm_ts3(float (&d)[32], const uint8_t* a_hi, const uint8_t* a_lo, int h, uint64_t dB, uint32_t b_step) {
    const uint64_t dA = wg::make_desc(wg::smem_u32(a_hi) + 8 * h * GF_T, GS_T, GF_T), dAl = wg::make_desc(wg::smem_u32(a_lo) + 8 * h * GF_T, GS_T, GF_T);
    wg::fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint32_t aa = k * 2 * GS_T, bb = k * b_step;
        wg::mma_m64n64k16<0, TB>(d, wg::desc_add(dA, aa), wg::desc_add(dB, bb), k ? 1u : 0u);
        wg::mma_m64n64k16<0, TB>(d, wg::desc_add(dA, aa), wg::desc_add(dB, 8 * GW_S + bb), 1u);   // W2 lo: rows 64..127 of the image
        wg::mma_m64n64k16<0, TB>(d, wg::desc_add(dAl, aa), wg::desc_add(dB, bb), 1u);
    }
    wg::commit();
    wg::wait_all();
}
__device__ __forceinline__ uint32_t fimg_off(int f, int s) { return (uint32_t)((f >> 3) * GS_T + (s >> 3) * GF_T + (s & 7) * 16 + (f & 7) * 2); }
// 16 features (8 packed fp16 pairs) of sample s, starting at feature f0 (a multiple of 16): two 16-byte vectors
__device__ __forceinline__ void store16_feat(uint8_t* img, int f0, int s, const uint32_t (&v)[8]) {
    uint8_t* p = img + fimg_off(f0, s);
    *reinterpret_cast<uint4*>(p) = make_uint4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<uint4*>(p + GS_T) = make_uint4(v[4], v[5], v[6], v[7]);
}
using b200perm::perm_index;
using b200perm::perm_index_bits;

// sum over the 32 lanes of NV values each (NV a power of two <= 32... here 32): lane L ends with the totals of
// values 2L*(NV/64).. — for NV = 32: lane L holds the total of value index L in v[0].
__device__ __forceinline__ float lane_transpose_reduce32(float (&v)[32], int lane) {
#pragma unroll
    for (int st = 0; st < 5; ++st) {
        const int half = 16 >> st, off = 16 >> st;
        const bool upper = (lane & off) != 0;
#pragma unroll
        for (int n = 0; n < half; ++n) {
            float send = upper ? v[n] : v[n + half];
            float keep = upper ? v[n + half] : v[n];
            v[n] = keep + __shfl_xor_sync(0xffffffffu, send, off);
        }
    }
    return v[0];   // value index = lane
}

// worker-only barrier (the MMA warpgroup never joins it)
__device__ __forceinline__ void worker_sync() { asm volatile("bar.sync 1, 512;" ::: "memory"); }
// barrier of the four warps that share one sample quadrant q (= one 32-sample slice of the tile, feature blocks c = 0..3).
// Everything the workers exchange per tile (X, Aux, Zp, the D entries of a sample) is exchanged between the four threads of ONE
// sample, i.e. inside such a group, so the per-tile barriers are group-local (ids 5..8, 128 threads) and the four groups — one
// per warp scheduler — drift freely within a tile; the tensor-core hand-overs (bar.arrive) and the mbarrier waits bound the drift.
__device__ __forceinline__ void group_sync(int q) { asm volatile("bar.sync %0, 128;" ::"r"(5 + q) : "memory"); }
// operand hand-over of one 64-sample half to the MMA warpgroup: the 256 worker threads of quadrants 2h, 2h+1 arrive without
// waiting, its 128 threads wait
__device__ __forceinline__ void ready_arrive(int id) { asm volatile("bar.arrive %0, 384;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void ready_wait(int id) { asm volatile("bar.sync %0, 384;" ::"r"(id) : "memory"); }
#ifdef B200RL_K7_TIMING   // debug build only: per-phase cycle sums seen by one watched worker thread
__device__ unsigned long long g_k7_phase[40];
__device__ int g_k7_watch = 0;   // watched worker thread (low 16 bits) of CTA (high bits; CTAs below n_actor = actor) whose timeline is recorded
#define K7_T(i) do { if (tid == (g_k7_watch & 0xFFFF) && (int)blockIdx.x == (g_k7_watch >> 16)) { long long now_ = clock64(); g_k7_phase[i] += (unsigned long long)(now_ - tprev_); tprev_ = now_; } } while (0)
#else
#define K7_T(i) do { } while (0)
#endif
// 16 worker warps + one MMA warpgroup (warps 16..19) that runs every wgmma: wgmma accumulators are registers of the warpgroup that
// issues it, so the GEMMs sit on their own warpgroup and the workers never wait for the tensor core except where they need a result.
// 640 threads leave 96 registers a thread; the MMA warpgroup holds at most one 64 x 64 accumulator (32 registers) at a time plus
// the GEMM2 epilogue's live state, and the workers take the rest (setmaxnreg): 128 x kRegsMma + 512 x kRegsWorker <= 640 x 96.
constexpr int NT7_ALL = NT7 + 128;
constexpr int kRegsMma = 64, kRegsWorker = 104;
static_assert(128 * kRegsMma + NT7 * kRegsWorker <= NT7_ALL * 96, "setmaxnreg split must fit the CTA's register allocation");
// Named barriers (11 of the 16): 0 __syncthreads, 1 worker_sync, 2 + h RdyA[h], 4 mma_sync, 5..8 group_sync(q), 9 + h RdyB[h].
// RdyA[h] / RdyB[h]: the workers of half h arrive (bar.arrive), the MMA warpgroup waits (bar.sync).
constexpr int kBarRdyA = 2, kBarRdyB = 9;   // + h
constexpr int kBarMma = 4;                  // named barrier of the MMA warpgroup's 128 threads alone
__device__ __forceinline__ void mma_sync() { asm volatile("bar.sync %0, 128;" ::"n"(kBarMma) : "memory"); }

// ACT: the trunks' activation as a compile-time constant (B200RL_ACT_RELU / B200RL_ACT_TANH; -1 = read it from the descriptors, for
// an actor and a critic with different activations).  With the activation known the relu build carries no tanhf expansions at
// all (the runtime-act kernel was 107 KB of SASS, most of it 64 inlined tanhf bodies that a relu run branches around).
template <int ACT>
__global__ void __launch_bounds__(NT7_ALL, 1)
ac_loss_grad_tc_kernel(MlpDesc actor, MlpDesc critic, const float* params /* no __restrict__: the fused optimiser step rewrites them in the tail */, AcHyper hp, AcBatch b, float* partial,
                       float* __restrict__ loss_partial, int64_t np_total, float scale_base /* power of two ~ 1 / inv_B */,
                       OptStep st /* st.params != null: the optimiser step runs in the tail of this launch */,
                       int n_actor /* CTAs [0, n_actor) work on the actor, the rest on the critic */) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    SmemBwd& sm = *reinterpret_cast<SmemBwd*>(smem_raw);
    // The actor's loss (softmax / Gaussian log-density, entropy, PPO ratio) makes its tiles longer than the critic's, so the CTAs
    // are split unevenly (tc_split.h) and both roles finish together.  Gradient partials: row
    // `cta` holds the actor half written by actor CTA `cta` and the critic half written by critic CTA `cta`; the role with more
    // CTAs zero-fills the other half of its surplus rows.
    const int role = (int)blockIdx.x < n_actor ? 0 : 1;
    const int cta = role ? (int)blockIdx.x - n_actor : (int)blockIdx.x;
    const int nctas = role ? (int)gridDim.x - n_actor : n_actor;
    const int nrows = max(n_actor, (int)gridDim.x - n_actor);
    // Scale of the dP2 / dP1 operands (a power of two): dz / inv_B is O(ratio * A_hat) <= ~10 for the actor and 2 w_critic (R - V) for
    // the critic (as large as the returns).  x 64 / x 4 keeps the lo parts of typical entries in fp16's normal range and leaves
    // room up to |dz| / inv_B ~ 1e3 (actor) / 1.6e4 (critic) before a hi part would overflow fp16 (-> inf -> NaN loss: loud, not silent).
    const float scale_p = scale_base * (role ? 4.0f : 64.0f);
    const MlpDesc d = role ? critic : actor;
    const int act = ACT >= 0 ? ACT : d.act;
    const bool relu = act == B200RL_ACT_RELU;
    const int64_t poff = role ? actor.nparams() : 0;
    const float* __restrict__ p = params + poff;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q = warp & 3, c = (warp >> 2) & 3;
    const int s = 32 * q + lane;
    const int half = q >> 1;   // 64-sample half of the tile (wgmma M block) this worker's sample is in
    {   // weights: small ones plain, W2 as two operand images
        const float* b1 = p + (int64_t)H * d.in;
        const float* W2 = b1 + H;
        const float* b2 = W2 + (int64_t)H * H;
        // relu(S z) = S relu(z) for a power-of-two S: the H1 operand scale is folded into W1 / b1 (bit-identical, one multiply less per feature)
        const float s1 = relu ? kScaleH : 1.0f;
        for (int k = tid; k < kInMax * H; k += NT7_ALL) sm.W1[k] = (k / H) < d.in ? p[k] * s1 : 0.f;
        for (int k = tid; k < H; k += NT7_ALL) { sm.b1[k] = b1[k] * s1; sm.b2[k] = b2[k]; }
        for (int k = tid; k < H * kNo; k += NT7_ALL) {
            int j = k / kNo, o = k % kNo;
            sm.W3[k] = o < d.nout ? p[head_w<false>(d, o, j)] : 0.f;
        }
        if (tid < kNo) sm.b3[tid] = tid < d.nout ? p[head_b<false>(d, tid)] : 0.f;
        tcfwd::fill_w2_image<NT7_ALL>(sm.B1, W2);
    }
    if (tid == 32) {   // every thread of the MMA warpgroup arrives once per phase
        wg::mbar_init(&sm.bar1[0], 128); wg::mbar_init(&sm.bar1[1], 128); wg::mbar_init(&sm.bar3, 128); wg::mbar_init(&sm.bar4, 128);
    }
    wg::fence_proxy_async();
    __syncthreads();
    // undo the operand scales (exact powers of two): D1 = H1 W2, D2 = dP2 W2, D3 = dP2^T [H1 | 1], D4 = dP1^T [x | 1]
    const float inv_s1 = 1.0f / (kScaleH * kScaleW), inv_s3 = 1.0f / (scale_p * kScaleH), inv_sp = 1.0f / scale_p, inv_s4 = 1.0f / (scale_p * kScaleX);
    const int64_t ntiles = (b.B + TM - 1) / TM;

    if (warp >= NT7 / 32) {
        // ================= MMA warpgroup ================================================================================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegsMma));
        const int t = tid - NT7, row0 = 16 * (t >> 5) + ((t & 31) >> 2), col0 = 2 * (t & 3);   // accumulator fragment (wgmma.cuh)
        const uint64_t dB1k = wg::make_desc(wg::smem_u32(sm.B1), G_F, GW_S);   // W2 image K-major (n = o, k = i): GEMM1
        const uint64_t dB1t = wg::make_desc(wg::smem_u32(sm.B1), GW_S, G_F);   // the same bytes MN-major (n = i, k = o): GEMM2
        float dacc[32];
        auto store_d = [&](int h) {   // GEMM1 / GEMM2 result of samples 64h .. 64h+63 -> D
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh)
                    *reinterpret_cast<float2*>(sm.D + d_off(64 * h + row0 + 8 * hh, 8 * j + col0)) = make_float2(dacc[4 * j + 2 * hh], dacc[4 * j + 2 * hh + 1]);
        };
        auto gemm1 = [&](int h, int buf) { gemm_ts3<0>(dacc, sm.AH[buf][0], sm.AH[buf][1], h, dB1k, 2 * G_F); };
        auto gemm2 = [&](int h) { gemm_ts3<1>(dacc, sm.FP_full, sm.FP_lo, h, dB1t, 2 * GW_S); };   // dH1 = dP2 x W2
        // GEMM2 epilogue, samples 64h .. 64h+63: dP1 = D2 .* act'(H1) -> the dP1^T image (A operand of GEMM4).  Each thread
        // writes its fragment's feature pairs as half2 words: a quad covers one 16-byte feature group of one sample and a warp
        // 128 contiguous bytes (conflict-free).
        auto store_dp1 = [&](int h, int pbuf) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int ss = 64 * h + row0 + 8 * hh;
                const uint64_t pos = relu ? sm.H1pos[pbuf][ss] >> col0 : 0u;   // bit 8j (+1): feature 8j + col0 (+1)
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const uint32_t off = fimg_off(8 * j + col0, ss);
                    // D2 carries scale_p * kScaleW; the dP1 operand wants scale_p: one exact power-of-two factor
                    float v0 = dacc[4 * j + 2 * hh] * (1.0f / kScaleW), v1 = dacc[4 * j + 2 * hh + 1] * (1.0f / kScaleW);
                    if (relu) {   // act'(H1) = (H1 > 0): the signs layer1() kept
                        v0 = ((pos >> (8 * j)) & 1u) ? v0 : 0.f;
                        v1 = ((pos >> (8 * j + 1)) & 1u) ? v1 : 0.f;
                    } else {      // this tile's H1 = (hi + lo) / scale
                        const float inv_h = 1.0f / kScaleH;
                        const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(sm.AH[pbuf][0] + off));
                        const float2 lf = __half22float2(*reinterpret_cast<const __half2*>(sm.AH[pbuf][1] + off));
                        v0 *= dact_f(act, (hf.x + lf.x) * inv_h);
                        v1 *= dact_f(act, (hf.y + lf.y) * inv_h);
                    }
                    uint32_t hi, lo;
                    split2(v0, v1, hi, lo);
                    *reinterpret_cast<uint32_t*>(sm.FQ_full + off) = hi;
                    *reinterpret_cast<uint32_t*>(sm.FQ_lo + off) = lo;
                }
            }
        };
        // GEMM3 (K = 128 samples, M = 64 features j): dP2^T hi x H1^T hi, lo x hi and hi x lo into one accumulator, then
        // [dP2^T hi | lo] x the x^T operand, whose feature 4 is 1.0 for every sample: sum_s dP2 = db2 lands in column 4 of an
        // N = 8 accumulator.  GEMM4 (K = 128 samples, M = 64 features f): dP1^T hi x [x hi, 1], hi x x lo, lo x [x hi, 1];
        // columns 0..3 = dW1, 4 = db1.  GEMM3's two parts go to the tensor core back to back as two commit groups, and the N = 64
        // result is added into AccW2 by the fragment's owner thread while the N = 8 part still runs (not between them); GEMM4
        // follows.  Each accumulator sees the same wgmma sequence as before.  (GEMM4 cannot join the batch: with its accumulator
        // live too, 64 registers are too few and ptxas serialises every wgmma of the kernel.)
        // Every MMA thread's share of the dP1^T image (GEMM4's A operand) is in place before the call (mma_sync).
        auto gemm34 = [&](int buf) {
            const uint64_t dPh = wg::make_desc(wg::smem_u32(sm.FP_full), GF_T, GS_T), dPl = wg::make_desc(wg::smem_u32(sm.FP_lo), GF_T, GS_T);
            const uint64_t dHh = wg::make_desc(wg::smem_u32(sm.AH[buf][0]), GF_T, GS_T), dHl = wg::make_desc(wg::smem_u32(sm.AH[buf][1]), GF_T, GS_T);
            const uint64_t dQh = wg::make_desc(wg::smem_u32(sm.FQ_full), GF_T, GS_T), dQl = wg::make_desc(wg::smem_u32(sm.FQ_lo), GF_T, GS_T);
            const uint64_t dX = wg::make_desc(wg::smem_u32(sm.XT[buf]), GF_T, GS_T);
            float d8[4] = {0.f, 0.f, 0.f, 0.f}, d4[4] = {0.f, 0.f, 0.f, 0.f};
            wg::fence();
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint32_t a = k * 2 * GF_T;
                wg::mma_m64n64k16<1, 1>(dacc, wg::desc_add(dPh, a), wg::desc_add(dHh, a), k ? 1u : 0u);
                wg::mma_m64n64k16<1, 1>(dacc, wg::desc_add(dPl, a), wg::desc_add(dHh, a), 1u);
                wg::mma_m64n64k16<1, 1>(dacc, wg::desc_add(dPh, a), wg::desc_add(dHl, a), 1u);
            }
            wg::commit();
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint32_t a = k * 2 * GF_T;
                wg::mma_m64n8k16<1, 1>(d8, wg::desc_add(dPh, a), wg::desc_add(dX, a), k ? 1u : 0u);
                wg::mma_m64n8k16<1, 1>(d8, wg::desc_add(dPl, a), wg::desc_add(dX, a), 1u);
            }
            wg::commit();
            wg::wait_groups<1>();                      // GEMM3's N = 64 part
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float2* a = reinterpret_cast<float2*>(sm.AccW2 + (row0 + 8 * hh) * kAccW2S + 8 * j + col0);
                    float2 v = *a;
                    v.x += dacc[4 * j + 2 * hh];
                    v.y += dacc[4 * j + 2 * hh + 1];
                    *a = v;
                }
            wg::wait_all();                            // db2
            if (col0 == 4) {
                sm.AccW2[64 * kAccW2S + row0] += d8[0];
                sm.AccW2[64 * kAccW2S + row0 + 8] += d8[2];
            }
            wg::mbar_arrive(&sm.bar3);                 // GEMM3 has read FP and AH[buf]
            wg::fence();
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint32_t a = k * 2 * GF_T;
                wg::mma_m64n8k16<1, 1>(d4, wg::desc_add(dQh, a), wg::desc_add(dX, a), k ? 1u : 0u);
                wg::mma_m64n8k16<1, 1>(d4, wg::desc_add(dQh, a), wg::desc_add(dX, GS_T + a), 1u);
                wg::mma_m64n8k16<1, 1>(d4, wg::desc_add(dQl, a), wg::desc_add(dX, a), 1u);
            }
            wg::commit();
            wg::wait_all();                            // GEMM4
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    if (col0 + e < 5) sm.AccD4[(row0 + 8 * hh) * 9 + col0 + e] += d4[2 * hh + e];
            wg::mbar_arrive(&sm.bar4);
        };
        // Per tile, per 64-sample half h: G2(t, h) + epilogue (dP1^T image) | G1(t+1, h); then G3(t) | G4(t) over all 128 samples.
        // Only G2 -> G1 of its own half sits between the hand-over of half h of tile t (RdyA[h]) and the P3 of tile t + 1 of
        // quadrants 2h, 2h+1 (bar1[h]): half 0's GEMM chain runs under half 1's loss work and the reverse.  G3(t) and G4(t) run under
        // P3 / P45(t+1).  D holds D1 only: rows 64h .. 64h+63 of D1(t) are read in P3(t) of half h, before it hands over RdyA[h](t).
        //
        // Phase accounting (W_h = the 256 worker threads of quadrants 2h, 2h+1; M = the 128 MMA threads; once per tile each):
        //   RdyA[h]  named, 384: W_h arrive after their dP2 stores of tile t, M waits before G2(t, h).  W_h arrive for t + 1 only
        //            behind bar1[h](t+1), which M completes after it has passed RdyA[h](t): no early arrival joins an open phase.
        //   RdyB[h]  named, 384: W_h arrive after layer1(t+1), M waits before G1(t+1, h).  W_h arrive for t + 2 behind
        //            bar1[h](t+1), which M completes after its RdyB[h](t+1) wait.
        //   bar1[h]  mbarrier, count 128: M arrives after store_d(h) of G1(t+1), W_h wait before P3(t+1).  Phase t+2 needs
        //            RdyB[h](t+2), which every thread of W_h arrives after its wait for phase t+1.
        //   bar3     mbarrier, count 128: M arrives after G3(t), all 512 workers wait in P45(t+1) before their dP2 stores (FP is
        //            G3(t)'s A operand) and so before layer1(t+2) overwrites AH[t&1] (G3(t)'s B operand; G1(t) and the tanh epilogue
        //            of t read it earlier in M's order).  Phase t+1 needs G2(t+1, 0 and 1), i.e. RdyA[0, 1](t+1), which every
        //            worker arrives after that wait.
        //   bar4     mbarrier, count 128: M arrives after G4(t), all workers wait before RdyA(t+1) (publish(t+2) rewrites XT[t&1]);
        //            phase t+1 needs RdyA[0, 1](t+1) as above.
        if (cta < ntiles) {
            for (int h = 0; h < 2; ++h) {
                ready_wait(kBarRdyB + h);              // H1 operand of the first tile
                gemm1(h, 0); store_d(h);
                wg::mbar_arrive(&sm.bar1[h]);
            }
        }
        int buf = 0;
        for (int64_t tile = cta; tile < ntiles; tile += nctas, buf ^= 1) {
            const bool has_next = tile + nctas < ntiles;
            for (int h = 0; h < 2; ++h) {
                ready_wait(kBarRdyA + h);              // dP2 image of this half; its workers have read their D1(t)
                gemm2(h); store_dp1(h, buf);
                if (has_next) {
                    ready_wait(kBarRdyB + h);          // H1 operand of this half of the next tile
                    gemm1(h, buf ^ 1); store_d(h);
                    wg::mbar_arrive(&sm.bar1[h]);
                }
            }
            wg::fence_proxy_async();                   // this thread's share of the dP1^T image -> visible to GEMM4 (after mma_sync)
            mma_sync();                                // every thread's share of the dP1^T image is in place
            gemm34(buf);                               // (GEMM4's x^T | 1 operand was written at publish time)
        }
    } else {
    // ================= 16 worker warps =======================================================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegsWorker));
    // persistent per-thread gradient partials (over this thread's sample slot), reduced once at the end
    float g3[2][16];                  // dW3[o][16c + k]   (db2, dW1, db1 and dW2 are reduced over the samples by the tensor core)
    float gb3a0 = 0.f, gb3a1 = 0.f;   // (c == 0 threads) sum_s dz[o]
#pragma unroll
    for (int k = 0; k < 16; ++k) { g3[0][k] = 0.f; g3[1][k] = 0.f; }
    float l0 = 0.f, l1 = 0.f;
    float mean = 0.f, inv_std = 1.f;
    if (hp.normalize_adv && b.norm2) { mean = b.norm2[0]; inv_std = b.norm2[1]; }
    uint32_t ph1 = 0, ph3 = 0, ph4 = 0;
    bool gemm4_pending = false;
    int xbuf = 0;                     // XT buffer of the tile being published (tile parity within this CTA)
    int pbuf = 0;                     // H1pos buffer of the tile layer1() runs on (tile parity within this CTA)
    // Random gather, per THREAD: each of the four feature-block threads of a sample loads the sample's whole 32-byte record
    // {state | action bits, logp_old, advantage, return} itself (two 16-byte loads from one sector; the three repeats hit L1), so
    // nothing is exchanged through shared memory and no barrier separates the gather from layer 1 or from the loss.  Software
    // pipeline: the records are requested one tile ahead and the permuted index two tiles ahead (an index array adds a dependent
    // load; the Feistel permutation is ALU work), so neither latency is ever waited for.  No arithmetic on loaded values here.
#ifdef B200RL_K7_TIMING
    long long tprev_ = clock64();
#endif
    const int pbits = b200perm::perm_bits(b.perm_n);
    const uint32_t pkey = ac_perm_key(b);
    auto index_of = [&](int64_t t) -> int32_t {      // rollout index of this thread's sample in tile t, -1 = padding
        const int64_t j = t * TM + s;
        if (t >= ntiles || j >= b.B) return -1;
        return b.idx ? b.idx[j] : (int32_t)perm_index_bits((uint32_t)(b.perm_offset + j), b.perm_n, pkey, pbits);
    };
    auto request = [&](int32_t g, float (&x)[kInMax], float (&a)[4]) {
#pragma unroll
        for (int k = 0; k < kInMax; ++k) { x[k] = 0.f; a[k] = 0.f; }
        if (g < 0) return;
        if (b.rec) {
            const float4 v0 = b.rec[2 * (int64_t)g], v1 = b.rec[2 * (int64_t)g + 1];
            x[0] = v0.x; x[1] = v0.y; x[2] = v0.z; x[3] = v0.w;
            a[0] = v1.x; a[1] = v1.y; a[2] = v1.z; a[3] = v1.w;
        } else {                                     // separate rollout columns (direct API calls)
#pragma unroll
            for (int i = 0; i < kInMax; ++i)         // static indices only: a runtime-indexed array would live in local memory
                if (i < b.ns) x[i] = b.states[(int64_t)b.ns * g + i];
            a[0] = reinterpret_cast<const float*>(b.actions)[g];
            a[1] = b.logp_old ? b.logp_old[g] : 0.f;
            a[2] = b.adv[g];
            a[3] = b.ret[g];
        }
    };
    float pfx[kInMax] = {0.f, 0.f, 0.f, 0.f}, pfa[4] = {0.f, 0.f, 0.f, 0.f};   // records of the NEXT tile (in flight)
    float aux[4] = {0.f, 0.f, 0.f, 0.f};   // {action bits, logp_old, (normalised) advantage, return} of the tile whose loss is evaluated next
    int32_t gi_next = -1;             // index of this thread's sample two tiles ahead
    bool gemm3_pending = false;
    float* const out = partial + (int64_t)cta * np_total + poff;
    float* const gW1 = out;
    float* const gb1 = out + (int64_t)H * d.in;
    float* const gW2 = gb1 + H;
    float* const gb2 = gW2 + (int64_t)H * H;
    for (int k = tid; k < 64 * kAccW2S + 64; k += NT7) sm.AccW2[k] = 0.f;
    for (int k = tid; k < 64 * 9; k += NT7) sm.AccD4[k] = 0.f;
    // ---- software pipeline (one tile = 128 samples; tensor core and CUDA cores work on different tiles / phases) ----
    //   workers        : ... P3(t) P45(t) | P0(t+1) P1(t+1) | P3(t+1) P45(t+1) ...
    //   MMA warpgroup  :              G2(t,0) + dP1 G1(t+1,0) | G2(t,1) + dP1 G1(t+1,1) | G3(t) G4(t) ...
    // G2(t) and its epilogue (dP1 = dH1 .* act'(H1) -> the GEMM4 operand) run under P0/P1(t+1), G3(t) / G4(t) under
    // P3 / P45(t+1); the MMA warpgroup starts each GEMM as soon as the workers have handed its operands over (ready_arrive), so
    // no worker waits for a GEMM whose result it does not need.  The hand-overs and the wait for GEMM1 are per 64-sample half
    // (quadrants 2h, 2h+1): half 0's workers start P3(t+1) while the tensor core still runs half 1's G2(t) / G1(t+1).
    // P0: the next tile's records leave the prefetch registers (x -> layer 1 and the x^T operand of GEMM4, scalars -> aux),
    // the records of the tile after it are requested, the index of the one after that computed / requested
    float xo[kInMax];
    auto publish = [&](int64_t t) {
#pragma unroll
        for (int i = 0; i < kInMax; ++i) xo[i] = pfx[i];
        aux[0] = pfa[0];
        aux[1] = role == 0 ? pfa[1] : 0.f;
        aux[2] = role == 0 ? (hp.normalize_adv ? (pfa[2] - mean) * inv_std : pfa[2]) : 0.f;
        aux[3] = role == 0 ? 0.f : pfa[3];
        if (c == 0) {
            uint32_t h01, l01, h23, l23;   // x^T operand of GEMM4 (features 0..3 hi, 8..11 lo)
            split2(xo[0] * kScaleX, xo[1] * kScaleX, h01, l01);
            split2(xo[2] * kScaleX, xo[3] * kScaleX, h23, l23);
            uint8_t* xt = sm.XT[xbuf] + fimg_off(0, s);
            *reinterpret_cast<uint4*>(xt) = make_uint4(h01, h23, 0x3C00u, 0u);          // features 0..3 = x hi, 4 = 1.0 (-> db1), 5..7 = 0
            *reinterpret_cast<uint4*>(xt + GS_T) = make_uint4(l01, l23, 0u, 0u);       // features 8..11 = x lo
        }
        K7_T(16);
        xbuf ^= 1;
        request(gi_next, pfx, pfa);                  // tile t + nctas
        gi_next = index_of(t + 2 * nctas);
        K7_T(17);
    };
    auto layer1 = [&]() {   // P1: H1 = act(W1 x + b1) -> A operand of GEMM1 (hi | lo fp16 images); relu: its signs -> H1pos
        uint32_t pos = 0;
        uint32_t hi8[8], lo8[8];
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) {
            const int f0 = 16 * c + 4 * ch;
            float4 bb = *reinterpret_cast<const float4*>(sm.b1 + f0);
            float h[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
            for (int k = 0; k < kInMax; ++k) {
                float4 w = *reinterpret_cast<const float4*>(sm.W1 + k * H + f0);
                h[0] = fmaf(w.x, xo[k], h[0]); h[1] = fmaf(w.y, xo[k], h[1]); h[2] = fmaf(w.z, xo[k], h[2]); h[3] = fmaf(w.w, xo[k], h[3]);
            }
            if (relu) {   // W1 / b1 carry the operand scale already
#pragma unroll
                for (int e = 0; e < 4; ++e) { pos |= (h[e] > 0.f ? 1u : 0u) << (4 * ch + e); h[e] = fmaxf(h[e], 0.f); }
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) h[e] = act_f(act, h[e]) * kScaleH;
            }
            split2(h[0], h[1], hi8[2 * ch], lo8[2 * ch]);
            split2(h[2], h[3], hi8[2 * ch + 1], lo8[2 * ch + 1]);
        }
        if (relu) reinterpret_cast<uint16_t*>(&sm.H1pos[pbuf][s])[c] = (uint16_t)pos;   // bits 16c .. 16c+15 of the sample's word
        store16_feat(sm.AH[pbuf][0], 16 * c, s, hi8);
        store16_feat(sm.AH[pbuf][1], 16 * c, s, lo8);
        pbuf ^= 1;
    };
    if (cta < ntiles) {   // prologue: P0 / P1 of the first tile (the MMA warpgroup runs its G1)
        request(index_of(cta), pfx, pfa);
        gi_next = index_of(cta + nctas);
        publish(cta);
        layer1();
        wg::fence_proxy_async();
        ready_arrive(kBarRdyB + half);
    }
#ifdef B200RL_K7_TIMING
    tprev_ = clock64();
#endif
    // P3 and P4+P5 of one tile (below) for NO head outputs.  The critic (n_out = 1) runs NO = 1 and skips the second head: its W3
    // column and b3 are zero and its dz is +0 there, and nothing reads its g3[1] / gb3a1 / l1.  Same bits as NO = 2: that head's term
    // of dh is w.y * dzs1 = +0, which the fmaf against +0 keeps (a -0 product still comes out +0).
    auto tile_loss = [&](auto no, int64_t tile, uint32_t(&hi8)[8], uint32_t(&lo8)[8]) {
        constexpr int NO = decltype(no)::value;
        // ---- P3: H2 = act(D1 + b2) (registers) + head partials ---------------------------------------
        float h2[16];
        {
            float v[16];
            d_ld16(sm.D, s, 16 * c, v);
            float zp[NO];
#pragma unroll
            for (int o = 0; o < NO; ++o) zp[o] = 0.f;
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const int f = 16 * c + k;
                h2[k] = act_f(act, fmaf(v[k], inv_s1, sm.b2[f]));   // operand scales undone (exact)
                if constexpr (NO == 2) {
                    float2 w = *reinterpret_cast<const float2*>(sm.W3 + f * kNo);
                    zp[0] = fmaf(w.x, h2[k], zp[0]); zp[1] = fmaf(w.y, h2[k], zp[1]);
                } else {
                    zp[0] = fmaf(sm.W3[f * kNo], h2[k], zp[0]);
                }
            }
#pragma unroll
            for (int o = 0; o < NO; ++o) sm.Zp[(c * kNo + o) * TM + s] = zp[o];
        }
        K7_T(1);
        group_sync(q);
        K7_T(2);
        // ---- P4+P5: loss (evaluated by all four feature-block threads of a sample: no exchange, no idle warps),
        //            dW3 / db2 partials, dP2 = (W3^T dz) .* act'(H2) -> dP2^T image (A operand of GEMM2 and GEMM3) ----------
        float z[kNo] = {0.f, 0.f};
#pragma unroll
        for (int o = 0; o < NO; ++o)
            z[o] = sm.b3[o] + ((sm.Zp[o * TM + s] + sm.Zp[(kNo + o) * TM + s]) + (sm.Zp[(2 * kNo + o) * TM + s] + sm.Zp[(3 * kNo + o) * TM + s]));
        const bool valid = (tile * TM + s) < b.B;
        // (evaluated by all four feature-block threads of a sample: identical arithmetic on each)
        const policy::LossOut<kNo> lo_ = policy::sample_loss(actor.heads2, actor.nout, NO == 2 ? 0 : 1, hp, b.inv_B, z, aux[0], aux[1], aux[2], aux[3]);
        float dz[kNo];
#pragma unroll
        for (int o = 0; o < kNo; ++o) dz[o] = valid ? lo_.dz[o] : 0.f;
        if (c == 0 && valid) {
            l0 += lo_.l0; gb3a0 += dz[0];
            if constexpr (NO == 2) { l1 += lo_.l1; gb3a1 += dz[1]; }
        }
        // dP2 operand = scale_p * (W3^T dz) .* act'(H2): the power-of-two operand scale rides on dz (exact, bit-identical to scaling dP2)
        const float dzs0 = dz[0] * scale_p, dzs1 = dz[1] * scale_p;
        float dp[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const int f = 16 * c + k;
            float dh;
            if constexpr (NO == 2) {
                float2 w = *reinterpret_cast<const float2*>(sm.W3 + f * kNo);
                dh = fmaf(w.x, dzs0, w.y * dzs1);
            } else {
                dh = fmaf(sm.W3[f * kNo], dzs0, 0.f);
            }
            dp[k] = relu ? (h2[k] > 0.f ? dh : 0.f) : dh * (1.f - h2[k] * h2[k]);
            g3[0][k] = fmaf(dz[0], h2[k], g3[0][k]);
            if constexpr (NO == 2) g3[1][k] = fmaf(dz[1], h2[k], g3[1][k]);
        }
#pragma unroll
        for (int m = 0; m < 8; ++m) split2(dp[2 * m], dp[2 * m + 1], hi8[m], lo8[m]);
    };
    for (int64_t tile = cta; tile < ntiles; tile += nctas) {
        const bool has_next = tile + nctas < ntiles;
        wg::mbar_wait(&sm.bar1[half], ph1);
        ph1 ^= 1u;
        K7_T(0);
        {
            uint32_t hi8[8], lo8[8];
            if (role) tile_loss(std::integral_constant<int, 1>{}, tile, hi8, lo8);
            else tile_loss(std::integral_constant<int, 2>{}, tile, hi8, lo8);
            K7_T(3);
            if (gemm3_pending) {   // the previous tile's GEMM2 / GEMM3 must have consumed the images before they are overwritten
                wg::mbar_wait(&sm.bar3, ph3);
                ph3 ^= 1u;
                gemm3_pending = false;
            }
            K7_T(4);
            store16_feat(sm.FP_full, 16 * c, s, hi8);
            store16_feat(sm.FP_lo, 16 * c, s, lo8);
        }
        K7_T(5);
        wg::fence_proxy_async();
        // The previous tile's GEMM4 must have consumed its XT buffer (the same parity as the next tile's, which publish() rewrites).
        // Waited before this tile's hand-over: GEMM4(t) depends on it, so no bar4 phase can complete twice before it is waited for.
        // (The MMA warpgroup runs GEMM4(t-1) before it waits for RdyA(t) anyway: the wait costs it nothing.)
        if (gemm4_pending) {
            wg::mbar_wait(&sm.bar4, ph4);
            ph4 ^= 1u;
        }
        K7_T(6);
        ready_arrive(kBarRdyA + half);   // this thread's share of the GEMM2 / GEMM3 operands is in place
        gemm3_pending = true;       // (Zp is rewritten in P3 of the next tile, behind its wait for GEMM1, i.e. after every thread has passed
        gemm4_pending = true;       //  this point: no barrier needed here)
        K7_T(7);
        if (has_next) {
            publish(tile + nctas);
            layer1();
            wg::fence_proxy_async();
            K7_T(8);
            ready_arrive(kBarRdyB + half);
            K7_T(9);
        }
#ifdef B200RL_K7_TIMING
        if (tid == (g_k7_watch & 0xFFFF) && (int)blockIdx.x == (g_k7_watch >> 16)) g_k7_phase[15] += 1;
#endif
    }
    // ---- drain: last GEMM3 / GEMM4 (their sums are in AccW2 / AccD4), then the head gradients (fixed-order reductions) -------
    if (gemm3_pending) wg::mbar_wait(&sm.bar3, ph3);
    if (gemm4_pending) wg::mbar_wait(&sm.bar4, ph4);
    worker_sync();                                       // (a CTA without tiles writes the zeros the accumulators were initialised with)
    for (int k = tid; k < H * H; k += NT7) gW2[k] = sm.AccW2[(k & 63) * kAccW2S + (k >> 6)] * inv_s3;     // gW2[j + 64 i]
    if (tid < H) {
        gb2[tid] = sm.AccW2[64 * kAccW2S + tid] * inv_sp;
        gb1[tid] = sm.AccD4[tid * 9 + 4] * inv_sp;
        for (int i = 0; i < d.in; ++i) gW1[tid + H * i] = sm.AccD4[tid * 9 + i] * inv_s4;
    }
    if (cta >= (int)gridDim.x - nctas) {   // surplus row: the other role has no CTA `cta`, its half of the row is zero
        const int64_t ooff = role ? 0 : actor.nparams(), on = role ? actor.nparams() : critic.nparams();
        float* orow = partial + (int64_t)cta * np_total + ooff;
        for (int64_t kk = tid; kk < on; kk += NT7) orow[kk] = 0.f;
    }
    float* red = reinterpret_cast<float*>(sm.FP_full);   // images + weight images: contiguous, all MMAs are done
    static_assert(offsetof(SmemBwd, XT) - offsetof(SmemBwd, FP_full) >= (2 * TM * 65 + 2 * 8 * 64) * 4, "drain scratch");
    // per-sample-slot partials of dW3[0], dW3[1] -> two [128 slots][64] matrices in shared memory -> column sums in
    // a fixed order: 8 segment sums of 16 slots each (all 512 threads), then the 8 segments in order (64 threads per matrix)
    {
        constexpr int RS = 65;                // row stride 65: the 32 lanes (= 32 sample slots) of a store hit 32 different banks
        float* seg = red + 2 * TM * RS;       // [2][8][64]
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            red[0 * TM * RS + s * RS + 16 * c + k] = g3[0][k];
            red[1 * TM * RS + s * RS + 16 * c + k] = g3[1][k];
        }
        worker_sync();
        {
            const int col = tid & 63, g = tid >> 6;   // 8 segments x 64 columns
#pragma unroll
            for (int m = 0; m < 2; ++m) {
                float a = 0.f;
#pragma unroll
                for (int ss = 0; ss < 16; ++ss) a += red[m * TM * RS + (16 * g + ss) * RS + col];
                seg[(m * 8 + g) * 64 + col] = a;
            }
        }
        worker_sync();
        if (tid < 2 * H) {
            const int m = tid >> 6, col = tid & 63;
            float a = 0.f;
#pragma unroll
            for (int g = 0; g < 8; ++g) a += seg[(m * 8 + g) * 64 + col];
            if (m < d.nout) out[head_w<false>(d, m, col)] = a;
        }
        worker_sync();
    }
    if (c == 0) { red[s] = gb3a0; red[TM + s] = gb3a1; }
    worker_sync();
    if (warp < d.nout) {   // one warp per head output: 4 slots per lane in order, then a fixed butterfly (a 128-step dependent chain on one thread was ~2 us)
        float a = (red[warp * TM + lane] + red[warp * TM + 32 + lane]) + (red[warp * TM + 64 + lane] + red[warp * TM + 96 + lane]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) out[head_b<false>(d, warp)] = a;
    }
    // loss sums (worker-only block reduction)
    float t0 = l0, t1 = l1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { t0 += __shfl_xor_sync(0xffffffffu, t0, o); t1 += __shfl_xor_sync(0xffffffffu, t1, o); }
    worker_sync();
    if (lane == 0) { sm.Red[warp] = t0; sm.Red[16 + warp] = t1; }
    worker_sync();
    if (tid == 0) {
        float a0 = 0.f, a1 = 0.f;
        for (int k = 0; k < 16; ++k) { a0 += sm.Red[k]; a1 += sm.Red[16 + k]; }
        float* lp = loss_partial + (int64_t)blockIdx.x * 4;
        lp[0] = role ? 0.f : a0; lp[1] = role ? 0.f : a1; lp[2] = role ? a0 : 0.f; lp[3] = 0.f;
    }
    // the separate reduction reads 2 * nrows loss rows (nn_ac_loss_grad's row count, the FFMA kernel's layout); the ones past
    // this grid's own are zero, not whatever an earlier launch (an FFMA one on the same network) left there
    if (blockIdx.x == 0)
        for (int k = tid; k < 4 * (2 * nrows - (int)gridDim.x); k += NT7) loss_partial[4 * (int64_t)gridDim.x + k] = 0.f;
    // ---- fused optimiser step (K8 inside K7's tail): K8's arithmetic (optim.cuh) and its CTA-order gradient and loss sums; the
    //      gradient-norm total is summed per lane, then by a butterfly, so it may round differently from K8's --------------------
    if (st.params) {
        const unsigned int G = gridDim.x;
        K7_T(24);                                // (everything since the last tile: drain, head-gradient reductions, partial rows)
        worker_sync();                           // every worker's partial / loss rows are written (CTA scope) ...
        K7_T(25);
        if (tid == 0) optim::grid_barrier(st.counters, G);   // grid barrier A: every CTA's rows are written
        worker_sync();
        K7_T(26);
        const int per = (int)((np_total + G - 1) / G);           // parameters per CTA (<= NT7: nn_tc_step_fits)
        const int64_t k = (int64_t)blockIdx.x * per + tid;
        const bool mine = tid < per && k < np_total;
        const unsigned int seq = st.tab.nranks > 1 ? *st.seq_ptr + 1u : 0u;
        // The CTA's slice of every partial row is staged through shared memory by ALL worker threads (every L2 read in flight at
        // once: one round trip instead of one per 16 rows), then one thread per parameter adds its column in CTA order.
        float* stage = reinterpret_cast<float*>(sm.FP_full);            // images are dead: all MMAs have completed
        const int nstage = per * nrows;                                  // <= 64 * 76 floats with the BASELINE network
        const int64_t k0 = (int64_t)blockIdx.x * per;
        {   // (fixed trip count, loads first: a rolled loop would wait for each L2 round trip before issuing the next)
            float t[kMaxStage];
#pragma unroll
            for (int j = 0; j < kMaxStage; ++j) {
                const int e = tid + j * NT7;
                const int row = e / per, col = e - row * per;
                t[j] = (e < nstage && k0 + col < np_total) ? __ldcg(partial + (int64_t)row * np_total + k0 + col) : 0.f;
            }
#pragma unroll
            for (int j = 0; j < kMaxStage; ++j) {
                const int e = tid + j * NT7;
                if (e < nstage) stage[e] = t[j];
            }
        }
        float* lstage = stage + nstage;
        if (blockIdx.x == 0) {
            float t[2];
#pragma unroll
            for (int j = 0; j < 2; ++j) t[j] = tid + j * NT7 < 4 * (int)G ? __ldcg(loss_partial + tid + j * NT7) : 0.f;
#pragma unroll
            for (int j = 0; j < 2; ++j) if (tid + j * NT7 < 4 * (int)G) lstage[tid + j * NT7] = t[j];
        }
        // Adam operands of this thread's parameter: requested now, consumed behind grid barrier B
        float m_k = 0.f, v_k = 0.f, p_k = 0.f;
        if (mine) { m_k = st.m[k]; v_k = st.v[k]; p_k = st.params[k]; }
        worker_sync();
        K7_T(27);
        float gk = 0.f;
        if (mine) {   // rows in CTA order; 8 shared-memory reads in flight
            for (int c0 = 0; c0 < nrows; c0 += 8) {
                float t[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) t[j] = c0 + j < nrows ? stage[(c0 + j) * per + tid] : 0.f;
#pragma unroll
                for (int j = 0; j < 8; ++j) if (c0 + j < nrows) gk += t[j];
            }
        }
        float lsum = 0.f;
        const bool loss_thread = blockIdx.x == 0 && tid < 4;
        if (loss_thread) {
            for (unsigned int c0 = 0; c0 < G; c0 += 8) {
                float t[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) t[j] = c0 + j < G ? lstage[(c0 + j) * 4 + tid] : 0.f;
#pragma unroll
                for (int j = 0; j < 8; ++j) if (c0 + j < G) lsum += t[j];
            }
        }
        if (st.tab.nranks > 1) {   // push the local sums into every peer's inbox, collect the peers' from the own inbox, sum in rank order
            const unsigned slot = seq & 1u;
            if (mine) p2p_push(st.tab, 0, slot, (size_t)k, __float_as_uint(gk), seq);
            if (loss_thread) p2p_push(st.tab, 0, slot, (size_t)np_total + tid, __float_as_uint(lsum), seq);
            if (mine) gk = p2p_sum_ranks(st.tab, 0, slot, (size_t)k, gk, seq);
            if (loss_thread) lsum = p2p_sum_ranks(st.tab, 0, slot, (size_t)np_total + tid, lsum, seq);
        }
        if (loss_thread) optim::publish_loss(st, tid, lsum);
        double sq = (double)gk * (double)gk;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
        if (lane == 0) sm.RedD[warp] = sq;
        worker_sync();
        K7_T(28);
        if (warp == 0) {
            if (lane == 0) {                     // grid barrier B: every CTA's sum of squares is published
                double t = 0.0;
                for (int w = 0; w < NT7 / 32; ++w) t += sm.RedD[w];
                st.cta_sumsq[blockIdx.x] = t;
                optim::grid_barrier(st.counters + 1, G);
            }
            __syncwarp();
            K7_T(29);
            // every lane fetches its share of the per-CTA sums (all reads in flight), adds them in CTA order, then a fixed
            // butterfly over the lanes: deterministic, and every CTA computes the identical total
            double part[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) part[j] = (unsigned)(lane + 32 * j) < G ? __ldcg(st.cta_sumsq + lane + 32 * j) : 0.0;
            double tot = 0.0;
#pragma unroll
            for (int j = 0; j < 8; ++j) tot += part[j];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
            if (lane == 0) {
                const float gn = (float)sqrt(tot);
                sm.step_scale = optim::clip_scale(gn, st.max_norm);
                if (blockIdx.x == 0) optim::publish_gnorm(st, gn);
            }
        }
        worker_sync();
        K7_T(30);
        const float bt1 = st.beta_t[0], bt2 = st.beta_t[1];
        if (mine) {
            gk *= sm.step_scale;
            st.grad[k] = gk;
            const optim::AdamOut a = optim::adam_update(gk, m_k, v_k, p_k, st.lr, st.b1, st.b2, st.eps, bt1, bt2);
            st.m[k] = a.m; st.v[k] = a.v; st.params[k] = a.p;
        }
        worker_sync();
        if (tid == 0) optim::close_step<3>(st, bt1, bt2, st.tab.nranks > 1, seq);
        K7_T(31);
    }
    }  // worker warps
    __syncthreads();
}

}  // namespace

// actor : critic CTA split (tc_split.h); B200RL_K7_ACTOR_CTAS overrides it for tuning runs
int nn_tc_actor_ctas(int grid, const MlpDesc& actor, const AcHyper& hp, int64_t ntiles) {
    static int forced = -2;
    if (forced == -2) { const char* e = getenv("B200RL_K7_ACTOR_CTAS"); forced = e ? atoi(e) : -1; }
    if (forced > 0 && forced < grid) return forced;
    (void)hp;
    return b200rl_tc_actor_ctas(grid, actor.heads2 != 0, ntiles);
}
int nn_tc_partial_rows(int grid, const MlpDesc& actor, const AcHyper& hp, int64_t B) {
    const int na = nn_tc_actor_ctas(grid, actor, hp, (B + TM - 1) / TM);
    return na > grid - na ? na : grid - na;
}
bool nn_tc_bwd_supported(const MlpDesc& actor, const MlpDesc& critic) {
    return actor.H == 64 && critic.H == 64 && actor.in <= kInMax && actor.nout <= 2 && critic.nout == 1;
}
// the optimiser step in K7's tail: every CTA co-resident (one per SM) and at most 256 of them (cta_sumsq), one worker thread per
// parameter of the CTA's slice, the slice of every partial row in kMaxStage registers per thread, the loss rows in two
bool nn_tc_step_fits(b200rl_ctx* ctx, int grid, const MlpDesc& actor, const AcHyper& hp, int64_t B, int64_t np) {
    const int64_t per = (np + grid - 1) / grid;
    return grid <= ctx->sm_count && grid <= 256 && per <= NT7 && per * nn_tc_partial_rows(grid, actor, hp, B) <= kMaxStage * NT7 &&
           4 * grid <= 2 * NT7;
}
int nn_tc_ac_loss_grad(b200rl_ctx* ctx, int grid, const MlpDesc& actor, const MlpDesc& critic, const float* params, const AcHyper& hp,
                       const AcBatch& b, float* partial, float* loss_partial, int64_t np, const OptStep* step) {
    const OptStep st = step ? *step : OptStep{};
    const int n_actor = nn_tc_actor_ctas(grid, actor, hp, (b.B + TM - 1) / TM);
    size_t smem = sizeof(SmemBwd) + 128;
    static unsigned long long attr_devices = 0;   // once per device
    if (first_use_on_device(attr_devices, ctx->device)) {
        CUDA_TRY(cudaFuncSetAttribute(ac_loss_grad_tc_kernel<B200RL_ACT_RELU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(ac_loss_grad_tc_kernel<B200RL_ACT_TANH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(ac_loss_grad_tc_kernel<-1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    // dP2 ~ inv_B x O(1..100): scale it into fp16's normal range with a power of two (exact, undone on the accumulators)
    const float scale_base = exp2f(floorf(log2f(1.0f / b.inv_B)));
    if (actor.act == critic.act && actor.act == B200RL_ACT_RELU)
        ac_loss_grad_tc_kernel<B200RL_ACT_RELU><<<grid, NT7_ALL, smem, ctx->stream>>>(actor, critic, params, hp, b, partial, loss_partial, np, scale_base, st, n_actor);
    else if (actor.act == critic.act && actor.act == B200RL_ACT_TANH)
        ac_loss_grad_tc_kernel<B200RL_ACT_TANH><<<grid, NT7_ALL, smem, ctx->stream>>>(actor, critic, params, hp, b, partial, loss_partial, np, scale_base, st, n_actor);
    else
        ac_loss_grad_tc_kernel<-1><<<grid, NT7_ALL, smem, ctx->stream>>>(actor, critic, params, hp, b, partial, loss_partial, np, scale_base, st, n_actor);
    LAUNCH_CHECK(ctx);
    return B200RL_OK;
}

#ifdef B200RL_K7_TIMING
extern "C" int b200rl_debug_k7_watch(int tid) {
    cudaDeviceSynchronize();
    return cudaMemcpyToSymbol(g_k7_watch, &tid, sizeof tid) == cudaSuccess ? 0 : -1;
}
extern "C" int b200rl_debug_k7_phases(unsigned long long* out16, int reset) {
    cudaDeviceSynchronize();
    if (cudaMemcpyFromSymbol(out16, g_k7_phase, sizeof(unsigned long long) * 40) != cudaSuccess) return -1;
    if (reset) { unsigned long long z[24] = {0}; cudaMemcpyToSymbol(g_k7_phase, z, sizeof z); }
    return 0;
}
#endif
