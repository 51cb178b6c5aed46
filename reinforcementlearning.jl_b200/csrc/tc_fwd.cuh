// tc_fwd.cuh — device building blocks of the tensor-core forward pass of one 2 x 64 MLP (K6), shared by the policy
// inference kernel and the fused rollout kernel (fwd_tc.cu).  One tile = 128 samples = two 64-sample wgmma blocks.
//
//   layer 1 (K <= 4)  : FP32 FFMA, thread = (sample, 32 features), written into shared memory as the A operand (hi | lo fp16)
//   layer 2 (64 x 64) : wgmma m64n64k16 f16 -> FP32, both operands in shared memory, the 3-term fp16 split
//                       x_hi = fp16(64 x), x_lo = fp16(64 x - x_hi) (22 mantissa bits, like 3xTF32, at half the instruction count;
//                       see nn_tc.cu for the range limits): per K = 16 step hi*hi, hi*lo and lo*hi into the same accumulator
//   heads             : FP32 FFMA on the layer-2 outputs, partial sums of the two 32-feature halves meet in shared memory
//
// Thread <-> data: warp w: sample quadrant q = w % 4 (samples 32q .. 32q+31), column half c = w / 4; thread = sample
// s = 32q + lane, features 32c .. 32c+31.  The tile image holds, per 64-sample block, the A operand [hi 8 KB | lo 8 KB]; once
// the block's wgmmas have completed, the warpgroup that ran them overwrites it with the FP32 accumulator (64 x 64).  Every
// multiply-add of the forward pass is an explicit fmaf / separate op: its arithmetic does not depend on the contraction flags of
// the including translation unit.  The operand format (split2, wimg_off, the W2 image) is shared with the tensor-core backward
// (nn_tc.cu).
#pragma once
#include "nn.cuh"
#include "wgmma.cuh"

namespace tcfwd {

constexpr int NT = 256;
constexpr int TM = 128;
constexpr int H = 64;
constexpr int G_F = 128;              // byte stride between 8-element (16-byte) chunks along K: one 8 x 16 B core matrix
constexpr int GW_S = 8 * G_F;         // weight image: stride between 8-row groups (K = 64 = 8 chunks)
constexpr int WIMG_BYTES = 16 * GW_S; // [hi (64 rows) ; lo (64 rows)] x [K = 64] fp16 weight image (SWIZZLE_NONE, K-major core matrices)
constexpr int BLK = 8 * GW_S * 2;     // one 64-sample block of the tile image: A operand [hi | lo], later its FP32 accumulator
constexpr int TILE_BYTES = 2 * BLK;
constexpr float kScale = 64.0f;       // power-of-two scale of both operands (exact; undone on the accumulator)

struct NetSm {   // one network's weights in shared memory
    alignas(128) uint8_t B[WIMG_BYTES];        // 64 W2 as (n = out, k = in), K-major fp16: rows 0..63 hi, 64..127 lo (one N = 128 operand)
    float W1[kInMax * H];                      // [i][o]
    float b1[H], b2[H];
    float W3[H * kOutMax];                     // [j][o]
    float b3[kOutMax];
};

// two fp32 values -> packed fp16 pairs {low half = a, high half = b}: hi parts, and the fp16 of what they miss (lo parts).
// (The subtraction is plain: in the tensor-core backward, compiled with contraction, it may fuse with the multiply that made
// a or b, as it always has; the forward's operands come from rounded operations, so nothing can fuse there.)
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
    const __half2 h = __floats2half2_rn(a, b);
    const float2 back = __half22float2(h);
    const __half2 l = __floats2half2_rn(a - back.x, b - back.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ uint32_t wimg_off(int n, int k) { return (uint32_t)((n >> 3) * GW_S + (k >> 3) * G_F + (n & 7) * 16 + (k & 7) * 2); }
// W2 (Flux layout W2[o + H*i]) -> the B operand image of a CTA of NTHREADS threads: kScale W2 as (n = out o, k = in i), K-major
// fp16, rows 0..63 hi, 64..127 lo.  kScale is a power of two, so the product is exact with or without contraction.
template <int NTHREADS>
__device__ __forceinline__ void fill_w2_image(uint8_t* img, const float* W2) {
    for (int k = threadIdx.x; k < H * H; k += NTHREADS) {
        const int o = k % H, i = k / H;
        const float v = W2[k] * kScale;
        const __half vh = __float2half_rn(v), vl = __float2half_rn(v - __half2float(vh));
        *reinterpret_cast<__half*>(img + wimg_off(o, i)) = vh;
        *reinterpret_cast<__half*>(img + wimg_off(H + o, i)) = vl;
    }
}
// FP32 accumulator of one block, row r, column col: 16-byte units XOR-swizzled by the row, so that 8 consecutive rows read
// at the same column hit 8 different bank groups
__device__ __forceinline__ uint32_t dacc_off(int r, int col) { return (uint32_t)(r * 256 + (((col >> 2) ^ (r & 15)) << 4) + (col & 3) * 4); }

// s1: scale folded into W1 / b1 (kScale for relu trunks: relu(S z) = S relu(z) exactly for a power of two S, so layer 1 then
// produces the scaled H1 operand without a multiply per feature; 1 otherwise)
// MAY_DUEL = false: the caller never loads a dueling network (nn.cuh head_w)
template <bool MAY_DUEL = true>
__device__ inline void load_net(NetSm& w, const MlpDesc& d, const float* __restrict__ p, float s1) {
    const int tid = threadIdx.x;
    const float* b1 = p + (int64_t)H * d.in;
    const float* W2 = b1 + H;
    const float* b2 = W2 + (int64_t)H * H;
    for (int k = tid; k < kInMax * H; k += NT) w.W1[k] = (k / H) < d.in ? __fmul_rn(p[k], s1) : 0.f;
    for (int k = tid; k < H; k += NT) { w.b1[k] = __fmul_rn(b1[k], s1); w.b2[k] = b2[k]; }
    for (int k = tid; k < H * kOutMax; k += NT) {
        int j = k / kOutMax, o = k % kOutMax;
        w.W3[k] = o < rows_of<MAY_DUEL>(d) ? p[head_w<MAY_DUEL>(d, o, j)] : 0.f;
    }
    if (tid < kOutMax) w.b3[tid] = tid < rows_of<MAY_DUEL>(d) ? p[head_b<MAY_DUEL>(d, tid)] : 0.f;
    fill_w2_image<NT>(w.B, W2);   // B operand of H2pre[s][o] = sum_i H1[s][i] W2[o][i]
}

// layer 1 of this thread's sample: H1[32c .. 32c+32) = act(W1 x + b1) -> A operand of its block (hi at +0, lo at +8 KB; the
// image layout of the weights, row = sample)
// (the loops over 16-feature halves here and 8-feature groups in head_partials are deliberately NOT unrolled: tanhf is ~40
// instructions, and with every instance inlined the rollout kernel was 290 KB of SASS whose dominant stall was instruction fetch)
// ACT: the activation as a compile-time constant (-1: read `act`); relu trunks expect load_net(.., s1 = kScale).  UNROLL: copies
// of the half loop (the arithmetic per feature and its order do not depend on it; 1 saves registers)
template <int ACT, int UNROLL = (ACT == B200RL_ACT_RELU ? 2 : 1)>
__device__ __forceinline__ void layer1_to_smem(const NetSm& w, int act_rt, const float (&x)[kInMax], int c, int s, uint8_t* tile) {
    const int act = ACT >= 0 ? ACT : act_rt;
    uint8_t* blk = tile + (s >> 6) * BLK;
    const int r = s & 63;
#pragma unroll(UNROLL)
    for (int half = 0; half < 2; ++half) {
        uint32_t hi8[8], lo8[8];
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) {
            const int f0 = 32 * c + 16 * half + 4 * ch;
            float4 bb = *reinterpret_cast<const float4*>(w.b1 + f0);
            float h[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
            for (int k = 0; k < kInMax; ++k) {
                float4 ww = *reinterpret_cast<const float4*>(w.W1 + k * H + f0);
                h[0] = fmaf(ww.x, x[k], h[0]); h[1] = fmaf(ww.y, x[k], h[1]); h[2] = fmaf(ww.z, x[k], h[2]); h[3] = fmaf(ww.w, x[k], h[3]);
            }
            if (ACT == B200RL_ACT_RELU) {
#pragma unroll
                for (int e = 0; e < 4; ++e) h[e] = fmaxf(h[e], 0.f);
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) h[e] = __fmul_rn(act_f(act, h[e]), kScale);
            }
            split2(h[0], h[1], hi8[2 * ch], lo8[2 * ch]);
            split2(h[2], h[3], hi8[2 * ch + 1], lo8[2 * ch + 1]);
        }
        const int f0 = 32 * c + 16 * half;
        *reinterpret_cast<uint4*>(blk + wimg_off(r, f0)) = make_uint4(hi8[0], hi8[1], hi8[2], hi8[3]);
        *reinterpret_cast<uint4*>(blk + wimg_off(r, f0 + 8)) = make_uint4(hi8[4], hi8[5], hi8[6], hi8[7]);
        *reinterpret_cast<uint4*>(blk + 8 * GW_S + wimg_off(r, f0)) = make_uint4(lo8[0], lo8[1], lo8[2], lo8[3]);
        *reinterpret_cast<uint4*>(blk + 8 * GW_S + wimg_off(r, f0 + 8)) = make_uint4(lo8[4], lo8[5], lo8[6], lo8[7]);
    }
}

// one warpgroup (wgid = its index in the CTA, 128 threads): D = A x W2^T of one 64-sample block as the 3-term fp16 split, all three
// terms accumulated into the same registers (12 wgmma m64n64k16: hi*hi, hi*lo, lo*hi per K step), then D over the block's A image.
// The caller has made the A image visible to the async proxy (fence + barrier).
__device__ __forceinline__ void gemm_block(uint8_t* blk, const NetSm& w, int wgid) {
    const uint64_t dA = wg::make_desc(wg::smem_u32(blk), G_F, GW_S), dAlo = wg::desc_add(dA, 8 * GW_S);
    const uint64_t dB = wg::make_desc(wg::smem_u32(w.B), G_F, GW_S), dBlo = wg::desc_add(dB, 8 * GW_S);
    float d[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) d[i] = 0.f;
    wg::fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint32_t adv = (uint32_t)(k * 2 * G_F);
        wg::mma_m64n64k16<0, 0>(d, wg::desc_add(dA, adv), wg::desc_add(dB, adv), k ? 1u : 0u);
        wg::mma_m64n64k16<0, 0>(d, wg::desc_add(dA, adv), wg::desc_add(dBlo, adv), 1u);
        wg::mma_m64n64k16<0, 0>(d, wg::desc_add(dAlo, adv), wg::desc_add(dB, adv), 1u);
    }
    wg::commit();
    wg::wait_all();
    asm volatile("bar.sync %0, 128;" ::"r"(9 + wgid) : "memory");   // every warp's operand reads are done before D overwrites A
    const int t = threadIdx.x & 127, row0 = 16 * (t >> 5) + ((t & 31) >> 2), col0 = 2 * (t & 3);
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
            *reinterpret_cast<float2*>(blk + dacc_off(row0 + 8 * h, 8 * j + col0)) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
}

// the layer-2 activation of the epilogue.  Relu is max.NaN: an H1 operand past fp16's range (relu H1 >= 1023.75, 64 H1 rounds to
// inf) makes hi*hi + lo*hi = inf - inf, a NaN accumulator for the sample, and fmaxf(NaN, 0) = 0 would turn that into finite head
// outputs (b3).  With max.NaN the NaN reaches every head output of the sample: past the envelope the forward is loud, not wrong.
__device__ __forceinline__ float act2_f(int act, float z) {
    if (act != B200RL_ACT_RELU) return tanhf(z);
    float r;
    asm("max.NaN.f32 %0, %1, 0f00000000;" : "=f"(r) : "f"(z));
    return r;
}
// epilogue of this thread's sample: H2[32c .. 32c+32) = act(D + b2), partial head sums over these 32 features (UNROLL: as above)
template <int ACT, int UNROLL = (ACT == B200RL_ACT_RELU ? 2 : 1)>
__device__ __forceinline__ void head_partials(const NetSm& w, int act_rt, int c, int s, const uint8_t* tile, float (&zp)[kOutMax]) {
    const int act = ACT >= 0 ? ACT : act_rt;
    const uint8_t* blk = tile + (s >> 6) * BLK;
    const int r = s & 63;
#pragma unroll
    for (int o = 0; o < kOutMax; ++o) zp[o] = 0.f;
#pragma unroll(UNROLL)
    for (int grp = 0; grp < 2; ++grp) {
        float v[16];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const float4 q4 = *reinterpret_cast<const float4*>(blk + dacc_off(r, 32 * c + 16 * grp + 4 * u));
            v[4 * u] = q4.x; v[4 * u + 1] = q4.y; v[4 * u + 2] = q4.z; v[4 * u + 3] = q4.w;
        }
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const int f = 32 * c + 16 * grp + k;
            float h2 = act2_f(act, fmaf(v[k], 1.0f / (kScale * kScale), w.b2[f]));   // operand scales undone (exact power of two)
            float4 ww = *reinterpret_cast<const float4*>(w.W3 + f * kOutMax);
            zp[0] = fmaf(ww.x, h2, zp[0]); zp[1] = fmaf(ww.y, h2, zp[1]); zp[2] = fmaf(ww.z, h2, zp[2]); zp[3] = fmaf(ww.w, h2, zp[3]);
        }
    }
}

}  // namespace tcfwd
