// wgmma.cuh — inline-PTX wrappers for the Hopper warpgroup tensor-core path (wgmma.mma_async, sm_90a) used by the dense
// (64 x 64) layers, and the mbarrier helpers the loss + backward kernel hands results over with.
//
// Operand layout used throughout (SWIZZLE_NONE, "interleave"): a matrix is cut into core matrices of 8 rows x 16 bytes
// (8 fp16) stored as 128 contiguous bytes.  In a descriptor LBO is the byte stride between core matrices along K and SBO the
// stride between core matrices along M / N, for K-major and MN-major (transposed) operands alike, so the same bytes serve as
// a K-major operand of one GEMM and an MN-major operand of another.  For an activation image indexed (sample s, feature f):
//     byte(s, f) = (s / 8) * G_S + (f / 8) * G_F + (s % 8) * 16 + (f % 8) * 2
// is a K-major operand with MN = s, K = f (SBO = G_S, LBO = G_F) and an MN-major one with MN = f, K = s (SBO = G_F, LBO = G_S).
//
// Accumulators are FP32 registers of the issuing warpgroup (4 aligned warps, all 128 threads execute every call).  Fragment of
// an m64nNk16 accumulator for thread t of the warpgroup:   d[4 j + 2 h + e] = D[16 (t / 32) + (t % 32) / 4 + 8 h][8 j + 2 (t % 4) + e]
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>

namespace wg {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// 64-bit shared-memory matrix descriptor, SWIZZLE_NONE (layout type 0, base offset 0)
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;
}
// descriptor advanced by `bytes` (a multiple of 16) along its start address
__device__ __forceinline__ uint64_t desc_add(uint64_t d, uint32_t bytes) { return d + (uint64_t)(bytes >> 4); }

// before the first wgmma of a sequence: orders earlier register and shared-memory accesses of this warpgroup before it
__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// every committed wgmma of this thread has completed: its accumulators are valid and its shared-memory reads are done
__device__ __forceinline__ void wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// every commit group of this thread but the N most recent has completed
template <int N>
__device__ __forceinline__ void wait_groups() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// generic-proxy st.shared -> visible to the async proxy (tensor-core operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// D (+)= A x B, A and B from shared memory; TA / TB = 1: the operand is MN-major (transposed)
template <int TA, int TB>
__device__ __forceinline__ void mma_m64n8k16(float (&d)[4], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %6, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 "
        "{%0, %1, %2, %3}, "
        "%4, %5, p, 1, 1, %7, %8;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TA), "n"(TB)
        : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void mma_m64n64k16(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, %35, %36;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
          "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
          "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TA), "n"(TB)
        : "memory");
}


__device__ __forceinline__ void mbar_init(uint64_t* mbar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(mbar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// release: this thread's earlier shared-memory writes are visible to a thread whose wait observes the phase completing
__device__ __forceinline__ void mbar_arrive(uint64_t* mbar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(mbar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* mbar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(mbar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// bounded wait: a lost completion traps (reported as a CUDA error) instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* mbar, uint32_t parity) {
    for (uint32_t spin = 0; !mbar_try_wait(mbar, parity); ++spin)
        if (spin > (1u << 24)) __trap();
}

}  // namespace wg
