// tc_ptx.cuh -- thin inline-PTX wrappers for the Hopper (sm_90a) primitives used by the tensor-core kernels:
// mbarrier, cp.async.bulk (TMA bulk copy), proxy fences, wgmma (m64nNk16, fp16 in, fp32 accumulate in registers) and its
// shared-memory matrix descriptor.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace lz {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Bounded wait: a protocol bug must trap, never hang the GPU.  No printf here: a call anywhere in a kernel makes ptxas serialise
// its wgmma pipeline (every MMA would wait for the previous one).
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    const uint32_t a = smem_u32(bar);
    for (uint32_t it = 0; it < (1u << 28); ++it) {
        uint32_t ok;
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                     : "=r"(ok) : "r"(a), "r"(parity) : "memory");
        if (ok) return;
    }
    asm volatile("trap;\n");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }

// ---- wgmma (sm_90a): D[64 x N] (+)= A[64 x 16] * B[16 x N], fp16 inputs from shared-memory descriptors, fp32 accumulators in the
// registers of the issuing warpgroup.  Accumulator fragment of thread (warp w of the warpgroup, lane l): d[4 j + {0, 1}] = row
// 16 w + l / 4, columns 8 j + 2 (l % 4) + {0, 1}; d[4 j + {2, 3}] = the same columns of row 16 w + l / 4 + 8.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }

// Pins accumulator registers at this point of the program: zeroing (or reading) them cannot be moved into a wgmma pipeline stage,
// which would make ptxas serialise every wgmma of the kernel
template <int N>
__device__ __forceinline__ void wg_fence_acc(float (&d)[N])
{
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define LZ_WG_R8(o) "+f"(d[o + 0]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t a, uint64_t b)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}\n"
                 : LZ_WG_R8(0) : "l"(a), "l"(b));
}
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t a, uint64_t b)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, "
                 "%15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
                 : LZ_WG_R8(0), LZ_WG_R8(8) : "l"(a), "l"(b));
}
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t a, uint64_t b)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, "
                 "%15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
                 : LZ_WG_R8(0), LZ_WG_R8(8), LZ_WG_R8(16), LZ_WG_R8(24) : "l"(a), "l"(b));
}
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t a, uint64_t b)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, "
                 "%15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, "
                 "%39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, "
                 "%63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
                 : LZ_WG_R8(0), LZ_WG_R8(8), LZ_WG_R8(16), LZ_WG_R8(24), LZ_WG_R8(32), LZ_WG_R8(40), LZ_WG_R8(48), LZ_WG_R8(56)
                 : "l"(a), "l"(b));
}
#undef LZ_WG_R8
template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t a, uint64_t b)
{
    if constexpr (N == 16) wgmma_n16(d, a, b);
    else if constexpr (N == 32) wgmma_n32(d, a, b);
    else if constexpr (N == 64) wgmma_n64(d, a, b);
    else wgmma_n128(d, a, b);
}

// Writes a warpgroup's m64nN accumulator fragment to a row-major fp32 array S[row][ld] at rows row0 .. row0 + 63, columns col0 ..
// (the read-outs then own one row per thread, as the epilogues are written)
template <int N>
__device__ __forceinline__ void wg_stage(float *S, int ld, int row0, int col0, const float (&d)[N / 2])
{
    const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    float *p0 = S + (size_t)(row0 + 16 * w + (lane >> 2)) * ld + col0 + 2 * (lane & 3), *p1 = p0 + 8 * ld;
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
        *reinterpret_cast<float2 *>(p0 + 8 * j) = make_float2(d[4 * j], d[4 * j + 1]);
        *reinterpret_cast<float2 *>(p1 + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
}

// K-major, no-swizzle shared-memory matrix descriptor of wgmma: start address >> 4 in [0,14), leading byte offset >> 4 in [16,30)
// (between the two 16-byte K core matrices of one k-step), stride byte offset >> 4 in [32,46) (between 8-row core matrices).
// Descriptors of the same operand differ only in the start-address field: 16-byte-unit offsets are added to a base.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo16, uint32_t sbo16)
{
    return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)(lbo16 & 0x3FFFu) << 16) | ((uint64_t)(sbo16 & 0x3FFFu) << 32);
}

// split 8 floats into fp16 hi / lo and store them as two 16-byte vectors
__device__ __forceinline__ void store_split8(unsigned char *hi_ptr, unsigned char *lo_ptr, const float *v)
{
    __half2 h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float a = v[2 * i], b = v[2 * i + 1];
        a = fminf(fmaxf(a, -65504.0f), 65504.0f);
        b = fminf(fmaxf(b, -65504.0f), 65504.0f);
        __half ha = __float2half_rn(a), hb = __float2half_rn(b);
        h[i] = __halves2half2(ha, hb);
        l[i] = __halves2half2(__float2half_rn(a - __half2float(ha)), __float2half_rn(b - __half2float(hb)));
    }
    *reinterpret_cast<uint4 *>(hi_ptr) = *reinterpret_cast<uint4 *>(h);
    *reinterpret_cast<uint4 *>(lo_ptr) = *reinterpret_cast<uint4 *>(l);
}


// the same for values known to be >= 0 (post-ReLU activations): only the upper clamp, packed conversions
__device__ __forceinline__ void store_split8_pos(unsigned char *hi_ptr, unsigned char *lo_ptr, const float *v)
{
    __half2 h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float a = fminf(v[2 * i], 65504.0f), b = fminf(v[2 * i + 1], 65504.0f);
        h[i] = __floats2half2_rn(a, b);
        const float2 back = __half22float2(h[i]);
        l[i] = __floats2half2_rn(a - back.x, b - back.y);
    }
    *reinterpret_cast<uint4 *>(hi_ptr) = *reinterpret_cast<uint4 *>(h);
    *reinterpret_cast<uint4 *>(lo_ptr) = *reinterpret_cast<uint4 *>(l);
}

}  // namespace lz
