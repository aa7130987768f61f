// lz_common.cuh -- shared host-side plumbing for the C ABI (error strings, CUDA checks).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "../../include/lzb200.h"

namespace lz {

void set_error(const char *fmt, ...);
void count_launch(int n = 1);      // launch accounting (lz_debug_launch_count): kernels enqueued by this library, graph nodes included

#define LZ_CUDA_CHECK(expr)                                                                    \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            lz::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            (void)cudaGetLastError(); /* clear the non-sticky error so later calls do not re-report it */ \
            return LZ_ECUDA;                                                                   \
        }                                                                                      \
    } while (0)

#define LZ_REQUIRE(cond, code, ...)          \
    do {                                     \
        if (!(cond)) {                       \
            lz::set_error(__VA_ARGS__);      \
            return (code);                   \
        }                                    \
    } while (0)

#define LZ_KERNEL_CHECK()                    \
    do {                                     \
        lz::count_launch();                  \
        LZ_CUDA_CHECK(cudaGetLastError());   \
    } while (0)

template <typename T>
inline int dev_alloc(T **p, size_t n)
{
    cudaError_t e = cudaMalloc((void **)p, n * sizeof(T));
    if (e != cudaSuccess) {
        set_error("cudaMalloc(%zu bytes) failed: %s", n * sizeof(T), cudaGetErrorString(e));
        return LZ_ENOMEM;
    }
    return LZ_OK;
}

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

constexpr int kNumSMs = 132;       // streaming multiprocessors of the H100 SXM the grid sizes are tuned for

}  // namespace lz
