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

// cudaFree of a live buffer waits for all work on the device; a null pointer skips the call
inline void dev_free(void *p)
{
    if (p) cudaFree(p);
}

// Device writes of the setup entry points (create, set_params, set_gumbel, finalize): they go on a library-owned non-blocking
// stream of the current device and are complete when the call returns, so they never queue behind work on the legacy default
// stream (a learner's backward pass, say) and a caller's stream may use what they wrote right away.  Defined in tree.cu.
int setup_memset(void *d, size_t bytes);                    // zeroes d[0, bytes)
int setup_upload(void *d, const void *h, size_t bytes);     // copies host bytes to the device
int setup_stream(cudaStream_t *s);                          // the stream itself: enqueue on it, then setup_sync
int setup_sync();

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

constexpr int kNumSMs = 132;       // streaming multiprocessors of the H100 SXM the grid sizes are tuned for

}  // namespace lz
