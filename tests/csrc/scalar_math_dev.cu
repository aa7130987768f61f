// scalar_math_dev.cu -- test harness (tests/test_gpu_scalar_readout.py): the library's scalar primitives applied on the device to
// an array of floats, and libm's expf / logf applied on the host, so that the device copies of net6.cuh's
// inverse_scalar_transform and lz_exact_math.h's lz_expf_exact / lz_logf_exact can be swept against their references.  The
// test builds it twice, with -fmad=false and with contraction on, as the library compiles these headers both ways.
#include <math.h>
#include <stdint.h>

#include "net6.cuh"
#include "lz_exact_math.h"

namespace {

__global__ void k_apply(int fn, const float *in, float *out, long long n)
{
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float x = in[i];
        out[i] = fn == 0 ? lz::inverse_scalar_transform(x) : fn == 1 ? lz_expf_exact(x) : lz_logf_exact(x);
    }
}

__global__ void k_support(float support_min, float support_step, int K, float *out)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < K) out[k] = lz::support_at(support_min, support_step, k);
}

}  // namespace

extern "C" {

// fn: 0 = inverse_scalar_transform, 1 = lz_expf_exact, 2 = lz_logf_exact; `stream` is a cudaStream_t
int sm_apply(int fn, const float *d_in, float *d_out, long long n, void *stream)
{
    if (fn < 0 || fn > 2 || n <= 0) return 1;
    k_apply<<<1024, 256, 0, (cudaStream_t)stream>>>(fn, d_in, d_out, n);
    return (int)cudaGetLastError();
}

// support value k = support_at(min, step, k) for k < K
int sm_support(float support_min, float support_step, int K, float *d_out, void *stream)
{
    if (K <= 0) return 1;
    k_support<<<(K + 255) / 256, 256, 0, (cudaStream_t)stream>>>(support_min, support_step, K, d_out);
    return (int)cudaGetLastError();
}

// libm on the host: fn 1 = expf, 2 = logf
int sm_host_libm(int fn, const float *in, float *out, long long n)
{
    if (fn == 1) for (long long i = 0; i < n; ++i) out[i] = expf(in[i]);
    else if (fn == 2) for (long long i = 0; i < n; ++i) out[i] = logf(in[i]);
    else return 1;
    return 0;
}

}  // extern "C"
