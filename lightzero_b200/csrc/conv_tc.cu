// conv_tc.cu -- generic wgmma 3x3 convolution for the DownSample tower (see conv_tc.cuh for the layout).
// One CTA = one band of image rows (or G small whole images): bulk-copies the band (+halo) of every k-group plane into shared
// memory once, then for each 128-row tile runs 9 taps x (Cin/16) k-steps x 3 fp16 hi/lo passes of wgmma (two warpgroups, 64 rows
// each, accumulators in registers) with row-shifted descriptors; the taps stream through a ring once per tile (L2-resident, 4-16 KB
// each).  The epilogue applies BN / residual / ReLU straight from the accumulator fragments and writes the next layer's TCL tensor
// (already split into fp16 hi/lo).
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "conv_tc.cuh"
#include "tc_ptx.cuh"

namespace lz {

constexpr int kCvConsumers = 256, kCvThreads = kCvConsumers + 32;   // two MMA / epilogue warpgroups + the producer warp
constexpr int kCvStages = 4;          // ring slots reserved in the barrier block; p.stages (2..4) are used

struct CvBars {
    uint64_t full[kCvStages], empty[kCvStages];
    uint64_t in_full;
};

struct CvGeom {                   // identical on host (shared-memory size) and device
    int nbands, rin, m_lo, mcount, NT, PR;
    size_t plane, part, phase, in_bytes, tap_bytes, smem;
};

__host__ __device__ inline CvGeom cv_geom(const ConvTc &p)
{
    CvGeom g;
    const int H = p.in.H, pitch = p.in.pitch, kg = p.in.C / 8;
    g.nbands = (H + p.band_h - 1) / p.band_h;
    g.rin = (p.band_h + 2) * pitch + 2;
    g.m_lo = pitch + 1;
    g.mcount = (p.G - 1) * g.rin + p.band_h * pitch;
    g.NT = (g.mcount + 127) / 128;
    g.PR = g.m_lo + g.NT * 128 + pitch + 2;
    if (g.PR < p.G * g.rin) g.PR = p.G * g.rin;
    g.plane = (size_t)g.PR * 16;
    g.part = (size_t)kg * g.plane;
    g.phase = 2 * g.part;
    g.in_bytes = (g.phase * p.in.nphase + 127) & ~(size_t)127;
    g.tap_bytes = (size_t)2 * kg * p.N * 16;
    g.smem = g.in_bytes + p.stages * g.tap_bytes + 1024;
    return g;
}

// fp16 hi / lo of two consecutive channels (4-byte stores)
__device__ __forceinline__ void store_split2(unsigned char *hi_ptr, unsigned char *lo_ptr, float a, float b)
{
    a = fminf(fmaxf(a, -65504.0f), 65504.0f);
    b = fminf(fmaxf(b, -65504.0f), 65504.0f);
    const __half ha = __float2half_rn(a), hb = __float2half_rn(b);
    *reinterpret_cast<__half2 *>(hi_ptr) = __halves2half2(ha, hb);
    *reinterpret_cast<__half2 *>(lo_ptr) = __halves2half2(__float2half_rn(a - __half2float(ha)), __float2half_rn(b - __half2float(hb)));
}

template <int N>
// N <= 64: <= 112 registers (32 or 16 accumulators per thread), so two CTAs can share an SM and overlap one CTA's band load /
// epilogue with the other's MMAs; N = 128 needs 64 accumulators per thread and runs one CTA per SM
__global__ void __launch_bounds__(kCvThreads, N == 128 ? 1 : 2) k_conv_tc(ConvTc p)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    const CvGeom g = cv_geom(p);
    unsigned char *in_s = smem;
    unsigned char *ring = smem + g.in_bytes;
    CvBars *bars = reinterpret_cast<CvBars *>(ring + p.stages * g.tap_bytes);
    const int nstages = p.stages;
    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;   // warp-uniform value: uniform role branches
    const int pitch = p.in.pitch, H = p.in.H, W = p.in.W, kg_in = p.in.C / 8;
    const int group = blockIdx.x / g.nbands, band = blockIdx.x - group * g.nbands;
    const int img0 = group * p.G, nimg = min(p.G, p.B - img0);
    const int y0 = band * p.band_h;
    const int rin0 = y0 * pitch - 1;
    const int npass = p.npass;

    if (tid == 0) {
        for (int i = 0; i < kCvStages; ++i) { mbar_init(&bars->full[i], 1); mbar_init(&bars->empty[i], kCvConsumers / 32); }
        mbar_init(&bars->in_full, 1);
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == kCvConsumers / 32) {
        // ================= producer: input band, then the 9 weight taps once per tile =================
        if (lane == 0) {
            const int grow0 = rin0 + 1;                                    // memory row of rho = rin0
            const int ncopy = min(g.rin, p.in.plane_rows - grow0);
            const uint32_t bytes = (uint32_t)ncopy * 16u;
            mbar_expect_tx(&bars->in_full, bytes * (uint32_t)(nimg * p.in.nphase * 2 * kg_in));
            for (int k = 0; k < nimg; ++k)
                for (int f = 0; f < p.in.nphase; ++f)
                    for (int part = 0; part < 2; ++part)
                        for (int kg = 0; kg < kg_in; ++kg) {
                            const unsigned char *src = p.in.base + (size_t)(img0 + k) * p.in.img_stride + f * p.in.phase_stride +
                                                       part * p.in.part_stride + ((size_t)kg * p.in.plane_rows + grow0) * 16;
                            unsigned char *dst = in_s + f * g.phase + part * g.part + kg * g.plane + (size_t)k * g.rin * 16;
                            bulk_g2s(dst, src, bytes, &bars->in_full);
                        }
            for (int n = 0; n < 9 * g.NT; ++n) {
                const int st = n % nstages, tap = n % 9;
                if (n >= nstages) mbar_wait(&bars->empty[st], ((n / nstages) - 1) & 1);
                mbar_expect_tx(&bars->full[st], (uint32_t)g.tap_bytes);
                bulk_g2s(ring + st * g.tap_bytes, p.w + (size_t)tap * g.tap_bytes, (uint32_t)g.tap_bytes, &bars->full[st]);
            }
        }
        return;
    }

    // ================= two warpgroups: rows [64 wg, 64 wg + 64) of every tile =================
    const int wg = warp >> 2;
    const uint32_t plane16 = (uint32_t)(g.plane >> 4);
    const uint64_t a_desc0 = make_desc(smem_u32(in_s), plane16, 8);
    const uint64_t b_desc0 = make_desc(smem_u32(ring), 2 * N, 8);        // tap block [kg][N hi rows | N lo rows][16 B]: LBO = 2N rows
    const uint32_t b_lo16 = (uint32_t)N;                                  // the lo rows of a k-group, in 16-byte units
    const uint32_t a_lo16 = (uint32_t)(g.part >> 4);
    const int nks = kg_in / 2;
    const int yend = min(y0 + p.band_h, H);
    const int qc = 2 * (lane & 3);                                        // first of the thread's two columns in each 8-column group
    mbar_wait(&bars->in_full, 0);
    for (int t = 0; t < g.NT; ++t) {
        float acc[N / 2];
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc[i] = 0.0f;
        for (int tap = 0; tap < 9; ++tap) {
            const int n = t * 9 + tap, st = n % nstages;
            mbar_wait(&bars->full[st], (n / nstages) & 1);
            const uint64_t b0 = b_desc0 + (uint64_t)((st * g.tap_bytes) >> 4);
            const uint64_t a0 = a_desc0 + (uint64_t)((p.tap_phase[tap] * g.phase) >> 4) + (uint64_t)(g.m_lo + p.tap_shift[tap] + t * 128 + wg * 64);
            wg_fence();
            for (int ks = 0; ks < nks; ++ks) {
                wgmma_f16<N>(acc, a0 + ks * 2 * plane16, b0 + ks * 4 * N);
                if (npass == 3) {
                    wgmma_f16<N>(acc, a0 + ks * 2 * plane16, b0 + b_lo16 + ks * 4 * N);
                    wgmma_f16<N>(acc, a0 + a_lo16 + ks * 2 * plane16, b0 + ks * 4 * N);
                }
            }
            wg_commit();
            if (tap > 0) {
                wg_wait<1>();
                __syncwarp();
                if (lane == 0) mbar_arrive(&bars->empty[(n - 1) % nstages]);
            }
        }
        wg_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars->empty[(t * 9 + 8) % nstages]);

        // ================= epilogue from the fragment: BN (+residual) (+ReLU) -> fp16 hi/lo -> next layer's TCL =================
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int m = g.m_lo + t * 128 + wg * 64 + 16 * (warp & 3) + (lane >> 2) + 8 * hr;
            const int k = m / g.rin;
            const int rho = rin0 + (m - k * g.rin);
            const int yy = rho / pitch - 1, xx = rho - (yy + 1) * pitch;
            const bool in_band = (k < nimg) && (rho >= pitch) && (yy >= y0) && (yy < yend);
            const bool valid = in_band && (xx < W);
#pragma unroll
            for (int j = 0; j < N / 8; ++j) {
                const int col = 8 * j + qc;
                const int grp = (N == 128) ? (col >> 6) : 0;      // N = 128: columns [64, 128) are the second output tensor
                const int c = col - grp * 64;                     // channel within the output tensor
                const Tcl &o = p.out[grp];
                const bool relu = p.relu[grp] != 0;
                size_t obase = 0;
                bool do_write = in_band;
                if (in_band) {
                    if (o.nphase == 1) {
                        obase = (size_t)(img0 + k) * o.img_stride + (size_t)(rho + 1) * 16;
                    } else if (valid) {                  // phase-split output for a stride-2 consumer
                        const int ph = (yy & 1) * 2 + (xx & 1);
                        const int rho2 = ((yy >> 1) + 1) * o.pitch + (xx >> 1);
                        obase = (size_t)(img0 + k) * o.img_stride + ph * o.phase_stride + (size_t)(rho2 + 1) * 16;
                    } else {
                        do_write = false;
                    }
                }
                float v0 = fmaf(acc[4 * j + 2 * hr], __ldg(p.scale + col), __ldg(p.shift + col));
                float v1 = fmaf(acc[4 * j + 2 * hr + 1], __ldg(p.scale + col + 1), __ldg(p.shift + col + 1));
                if (p.res.base && grp == 0 && valid) {
                    const unsigned char *rp = p.res.base + (size_t)(img0 + k) * p.res.img_stride +
                                              ((size_t)(c >> 3) * p.res.plane_rows + rho + 1) * 16 + (c & 7) * 2;
                    const float2 a = __half22float2(*reinterpret_cast<const __half2 *>(rp));
                    const float2 b = __half22float2(*reinterpret_cast<const __half2 *>(rp + p.res.part_stride));
                    v0 += a.x + b.x;
                    v1 += a.y + b.y;
                }
                v0 = valid ? (relu ? fmaxf(v0, 0.0f) : v0) : 0.0f;
                v1 = valid ? (relu ? fmaxf(v1, 0.0f) : v1) : 0.0f;
                if (do_write) {
                    unsigned char *op = o.base + obase + (size_t)(c >> 3) * o.plane_rows * 16 + (c & 7) * 2;
                    store_split2(op, op + o.part_stride, v0, v1);
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- pools
__device__ __forceinline__ void tcl_load8(const Tcl &t, int img, int kg, int rho, float (&v)[8])
{
    const unsigned char *pp = t.base + (size_t)img * t.img_stride + ((size_t)kg * t.plane_rows + rho + 1) * 16;
    const uint4 rh = __ldg(reinterpret_cast<const uint4 *>(pp));
    const uint4 rl = __ldg(reinterpret_cast<const uint4 *>(pp + t.part_stride));
    const __half2 *hh = reinterpret_cast<const __half2 *>(&rh), *hl = reinterpret_cast<const __half2 *>(&rl);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 a = __half22float2(hh[j]), b = __half22float2(hl[j]);
        v[2 * j] = a.x + b.x;
        v[2 * j + 1] = a.y + b.y;
    }
}

// AvgPool2d(3, 2, 1), divisor 9.  The zero pad column / rows of TCL supply the padding.
__global__ void k_pool_tcl(Tcl in, Tcl out, float *out_nchw, int B, int Hout)
{
    const int kgs = in.C / 8;
    const size_t n = (size_t)B * kgs * Hout * Hout;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int xo = (int)(i % Hout), yo = (int)((i / Hout) % Hout);
        const int kg = (int)((i / ((size_t)Hout * Hout)) % kgs), img = (int)(i / ((size_t)Hout * Hout * kgs));
        float s[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j] = 0.0f;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int yy = 2 * yo + ky - 1;
            if (yy < 0 || yy >= in.H) continue;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int xx = 2 * xo + kx - 1;
                if (xx < 0 || xx >= in.W) continue;
                float v[8];
                tcl_load8(in, img, kg, (yy + 1) * in.pitch + xx, v);
#pragma unroll
                for (int j = 0; j < 8; ++j) s[j] += v[j];
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j] = s[j] / 9.0f;
        if (out_nchw) {
#pragma unroll
            for (int j = 0; j < 8; ++j) out_nchw[((size_t)img * in.C + kg * 8 + j) * Hout * Hout + yo * Hout + xo] = s[j];
        } else {
            unsigned char *op = out.base + (size_t)img * out.img_stride + ((size_t)kg * out.plane_rows + (yo + 1) * out.pitch + xo + 1) * 16;
            store_split8(op, op + out.part_stride, s);
        }
    }
}

// ---------------------------------------------------------------------------------------------- host
int conv_tc_prepare_launch()
{
    const int big = 227 * 1024;
    LZ_CUDA_CHECK(cudaFuncSetAttribute(k_conv_tc<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, big));
    LZ_CUDA_CHECK(cudaFuncSetAttribute(k_conv_tc<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, big));
    LZ_CUDA_CHECK(cudaFuncSetAttribute(k_conv_tc<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, big));
    return LZ_OK;
}

int conv_tc_launch(const ConvTc &p, cudaStream_t s)
{
    const CvGeom g = cv_geom(p);
    LZ_REQUIRE(g.smem <= 227 * 1024, LZ_EINVAL, "conv_tc: band needs %zu B shared memory", g.smem);
    LZ_REQUIRE(g.tap_bytes <= 16384 && (p.in.C % 16) == 0, LZ_EINVAL, "conv_tc: unsupported channel counts");
    const int groups = (p.B + p.G - 1) / p.G;
    const int grid = groups * g.nbands;
    switch (p.N) {
        case 32: k_conv_tc<32><<<grid, kCvThreads, g.smem, s>>>(p); break;
        case 64: k_conv_tc<64><<<grid, kCvThreads, g.smem, s>>>(p); break;
        case 128: k_conv_tc<128><<<grid, kCvThreads, g.smem, s>>>(p); break;
        default: LZ_REQUIRE(false, LZ_EINVAL, "conv_tc: N must be 32, 64 or 128");
    }
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

size_t conv_tc_packed_bytes(int cin, int ncols) { return (size_t)9 * 2 * (cin / 8) * ncols * 16; }

float conv_tc_pack(const float *w, int cin, int cout, int ncols, int col0, unsigned char *dst)
{
    float mx = 0.0f;
    for (size_t i = 0; i < (size_t)cout * cin * 9; ++i) mx = std::max(mx, fabsf(w[i]));
    int e = 0;
    if (mx > 0.0f) frexpf(mx, &e);
    const float scale = ldexpf(1.0f, 13 - e);
    // tap block: [k-group ci / 8][ncols hi rows | ncols lo rows][ci % 8]: [B_hi | B_lo] of a k-group is one contiguous 2 x ncols-row operand
    const size_t tap_halves = (size_t)2 * (cin / 8) * ncols * 8, part_halves = (size_t)ncols * 8;
    __half *h = reinterpret_cast<__half *>(dst);
    for (int t = 0; t < 9; ++t)
        for (int co = 0; co < cout; ++co)
            for (int ci = 0; ci < cin; ++ci) {
                const float sv = w[((size_t)co * cin + ci) * 9 + t] * scale;
                const __half hi = __float2half_rn(sv);
                const __half lo = __float2half_rn(sv - __half2float(hi));
                const size_t off = (size_t)t * tap_halves + ((size_t)(ci / 8) * 2 * ncols + col0 + co) * 8 + (ci % 8);
                h[off] = hi;
                h[off + part_halves] = lo;
            }
    return scale;
}

int pool_tcl_launch(const Tcl &in, const Tcl &out, int B, cudaStream_t s)
{
    const size_t n = (size_t)B * (in.C / 8) * out.H * out.W;
    k_pool_tcl<<<(int)std::min<size_t>((n + 255) / 256, kNumSMs * 32), 256, 0, s>>>(in, out, nullptr, B, out.H);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

int pool_tcl_to_nchw_launch(const Tcl &in, float *out, int B, int Hout, cudaStream_t s)
{
    const size_t n = (size_t)B * (in.C / 8) * Hout * Hout;
    Tcl dummy = in;
    k_pool_tcl<<<(int)std::min<size_t>((n + 255) / 256, kNumSMs * 32), 256, 0, s>>>(in, dummy, out, B, Hout);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

}  // namespace lz
