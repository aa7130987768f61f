// conv_tc.cu -- generic wgmma 3x3 convolution for the DownSample tower (see conv_tc.cuh for the layout).
// One CTA = one band of image rows (or G small whole images): bulk-copies the band (+halo) of every k-group plane into shared
// memory once, then for each 128-row tile runs 9 taps x (Cin/16) k-steps x 3 fp16 hi/lo passes of wgmma (two warpgroups, 64 rows
// each, accumulators in registers) with row-shifted descriptors; the taps stream through a ring once per tile group (L2-resident,
// 4-16 KB each; see tc_group).  The epilogue applies BN / residual / ReLU straight from the accumulator fragments and writes the next layer's TCL tensor
// (already split into fp16 hi/lo).  k_resblock_tc runs both convs of a plain ResBlock the same way, with conv1's output kept in
// shared memory.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "conv_tc.cuh"
#include "model.cuh"
#include "tc_ptx.cuh"

namespace lz {

// Two MMA / epilogue warpgroups + the producer, in one of two layouts (the kernels' Wide parameter):
//   narrow: a single producer warp, 288 threads.  They are allocated registers as 12 warps, which caps every thread at 168.
//   wide:   a whole producer warpgroup, 384 threads, that hands its registers to the MMA warpgroups (kProducerRegs /
//           kConsumerRegs, tc_ptx.cuh), which then hold more accumulator slabs.
// The wide layout only pays where a plan's tiles need more slabs than the narrow one holds: a launch whose tile groups would not
// grow measured 1-4 % slower in it (H100 80GB HBM3, 700 W), so each launch picks the layout from its plan (conv_tc_launch, rb_wide).
constexpr int kCvConsumers = 256;
template <bool Wide>
constexpr int kCvThreads = kCvConsumers + (Wide ? 128 : 32);
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

// A conv's NT tiles run in groups of at most MT tiles, split evenly (5 tiles with MT = 4: 3 + 2): ng groups of `per` tiles, the
// last one possibly shorter
__host__ __device__ inline void tile_groups(int NT, int MT, int &ng, int &per)
{
    ng = (NT + MT - 1) / MT;
    per = (NT + ng - 1) / ng;
}

// The MMAs of one tile group, tap-major: for each of the 9 taps (ring slots n0 .. n0 + 8, each fetched once per group and released
// as soon as its wgmmas are done), every k-step of every tile of the group.  The warpgroup's 64-row slabs of the nt <= MT tiles
// are independent accumulator chains, so the tensor pipe has nt chains to interleave instead of waiting on one chain's wgmma
// latency, and each tap crosses the ring once per group rather than once per tile.  Each row's sums keep the tap -> k-step ->
// pass order.  tap_a(tap) is tile 0's A descriptor at that tap; tile_ready(s) runs before tile s's first wgmma.
// KS > 0: KS k-steps, unrolled (the ResBlocks, Cin = N).  KS = 0: nks k-steps in a rolled loop (k_conv_tc: fewer live descriptor
// registers, no spill at N = 128, and its 84-px launch ran 457 -> 406 us on an H100 80GB HBM3 at 700 W).
template <int N, int MT, int KS, typename TapA, typename TileReady>
__device__ __forceinline__ void tc_group(float (&acc)[MT][N / 2], int nt, TapA tap_a, TileReady tile_ready, int nks, int npass,
                                         uint32_t plane16, uint32_t a_lo16, uint64_t b_desc0, size_t tap_bytes, int nstages,
                                         uint64_t *full, uint64_t *empty, int n0, int lane)
{
    const uint32_t b_lo16 = (uint32_t)N;                                  // the lo rows of a k-group, in 16-byte units
#pragma unroll
    for (int s = 0; s < MT; ++s)
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc[s][i] = 0.0f;
    for (int tap = 0; tap < 9; ++tap) {
        const int n = n0 + tap, st = n % nstages;
        mbar_wait(&full[st], (n / nstages) & 1);
        const uint64_t b0 = b_desc0 + (uint64_t)((st * tap_bytes) >> 4);
        const uint64_t a0 = tap_a(tap);
        auto kstep = [&](int ks) {
#pragma unroll
            for (int s = 0; s < MT; ++s) {
                if (s >= nt) break;
                if (tap == 0 && ks == 0) tile_ready(s);
                const uint64_t as = a0 + s * 128 + ks * 2 * plane16;
                wgmma_f16<N>(acc[s], as, b0 + ks * 4 * N);
                if (npass == 3) {
                    wgmma_f16<N>(acc[s], as, b0 + b_lo16 + ks * 4 * N);
                    wgmma_f16<N>(acc[s], as + a_lo16, b0 + ks * 4 * N);
                }
            }
        };
        wg_fence();
        if constexpr (KS > 0) {
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) kstep(ks);
        } else {
#pragma unroll 1
            for (int ks = 0; ks < nks; ++ks) kstep(ks);
        }
        wg_commit();
        if (tap > 0) {
            wg_wait<1>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[(n - 1) % nstages]);
        }
    }
    wg_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[(n0 + 8) % nstages]);
}

// Tiles in flight per warpgroup (accumulator slabs of N / 2 registers each).  Narrow: one.  N = 64 stays within 112 registers, so two
// CTAs share an SM and one CTA's band load and epilogue overlap the other's MMAs; N = 128 runs one CTA per SM.  Wide (N = 128 only):
// two slabs (128 accumulators, which spilled in the epilogue at 168 registers, CUDA 12.9), for bands of two or more tiles.
template <bool Wide>
constexpr int kCvTiles = Wide ? 2 : 1;

template <int N, bool Wide>
__global__ void __launch_bounds__(kCvThreads<Wide>, N == 128 ? 1 : 2) k_conv_tc(ConvTc p)
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
    constexpr int MT = kCvTiles<Wide>;
    int ng, per;
    tile_groups(g.NT, MT, ng, per);

    if (tid == 0) {
        for (int i = 0; i < kCvStages; ++i) { mbar_init(&bars->full[i], 1); mbar_init(&bars->empty[i], kCvConsumers / 32); }
        mbar_init(&bars->in_full, 1);
        fence_mbar_init();
    }
    __syncthreads();

    if (warp >= kCvConsumers / 32) {
        // ================= producer: input band, then the 9 weight taps once per tile group =================
        if constexpr (Wide) wg_reg_dealloc<kProducerRegs>();
        if (warp == kCvConsumers / 32 && lane == 0) {
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
            for (int n = 0; n < 9 * ng; ++n) {
                const int st = n % nstages, tap = n % 9;
                if (n >= nstages) mbar_wait(&bars->empty[st], ((n / nstages) - 1) & 1);
                mbar_expect_tx(&bars->full[st], (uint32_t)g.tap_bytes);
                bulk_g2s(ring + st * g.tap_bytes, p.w + (size_t)tap * g.tap_bytes, (uint32_t)g.tap_bytes, &bars->full[st]);
            }
        }
        return;
    }

    // ================= two warpgroups: rows [64 wg, 64 wg + 64) of every tile =================
    if constexpr (Wide) wg_reg_alloc<kConsumerRegs>();
    const int wg = warp >> 2;
    const uint32_t plane16 = (uint32_t)(g.plane >> 4);
    const uint64_t a_desc0 = make_desc(smem_u32(in_s), plane16, 8);
    const uint64_t b_desc0 = make_desc(smem_u32(ring), 2 * N, 8);        // tap block [kg][N hi rows | N lo rows][16 B]: LBO = 2N rows
    const uint32_t a_lo16 = (uint32_t)(g.part >> 4);
    const int yend = min(y0 + p.band_h, H);
    const int qc = 2 * (lane & 3);                                        // first of the thread's two columns in each 8-column group
    mbar_wait(&bars->in_full, 0);
    for (int gi = 0; gi < ng; ++gi) {
        const int t0 = gi * per, nt = min(per, g.NT - t0);
        float acc[MT][N / 2];
        auto tap_a = [&](int tap) {
            return a_desc0 + (uint64_t)((p.tap_phase[tap] * g.phase) >> 4) + (uint64_t)(g.m_lo + p.tap_shift[tap] + t0 * 128 + wg * 64);
        };
        tc_group<N, MT, 0>(acc, nt, tap_a, [](int) {}, kg_in / 2, p.npass, plane16, a_lo16, b_desc0, g.tap_bytes, nstages, bars->full,
                           bars->empty, gi * 9, lane);

        // ================= epilogue from the fragment: BN (+residual) (+ReLU) -> fp16 hi/lo -> next layer's TCL =================
#pragma unroll
        for (int e = 0; e < 2 * MT; ++e) {
            const int s = e >> 1, hr = e & 1;
            if (s >= nt) break;
            const int m = g.m_lo + (t0 + s) * 128 + wg * 64 + 16 * (warp & 3) + (lane >> 2) + 8 * hr;
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
                float v0 = fmaf(acc[s][4 * j + 2 * hr], __ldg(p.scale + col), __ldg(p.shift + col));
                float v1 = fmaf(acc[s][4 * j + 2 * hr + 1], __ldg(p.scale + col + 1), __ldg(p.shift + col + 1));
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
                if (in_band) {
                    unsigned char *op = o.base + (size_t)(img0 + k) * o.img_stride + ((size_t)(c >> 3) * o.plane_rows + rho + 1) * 16 + (c & 7) * 2;
                    store_split2(op, op + o.part_stride, v0, v1);
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- fused ResBlock
// k_resblock_tc runs relu(bn2(conv2(relu(bn1(conv1(x))))) + x) for one band of h output rows (or G whole images) per CTA.  Both
// shared-memory buffers use the TCL plane layout with a per-image stride of S = (h + 4) pitch + 2 rows:
//   input x:          row j of image k = memory row (y0 - 1) pitch + j - k S,  i.e. image rows [y0 - 2, y0 + h + 2)
//   intermediate t1:  row i of image k = memory row y0 pitch + i - k S,        i.e. image rows [y0 - 1, y0 + h + 1)
// conv1 computes the h + 2 rows [y0 - 1, y0 + h] (the halo rows conv2 needs are recomputed) exactly like k_conv_tc on the band
// (y0 - 1, h + 2): its output row m is t1 row m - pitch, stored as fp16 hi/lo, and rows outside the image (or the pad column) are
// stored as zeros, so conv2 reads t1 through the same row-shifted descriptors as an HBM band.  conv2's output row m takes its
// residual from x row m + pitch.  Each output row's sums run in the same tap -> k-step -> pass order as two k_conv_tc launches,
// and t1 holds the same fp16 split they pass through HBM, so the results are bit-identical to them.
// The input band lands in 128-row chunks, each with its own mbarrier: conv1's first pair of tiles starts once its rows are in,
// while the rest of the band is still loading (with ~200 KB of shared memory per CTA, no second CTA can hide the load).
// Reads past a buffer's last plane (only by tile rows past the last useful one, < 128 rows) land in the next buffer or the ring.
constexpr int kRbChunks = 16;

struct RbBars {
    uint64_t full[kCvStages], empty[kCvStages];
    uint64_t chunk[kRbChunks];
};

struct RbGeom {                   // identical on host (shared-memory size, band picker) and device
    int nbands, S, m_lo, NT1, NT2, PR, nchunk;
    size_t plane, part, buf, tap_bytes, smem;
};

__host__ __device__ inline RbGeom rb_geom(const ResBlockTc &p)
{
    RbGeom g;
    const int H = p.in.H, pitch = p.in.pitch, kg = p.in.C / 8;
    g.nbands = (H + p.band_h - 1) / p.band_h;
    g.S = (p.band_h + 4) * pitch + 2;
    g.m_lo = pitch + 1;
    g.NT1 = ((p.G - 1) * g.S + (p.band_h + 2) * pitch + 127) / 128;
    g.NT2 = ((p.G - 1) * g.S + p.band_h * pitch + 127) / 128;
    g.PR = p.G * g.S;
    g.nchunk = (g.PR + 127) / 128;
    g.plane = (size_t)g.PR * 16;
    g.part = (size_t)kg * g.plane;
    g.buf = (2 * g.part + 127) & ~(size_t)127;
    g.tap_bytes = (size_t)2 * kg * p.in.C * 16;
    g.smem = 2 * g.buf + p.stages * g.tap_bytes + 1024;
    return g;
}

// Tiles in flight per warpgroup: the accumulator slabs (N / 2 registers each) of a whole conv at N = 32 (84-px resblocks1: NT1 = 6,
// NT2 = 5; 151 registers, narrow), two slabs at N = 64 narrow and four wide (128 accumulators; three or four spilled in the epilogue
// at 168 registers, CUDA 12.9).  The kernel runs one CTA per SM (~200 KB of shared memory), so only independent chains within the
// CTA hide wgmma latency.
template <int N, bool Wide>
constexpr int kRbTiles = N == 32 ? 6 : (Wide ? 4 : 2);

// The slabs a ResBlock plan runs with: the wide layout once a conv has more tiles than the narrow one holds (N = 64 only)
__host__ __device__ inline bool rb_wide(int C, const RbGeom &g) { return C == 64 && (g.NT1 > kRbTiles<64, false> || g.NT2 > kRbTiles<64, false>); }
__host__ __device__ inline int rb_tiles(int C, const RbGeom &g)
{
    return C == 32 ? kRbTiles<32, false> : (rb_wide(C, g) ? kRbTiles<64, true> : kRbTiles<64, false>);
}

template <int N, bool Wide>
__global__ void __launch_bounds__(kCvThreads<Wide>, 1) k_resblock_tc(ResBlockTc p)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    const RbGeom g = rb_geom(p);
    unsigned char *in_s = smem, *mid_s = smem + g.buf, *ring = smem + 2 * g.buf;
    RbBars *bars = reinterpret_cast<RbBars *>(ring + p.stages * g.tap_bytes);
    const int nstages = p.stages;
    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;   // warp-uniform value: uniform role branches
    const int pitch = p.in.pitch, H = p.in.H, W = p.in.W, kg_in = N / 8;
    const int group = blockIdx.x / g.nbands, band = blockIdx.x - group * g.nbands;
    const int img0 = group * p.G, nimg = min(p.G, p.B - img0);
    const int y0 = band * p.band_h;
    constexpr int MT = kRbTiles<N, Wide>;
    int ng1, per1, ng2, per2;
    tile_groups(g.NT1, MT, ng1, per1);
    tile_groups(g.NT2, MT, ng2, per2);
    const int ntaps = 9 * (ng1 + ng2);                                    // the taps stream once per tile group

    if (tid == 0) {
        for (int i = 0; i < kCvStages; ++i) { mbar_init(&bars->full[i], 1); mbar_init(&bars->empty[i], kCvConsumers / 32); }
        for (int c = 0; c < g.nchunk; ++c) mbar_init(&bars->chunk[c], 1);
        fence_mbar_init();
    }
    __syncthreads();

    if (warp >= kCvConsumers / 32) {
        // ================= producer: the first ring fill, the input band chunk by chunk, then conv1's and conv2's taps =================
        if constexpr (Wide) wg_reg_dealloc<kProducerRegs>();
        if (warp == kCvConsumers / 32 && lane == 0) {
            auto load_tap = [&](int n) {
                const int st = n % nstages, tap = n % 9;
                if (n >= nstages) mbar_wait(&bars->empty[st], ((n / nstages) - 1) & 1);
                mbar_expect_tx(&bars->full[st], (uint32_t)g.tap_bytes);
                bulk_g2s(ring + st * g.tap_bytes, p.w[n >= 9 * ng1] + (size_t)tap * g.tap_bytes, (uint32_t)g.tap_bytes, &bars->full[st]);
            };
            for (int n = 0; n < nstages; ++n) load_tap(n);   // queued ahead of the band, so that conv1's first tile waits on its rows only
            // rows outside the tensor (above the first band, below the last) are not copied: they only feed conv1 rows outside
            // the image, which are stored as zeros whatever they hold
            const int g0 = (y0 - 1) * pitch;
            const int r0 = max(0, -g0), r1 = min(g.S, p.in.plane_rows - g0);
            for (int c = 0; c < g.nchunk; ++c) {
                uint32_t rows = 0;
                for (int k = 0; k < nimg; ++k) rows += (uint32_t)max(0, min(k * g.S + r1, c * 128 + 128) - max(k * g.S + r0, c * 128));
                mbar_expect_tx(&bars->chunk[c], rows * 16u * (uint32_t)(2 * kg_in));
                for (int k = 0; k < nimg; ++k) {
                    const int lo = max(k * g.S + r0, c * 128), hi = min(k * g.S + r1, c * 128 + 128);
                    if (hi <= lo) continue;
                    for (int part = 0; part < 2; ++part)
                        for (int kg = 0; kg < kg_in; ++kg) {
                            const unsigned char *src = p.in.base + (size_t)(img0 + k) * p.in.img_stride + part * p.in.part_stride +
                                                       ((size_t)kg * p.in.plane_rows + g0 + lo - k * g.S) * 16;
                            bulk_g2s(in_s + part * g.part + kg * g.plane + (size_t)lo * 16, src, (uint32_t)(hi - lo) * 16u, &bars->chunk[c]);
                        }
                }
            }
            for (int n = nstages; n < ntaps; ++n) load_tap(n);
        }
        return;
    }

    // ================= two warpgroups: rows [64 wg, 64 wg + 64) of every tile =================
    if constexpr (Wide) wg_reg_alloc<kConsumerRegs>();
    const int wg = warp >> 2;
    const uint32_t plane16 = (uint32_t)(g.plane >> 4);
    const uint64_t in_desc = make_desc(smem_u32(in_s), plane16, 8), mid_desc = make_desc(smem_u32(mid_s), plane16, 8);
    const uint64_t b_desc0 = make_desc(smem_u32(ring), 2 * N, 8);        // tap block [kg][N hi rows | N lo rows][16 B]: LBO = 2N rows
    const uint32_t a_lo16 = (uint32_t)(g.part >> 4);
    const int qc = 2 * (lane & 3);                                        // first of the thread's two columns in each 8-column group
    // t1 row 0 (the pad column left of image 0's first halo row) is read by conv2 but is no conv1 output row
    if (tid < 2 * kg_in) *reinterpret_cast<uint4 *>(mid_s + tid * g.plane) = make_uint4(0u, 0u, 0u, 0u);

    // ================= conv1 -> BN -> ReLU -> t1 (shared memory) =================
    int ready = 0;                                                        // input chunks known to have landed
    for (int gi = 0; gi < ng1; ++gi) {
        const int t0 = gi * per1, nt = min(per1, g.NT1 - t0);
        float acc[MT][N / 2];
        auto tap_a = [&](int tap) { return in_desc + (uint64_t)(g.m_lo + t0 * 128 + wg * 64 + p.tap_shift[tap]); };
        // tile t reads rows [128 t, 128 t + 128 + 2 pitch + 2) over its 9 taps: in the first tap it waits for their chunks only,
        // so its MMAs start while the rest of the band is still landing
        auto tile_ready = [&](int s) {
            const int need = min(g.nchunk, ((t0 + s) * 128 + 128 + 2 * pitch + 1) / 128 + 1);
            for (; ready < need; ++ready) mbar_wait(&bars->chunk[ready], 0);
        };
        tc_group<N, MT, N / 16>(acc, nt, tap_a, tile_ready, N / 16, p.npass, plane16, a_lo16, b_desc0, g.tap_bytes, nstages, bars->full,
                                bars->empty, gi * 9, lane);
#pragma unroll
        for (int e = 0; e < 2 * MT; ++e) {
            const int s = e >> 1, hr = e & 1;
            if (s >= nt) break;
            const int m = g.m_lo + (t0 + s) * 128 + wg * 64 + 16 * (warp & 3) + (lane >> 2) + 8 * hr;
            const int i = m - pitch;
            const int k = m / g.S;
            const int rho = (y0 - 1) * pitch - 1 + (m - k * g.S);
            const int yy = rho / pitch - 1, xx = rho - (yy + 1) * pitch;
            const bool valid = (k < nimg) && (rho >= pitch) && (yy >= y0 - 1) && (yy <= y0 + p.band_h) && (yy < H) && (xx < W);
            if (i >= g.PR) continue;
#pragma unroll
            for (int j = 0; j < N / 8; ++j) {
                const int col = 8 * j + qc;
                float v0 = fmaf(acc[s][4 * j + 2 * hr], __ldg(p.scale[0] + col), __ldg(p.shift[0] + col));
                float v1 = fmaf(acc[s][4 * j + 2 * hr + 1], __ldg(p.scale[0] + col + 1), __ldg(p.shift[0] + col + 1));
                v0 = valid ? fmaxf(v0, 0.0f) : 0.0f;
                v1 = valid ? fmaxf(v1, 0.0f) : 0.0f;
                unsigned char *op = mid_s + (size_t)(col >> 3) * g.plane + (size_t)i * 16 + (col & 7) * 2;
                store_split2(op, op + g.part, v0, v1);
            }
        }
    }
    for (; ready < g.nchunk; ++ready) mbar_wait(&bars->chunk[ready], 0);   // the residual reads every input row
    fence_proxy_async();                                                  // t1's stores -> conv2's wgmma reads
    asm volatile("bar.sync 1, %0;\n" ::"n"(kCvConsumers) : "memory");

    // ================= conv2 -> BN -> + x -> ReLU -> output TCL =================
    const int yend = min(y0 + p.band_h, H);
    for (int gi = 0; gi < ng2; ++gi) {
        const int t0 = gi * per2, nt = min(per2, g.NT2 - t0);
        float acc[MT][N / 2];
        auto tap_a = [&](int tap) { return mid_desc + (uint64_t)(g.m_lo + t0 * 128 + wg * 64 + p.tap_shift[tap]); };
        tc_group<N, MT, N / 16>(acc, nt, tap_a, [](int) {}, N / 16, p.npass, plane16, a_lo16, b_desc0, g.tap_bytes, nstages, bars->full,
                                bars->empty, (ng1 + gi) * 9, lane);
#pragma unroll
        for (int e = 0; e < 2 * MT; ++e) {
            const int s = e >> 1, hr = e & 1;
            if (s >= nt) break;
            const int m = g.m_lo + (t0 + s) * 128 + wg * 64 + 16 * (warp & 3) + (lane >> 2) + 8 * hr;
            const int k = m / g.S;
            const int rho = y0 * pitch - 1 + (m - k * g.S);
            const int yy = rho / pitch - 1, xx = rho - (yy + 1) * pitch;
            const bool in_band = (k < nimg) && (rho >= pitch) && (yy >= y0) && (yy < yend);
            const bool valid = in_band && (xx < W);
            const Tcl &o = p.out;
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
#pragma unroll
            for (int j = 0; j < N / 8; ++j) {
                const int col = 8 * j + qc;
                float v0 = fmaf(acc[s][4 * j + 2 * hr], __ldg(p.scale[1] + col), __ldg(p.shift[1] + col));
                float v1 = fmaf(acc[s][4 * j + 2 * hr + 1], __ldg(p.scale[1] + col + 1), __ldg(p.shift[1] + col + 1));
                if (valid) {
                    const unsigned char *rp = in_s + (size_t)(col >> 3) * g.plane + (size_t)(m + pitch) * 16 + (col & 7) * 2;
                    const float2 a = __half22float2(*reinterpret_cast<const __half2 *>(rp));
                    const float2 b = __half22float2(*reinterpret_cast<const __half2 *>(rp + g.part));
                    v0 += a.x + b.x;
                    v1 += a.y + b.y;
                }
                v0 = valid ? fmaxf(v0, 0.0f) : 0.0f;
                v1 = valid ? fmaxf(v1, 0.0f) : 0.0f;
                if (do_write) {
                    unsigned char *op = o.base + obase + (size_t)(col >> 3) * o.plane_rows * 16 + (col & 7) * 2;
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

// TCL -> fp32 NCHW, no pooling (the 64-pixel tower ends on the 8x8 grid: DownSample has no pooling2 there, common.py:357-359).
// Each value is hi + lo, the same sum tcl_load8 gives the pools.
__global__ void k_tcl_to_nchw(Tcl in, float *out_nchw, int B)
{
    const int kgs = in.C / 8, H = in.H, W = in.W;
    const size_t n = (size_t)B * kgs * H * W;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(i % W), y = (int)((i / W) % H);
        const int kg = (int)((i / ((size_t)W * H)) % kgs), img = (int)(i / ((size_t)W * H * kgs));
        float v[8];
        tcl_load8(in, img, kg, (y + 1) * in.pitch + x, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) out_nchw[((size_t)img * in.C + kg * 8 + j) * H * W + y * W + x] = v[j];
    }
}

// ---------------------------------------------------------------------------------------------- host
int conv_tc_prepare_launch()
{
    const int big = 227 * 1024;
    LZ_CUDA_CHECK(cudaFuncSetAttribute(k_conv_tc<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, big));
    LZ_CUDA_CHECK(cudaFuncSetAttribute(k_conv_tc<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, big));
    LZ_CUDA_CHECK(cudaFuncSetAttribute(k_conv_tc<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, big));
    LZ_CUDA_CHECK(cudaFuncSetAttribute(k_resblock_tc<32, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, big));
    LZ_CUDA_CHECK(cudaFuncSetAttribute(k_resblock_tc<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, big));
    LZ_CUDA_CHECK(cudaFuncSetAttribute(k_resblock_tc<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, big));
    return LZ_OK;
}

int conv_tc_launch(const ConvTc &p, cudaStream_t s)
{
    const CvGeom g = cv_geom(p);
    LZ_REQUIRE(g.smem <= 227 * 1024, LZ_EINVAL, "conv_tc: band needs %zu B shared memory", g.smem);
    LZ_REQUIRE(g.tap_bytes <= 16384 && (p.in.C % 16) == 0, LZ_EINVAL, "conv_tc: unsupported channel counts");
    LZ_REQUIRE(p.out[0].nphase == 1 && (p.N < 128 || p.out[1].nphase == 1), LZ_EINVAL, "conv_tc: phase-split output is not supported");
    const int groups = (p.B + p.G - 1) / p.G;
    const int grid = groups * g.nbands;
    // N = 128: the wide layout for bands of two or more tiles (two slabs); a one-tile band gains nothing from it
    switch (p.N) {
        case 64: k_conv_tc<64, false><<<grid, kCvThreads<false>, g.smem, s>>>(p); break;
        case 128:
            if (g.NT > kCvTiles<false>) k_conv_tc<128, true><<<grid, kCvThreads<true>, g.smem, s>>>(p);
            else k_conv_tc<128, false><<<grid, kCvThreads<false>, g.smem, s>>>(p);
            break;
        default: LZ_REQUIRE(false, LZ_EINVAL, "conv_tc: N must be 64 or 128");
    }
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

// Scores useful output rows (both convs) over issued MMA rows, which count conv1's halo recompute and the 128-row tile padding of
// both convs.  A band of ~200 KB leaves room for one CTA per SM, so there is no co-residency term as in the plain conv's picker;
// instead a conv of several tiles whose tile groups (rb_tiles) leave one tile on its own is marked down: that group runs its 9 taps
// on a single accumulator chain per warpgroup.
int resblock_tc_plan(ResBlockTc &p)
{
    const int H = p.in.H, W = p.in.W;
    auto lone_tile = [](int NT, int MT) {
        int ng, per;
        tile_groups(NT, MT, ng, per);
        return NT > 1 && NT - (ng - 1) * per == 1;
    };
    ResBlockTc q = p;
    double best = -1.0;
    for (int G = 1; G <= 4; ++G)
        for (int bh = (G > 1 ? H : 1); bh <= H; ++bh)
            for (int st = 2; st <= 4; st += 2) {
                q.G = G; q.band_h = bh; q.stages = st;
                const RbGeom g = rb_geom(q);
                if (g.smem > 227 * 1024 || g.nchunk > kRbChunks) continue;
                double score = (double)(2 * G * H * W) / ((double)g.nbands * (g.NT1 + g.NT2) * 128);
                score *= (st == 4) ? 1.0 : 0.97;
                const int MT = rb_tiles(p.in.C, g);
                if (lone_tile(g.NT1, MT)) score *= 0.9;
                if (lone_tile(g.NT2, MT)) score *= 0.9;
                if (score > best + 1e-9) { best = score; p.G = G; p.band_h = bh; p.stages = st; }
            }
    LZ_REQUIRE(best > 0.0, LZ_EINVAL, "resblock_tc: no band of a %dx%d, %d-channel block fits shared memory", H, W, p.in.C);
    return LZ_OK;
}

int resblock_tc_launch(const ResBlockTc &p, cudaStream_t s)
{
    const RbGeom g = rb_geom(p);
    LZ_REQUIRE(g.smem <= 227 * 1024 && g.nchunk <= kRbChunks, LZ_EINVAL, "resblock_tc: band needs %zu B shared memory", g.smem);
    LZ_REQUIRE(p.in.nphase == 1 && p.out.C == p.in.C, LZ_EINVAL, "resblock_tc: unsupported input / output layout");
    const int grid = (p.B + p.G - 1) / p.G * g.nbands;
    switch (p.in.C) {
        case 32: k_resblock_tc<32, false><<<grid, kCvThreads<false>, g.smem, s>>>(p); break;
        case 64:
            if (rb_wide(64, g)) k_resblock_tc<64, true><<<grid, kCvThreads<true>, g.smem, s>>>(p);
            else k_resblock_tc<64, false><<<grid, kCvThreads<false>, g.smem, s>>>(p);
            break;
        default: LZ_REQUIRE(false, LZ_EINVAL, "resblock_tc: channels must be 32 or 64");
    }
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

size_t conv_tc_packed_bytes(int cin, int ncols) { return (size_t)9 * 2 * (cin / 8) * ncols * 16; }

float conv_tc_pack(const float *w, int cin, int cout, int ncols, int col0, unsigned char *dst)
{
    float mx = 0.0f;
    for (size_t i = 0; i < (size_t)cout * cin * 9; ++i) mx = std::max(mx, fabsf(w[i]));
    const float scale = pow2_scale(mx);
    // tap block: [k-group ci / 8][ncols hi rows | ncols lo rows][ci % 8]: [B_hi | B_lo] of a k-group is one contiguous 2 x ncols-row operand
    const size_t tap_halves = (size_t)2 * (cin / 8) * ncols * 8, part_halves = (size_t)ncols * 8;
    __half *h = reinterpret_cast<__half *>(dst);
    for (int t = 0; t < 9; ++t)
        for (int co = 0; co < cout; ++co)
            for (int ci = 0; ci < cin; ++ci) {
                const size_t off = (size_t)t * tap_halves + ((size_t)(ci / 8) * 2 * ncols + col0 + co) * 8 + (ci % 8);
                split_hi_lo(w[((size_t)co * cin + ci) * 9 + t] * scale, h[off], h[off + part_halves]);
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

int tcl_to_nchw_launch(const Tcl &in, float *out, int B, cudaStream_t s)
{
    k_tcl_to_nchw<<<tcl_to_nchw_ctas(in, B), 256, 0, s>>>(in, out, B);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

int tcl_to_nchw_ctas(const Tcl &in, int B)
{
    const size_t n = (size_t)B * (in.C / 8) * in.H * in.W;
    return (int)std::min<size_t>((n + 255) / 256, kNumSMs * 32);
}

}  // namespace lz
