// net_tc.cu -- tensor-core (wgmma) path of the MuZero latent-grid networks for sm_90a.
//
// One CTA runs the WHOLE recurrent_inference (or the latent-grid tail of initial_inference) for up to 8 roots (6x6 grid; 4 on the
// 8x8 grid of 64-pixel observations, see TcGeo) -- and, in persistent
// mode, the whole num_simulations loop of their search (tree back-up + descent by one warp per tree, tree_persist.cuh): five 3x3
// convolutions, three 1x1 head convolutions and the heads' fully connected layers as wgmma with fp32 accumulators in registers;
// BatchNorm / residual / ReLU epilogues and the softmax expectation + inverse scalar transform on chip.  Activations never leave the SM.
//
// fp32 accuracy on fp16 tensor cores ("3xFP16"): every fp32 operand v is split v = hi + lo with hi = fp16(v), lo = fp16(v - hi) (22
// significant bits); D += A_hi*B_hi + A_hi*B_lo + A_lo*B_hi with fp32 accumulation drops only the 2^-22 lo*lo term.  The tap block of the
// weights stores B_hi and B_lo as 128 consecutive operand rows ([B_hi | B_lo]); each 3x3 k-step is three m64n64k16 wgmma into one
// accumulator.  Weights are pre-split on the host and pre-scaled by a power of two (exact; folded back into the BatchNorm scale) so
// their lo parts stay in fp16's normal range.  Mode 2 ("fast") issues only the hi*hi pass.
//
// Implicit GEMM without im2col: activations live in shared memory as [k-group of 8 channels][row][8 halves] (the wgmma K-major
// no-swizzle canonical layout with SBO = 128 B, so row r of the operand is at start + 16*r bytes).  Rows are the pixels of a 7-wide
// padded grid (49 rows per root, column 6 and row 6 zero; 9-wide, 81 rows on the 8x8 grid), so the input of output row m for tap
// (dy,dx) is row m + 7*dy + dx: each of the 9 taps is the SAME buffer addressed through a descriptor whose start address is shifted
// by (7*dy+dx)*16 bytes.  The zero pad
// rows double as the conv padding between rows and between consecutive roots.  The rows are cut into 128-row tiles; warpgroup g
// computes rows [64 g, 64 g + 64) of every tile and keeps all of a layer's accumulators in registers (3 tiles x 32 per thread) until
// every MMA of the layer has read the buffer; the epilogue then rewrites the buffer IN PLACE, one tile at a time through a 128-row
// fp32 staging array (one row per thread, as the epilogue is written).  The ResBlock skip tensors are parked in an L2-resident
// scratch (thread-private rows, .cg accesses).
//
// Warp roles (384 threads): warps 0-7 = two consumer warpgroups (MMA issue, epilogues, heads, trees; warp w's read-out rows are
// 32*(w%4).. of a tile, its columns the 32-column half w/4), warps 8-11 = the producer warpgroup, which gives its registers to the
// consumers (setmaxnreg); warp 8 lane 0 is the weight producer (cp.async.bulk global->shared ring, mbarrier complete_tx; every
// consumer warp releases a slot once its MMAs have read it).
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <type_traits>

#include "model.cuh"
#include "net_tc.cuh"
#include "tc_ptx.cuh"
#include "tree.cuh"
#include "tree_persist.cuh"

namespace lz {


// ---------------------------------------------------------------------------------------------- geometry
constexpr int kEpiWarps = 8, kEpiThreads = kEpiWarps * 32;   // two consumer warpgroups
constexpr int kTcThreads = kEpiThreads + 128;                // + the producer warpgroup (its warp 8 streams the weights)
constexpr int kMaxTiles = 3;                     // 384 output rows: 3 tiles of 128 (the register accumulator budget)
constexpr int kTapKgBytes = 128 * 16;            // one k-group (8 input channels) of a tap: 64 hi rows then 64 lo rows of 16 B
constexpr int kTapBytes = 8 * kTapKgBytes;       // one 3x3 tap, [kg 8][co: 64 hi | 64 lo][ci % 8]: 16384 B
constexpr int kStages = 3;                       // 16 KB ring stages: conv taps, then the heads' FC weight blocks
constexpr int kHeadWBytes = 3 * 2 * 16 * 64 * 2; // three 1x1 heads (hc <= 16), hi + lo: 12288 B
constexpr int kBnSmemBytes = kTcMaxLayers * 128 * 4;   // folded BatchNorm tables of the program's layers
constexpr int kStgLd = 68;                       // fp32 staging rows: 64 columns + 4 (conflict-free 16-byte row reads)
constexpr int kStgBytes = 128 * kStgLd * 4;      // one 128-row tile of accumulators: 34,816 B
// tree <-> network hand-off of the persistent search, per root slot of the CTA: leaf slot, action | value, reward, policy logits
// (the global copies are still written for the step-wise entry points; reading them back would cost an L2 round trip per use)
constexpr int kHoWords = 4 + 32;
// the tree of a warp (tree_persist.cuh) parked in shared memory while the warp does network work: 16 uniform words + 3 x 32
// per-lane words
constexpr int kTreeParkWords = 16 + 3 * 32;
constexpr int kHbHeadBytes = 4 * 16 * 16;        // FC2 B operand of one head: [4 k-groups][8 roots hi | 8 roots lo][16 B] = 1 KB
constexpr int kFc1StageBytes = 2 * 2 * 2 * 96 * 16;   // 12,288 B: only the 96 real rows (3 heads x 32 units) of the M = 128 operand are streamed

// The latent grid HW x HW (6 for 84 / 96-pixel observations, 8 for 64) fixes everything that depends on the pixel count.  Rows
// are the pixels of a padded (HW + 1)-wide grid, (HW + 1)^2 rows per root; the last HW + 2 rows of a root (pixel (HW - 1, HW) and
// grid row HW) are padding, so the output rows that hold pixels end at R (HW + 1)^2 - (HW + 2):
//   HW = 6: 8 roots -> 392 - 8 = 384 rows = 3 tiles; activation buffer (8 + 384 + 8) rows x 16 B x 16 planes = 102,400 B
//   HW = 8: 4 roots -> 324 - 10 = 314 rows -> 3 tiles (5 roots would need 4); (10 + 384 + 10) rows -> 103,424 B
// The taps read up to |pitch * dy + dx| <= HW + 2 rows beyond the tiles: the zeroed margins.
template <int HW>
struct TcGeo {
    static constexpr int kPix = HW * HW;                          // pixels per root (the P of a [64][P] latent)
    static constexpr int kPitch = HW + 1, kRowsPerRoot = kPitch * kPitch;
    static constexpr int kMaxRoots = HW == 6 ? 8 : 4;
    static constexpr int kRootsLog2 = HW == 6 ? 3 : 2;
    static constexpr int kMargin = kPitch + 1;
    static constexpr int kRowsAlloc = kMargin + kMaxTiles * 128 + kMargin;
    static constexpr int kPlaneBytes = kRowsAlloc * 16;          // one k-group (8 fp16 channels) of all rows
    static constexpr int kPartBytes = 8 * kPlaneBytes;           // 64 channels
    static constexpr int kActBytes = 2 * kPartBytes;             // hi + lo
    // heads (see the heads section): FC1 has 16 P inputs (head channels <= 16) = 2 P k-groups; its B operand holds, per k-group,
    // 4 kMaxRoots hi rows (row head * kMaxRoots + root, 3 heads + padding) then as many lo rows, +16 B to spread the banks:
    //   HW = 6: 72 k-groups x (64 rows + 1) x 16 B = 74,880 B, m64n64 MMAs
    //   HW = 8: 128 k-groups x (32 rows + 1) x 16 B = 67,584 B, m64n32 MMAs (the 8-root layout would take 133 KB)
    static constexpr int kFc1Kg = 2 * kPix;
    static constexpr int kFbN = 8 * kMaxRoots;                   // B operand rows = MMA N: hi + lo
    static constexpr int kFbKgBytes = kFbN * 16 + 16;
    static constexpr int kFbBytes = kFc1Kg * kFbKgBytes;         // overlays the activation buffer
    static constexpr int kFrBytes = 2 * kFc1Kg * kMaxRoots * 16; // reward features parked from their hook: [hi | lo][k-group][root][16 B]
    static constexpr int kFc1Stages = 16 * kPix / 32;            // 32 inputs per 12 KB stage (2 k-steps x (A_hi + A_lo))
    // FC2 accumulators, hi + lo added: [tile][128 outputs][8 root columns] fp32 over the dead FC1 operand (HW = 8 uses columns
    // 0-3).  lz_model_finalize takes heads of up to 608 outputs on this path (support and action space alike): 3 x 5 = 15 tiles
    static constexpr int kF2MaxTiles = HW == 6 ? 18 : 16;
    static constexpr int kSmemMain = kActBytes + kStages * kTapBytes + kHeadWBytes + 1024 + kBnSmemBytes + kStgBytes;
    static constexpr int kHeadScratch = kFrBytes + kEpiWarps * kTreeParkWords * 4;   // parked reward features + parked trees
    static constexpr int kHandoffBytes = kMaxRoots * kHoWords * 4;
    static constexpr int kSmemBytes = kSmemMain + kHeadScratch + kHandoffBytes;      // 231,552 B (HW = 6), 229,952 B (HW = 8)
    static_assert(kSmemBytes <= 227 * 1024, "k_net_tc exceeds the 227 KB of shared memory of a block");
    static_assert(kMaxRoots * kRowsPerRoot - (HW + 2) <= kMaxTiles * 128, "the roots of a CTA must fit the register tiles");
    static_assert(kF2MaxTiles * 128 * 8 * 4 <= kFbBytes, "FC2 staging must fit under the FC1 operand");
    static_assert(3 * ((608 + 127) / 128) <= kF2MaxTiles, "FC2 staging must hold the largest heads");
    static_assert(kFbBytes + 3 * kHbHeadBytes + 2 * 2 * 4 * 4 * 3 * 4 <= kActBytes, "the head scratch must fit the activation buffer");
};

struct TcBars {
    uint64_t full[kStages], empty[kStages];     // producer -> consumers (complete_tx) / consumer warps -> producer (8 arrivals)
};

// the consumer warpgroups' barrier (named barrier 1; the producer warp never joins it)
__device__ __forceinline__ void epi_sync() { asm volatile("bar.sync 1, %0;\n" ::"n"(kEpiThreads) : "memory"); }

// ---------------------------------------------------------------------------------------------- heads
// The fully connected parts of the heads (reward / value / policy: Linear(hc*36 -> hid) + BN + ReLU, Linear(hid -> K),
// muzero_model.py:465-502, common.py:1130-1187) run on the TENSOR CORES at the end of a simulation with the roles swapped: the
// weights are the M operand (streamed through the same 16 KB ring as the conv taps, fp16 hi/lo), the up to 8 roots are N columns:
//   FC1  D[(head, unit) 96 of 128 rows][(head, root) 32 columns] += W1^T[rows][K = 576 inputs] x F[K][columns]; only the diagonal
//        (head == head) blocks are read back (one MMA stream for all three heads, A-operand-bound);
//   FC2  per head and per 128-output tile: D[output k][root] = W2[k][K = 32 units] x H[units][root]: a thread of the read-out owns
//        output k = tile * 128 + 32 * (warp % 4) + lane for four roots -- exactly the distribution of the canonical softmax order
//        (net6.cuh), so the softmax expectation runs straight out of the staged accumulators, the 601 logits are never stored.
// Both products keep the fp32-accurate 3xFP16 scheme: A_hi x [B_hi | B_lo] and A_lo x [B_hi | B_lo] (the extra lo x lo term is
// harmless), the two column halves are added at read-out.  Warpgroup g computes rows [64 g, 64 g + 64) of each product.
// On the 8x8 grid (1,024 FC1 inputs, 4 roots per CTA) the FC1 B operand has 16 + 16 rows and FC1 is m64n32 (TcGeo<8>).

__device__ __forceinline__ void put_half(unsigned char *p, float v, float &rem)
{
    const __half h = __float2half_rn(fminf(v, 65504.0f));
    *reinterpret_cast<__half *>(p) = h;
    rem = v - __half2float(h);
}

// Row m of the CTA's padded pixel grid -> (root slot r in the CTA, pixel p); false for pad rows / absent roots.
template <int HW>
__device__ __forceinline__ bool row_decode(int R, int nvalid, int m, int &r, int &p)
{
    using G = TcGeo<HW>;
    const int rr = m / G::kRowsPerRoot, q = m - rr * G::kRowsPerRoot, y = q / G::kPitch, x = q - y * G::kPitch;
    r = rr;
    p = y * HW + x;
    return (rr < R) && (r < nvalid) && (y < HW) && (x < HW);
}

// Staged 1x1-conv accumulators of one tile (S columns [0,16) reward, [16,32) value, [32,48) policy) -> BatchNorm + ReLU -> fp16 hi/lo
// features in FC1's B-operand layout, for the heads in hmask (bit 0 reward -> its parking buffer fr, bit 1 value / bit 2 policy ->
// rows kMaxRoots + r / 2 kMaxRoots + r of fb).  Feature k = c * P + p of root r sits at k-group k / 8, row (head * kMaxRoots + r),
// element k % 8.  No barrier inside.
template <int HW>
__device__ __forceinline__ void head_scatter(const TcNet &net, int hmask, unsigned char *fr, unsigned char *fb, const float *S, int t,
                                             int R, int nvalid)
{
    using G = TcGeo<HW>;
    constexpr int kP = G::kPix, kRt = G::kMaxRoots, kLo = 4 * kRt * 16;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q4 = warp & 3, half = warp >> 2, rowid = q4 * 32 + lane;
    int r, p;
    const bool valid = row_decode<HW>(R, nvalid, t * 128 + rowid, r, p);
    if (!valid) return;
    const float *v = S + (size_t)rowid * kStgLd;
    // warps 0-3 scatter reward + value features, warps 4-7 policy features
    if (half == 0 && (hmask & 1)) {
        for (int c = 0; c < net.hc[0]; ++c) {
            const int k = c * kP + p;
            unsigned char *d = fr + ((k >> 3) * kRt + r) * 16 + (k & 7) * 2;
            float rem;
            put_half(d, fmaxf(fmaf(v[c], __ldg(net.head_bn + c), __ldg(net.head_bn + 16 + c)), 0.0f), rem);
            *reinterpret_cast<__half *>(d + G::kFrBytes / 2) = __float2half_rn(rem);
        }
    }
    if (half == 0 && (hmask & 2)) {
        for (int c = 0; c < net.hc[1]; ++c) {
            const int k = c * kP + p;
            unsigned char *d = fb + (k >> 3) * G::kFbKgBytes + (kRt + r) * 16 + (k & 7) * 2;
            float rem;
            put_half(d, fmaxf(fmaf(v[16 + c], __ldg(net.head_bn + 32 + c), __ldg(net.head_bn + 48 + c)), 0.0f), rem);
            *reinterpret_cast<__half *>(d + kLo) = __float2half_rn(rem);
        }
    }
    if (half == 1 && (hmask & 4)) {
        for (int c = 0; c < net.hc[2]; ++c) {
            const int k = c * kP + p;
            unsigned char *d = fb + (k >> 3) * G::kFbKgBytes + (2 * kRt + r) * 16 + (k & 7) * 2;
            float rem;
            put_half(d, fmaxf(fmaf(v[32 + c], __ldg(net.head_bn + 64 + c), __ldg(net.head_bn + 80 + c)), 0.0f), rem);
            *reinterpret_cast<__half *>(d + kLo) = __float2half_rn(rem);
        }
    }
}

// FC1 read-out (warps 0-2: staged rows 32 h + unit j of head h; columns h * kMaxRoots + root, lo parts 4 kMaxRoots further):
// BatchNorm + ReLU, then the hidden activations as FC2's B operand hb[head][k-group j / 8][root | 8 + root (lo)][j % 8].  Root
// columns past kMaxRoots (the 8x8 grid) get zeros.
template <int HW>
__device__ __forceinline__ void heads_hidden(const TcNet &net, int hmask, unsigned char *hb, const float *S)
{
    constexpr int kRt = TcGeo<HW>::kMaxRoots;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp >= 3 || !((hmask >> warp) & 1)) return;
    const int h = warp, j = lane;
    const Head &H = h == 0 ? net.reward : (h == 1 ? net.value : net.policy);
    const float *a = S + (size_t)(warp * 32 + lane) * kStgLd + h * kRt, *b = a + 4 * kRt;
    const float inv = net.fc[h].fc1_inv;
    const float s2 = (j < H.hid) ? __ldg(H.s2 + j) : 0.0f, t2 = (j < H.hid) ? __ldg(H.t2 + j) : 0.0f;
    unsigned char *dst = hb + h * kHbHeadBytes + (j >> 3) * 256 + (j & 7) * 2;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const float pre = r < kRt ? (a[r] + b[r]) * inv : 0.0f;
        const float hid = (r < kRt && j < H.hid) ? fmaxf(fmaf(pre, s2, t2), 0.0f) : 0.0f;
        float rem;
        put_half(dst + r * 16, hid, rem);
        *reinterpret_cast<__half *>(dst + (8 + r) * 16) = __float2half_rn(rem);
    }
}

// FC2 read-out: thread (g = root group of 4, wg = warp % 4, lane) owns output k = tile * 128 + wg * 32 + lane of roots
// 4 g .. 4 g + 3 (f2: the staged FC2 accumulators, hi + lo columns already added): logits = D / scale + bias; raw logits to global when asked for; the categorical heads fold them into the
// canonical one-pass softmax expectation (net6.cuh) and the inverse scalar transform.  Same arithmetic per (head, root) as
// categorical_to_scalar; the two categorical heads are reduced TOGETHER (their 8 max / 16 sum butterflies interleaved, two CTA
// barriers instead of six: the read-out is a latency chain, not a throughput problem).  red: 2 x 2 x 4 x 4 x 3 floats of scratch.
__device__ __forceinline__ void heads_outputs(const TcNet &net, const TcIO &io, int hmask, const float *f2, float *red, int nvalid, int root0,
                                              const float *b2_s, float *ho)
{
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = warp >> 2, wg = warp & 3;
    const int row = wg * 32 + lane;
    float m[2][4], sm[2][4], ws[2][4];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int q = 0; q < 4; ++q) { m[h][q] = -INFINITY; sm[h][q] = 0.0f; ws[h][q] = 0.0f; }
    int tile = 0, boff = 0;
    int hdone = 0;
#ifndef LZ_NO_JOINT_HEADS
    if ((hmask & 3) == 3 && net.reward.K == net.value.K && !io.reward_logits && !io.value_logits) {
        // the two categorical heads of the search (same support size, no raw logits wanted) in ONE loop: 8 independent softmax
        // recurrences per thread instead of 4 -- the read-out is a chain of dependent latencies, so this nearly halves it
        const int K = net.reward.K, nblk = (K + 127) >> 7;
        const float inv0 = net.fc[0].fc2_inv, inv1 = net.fc[1].fc2_inv;
        const float *b20 = b2_s ? b2_s : net.reward.b2, *b21 = b2_s ? b2_s + K : net.value.b2;
#pragma unroll 1
        for (int blk = 0; blk < nblk; ++blk) {
            const int k = blk * 128 + wg * 32 + lane;
            const float bias0 = (k < K) ? b20[k] : 0.0f, bias1 = (k < K) ? b21[k] : 0.0f;
            const float4 s0 = *reinterpret_cast<const float4 *>(f2 + ((size_t)blk * 128 + row) * 8 + g * 4);
            const float4 s1 = *reinterpret_cast<const float4 *>(f2 + ((size_t)(nblk + blk) * 128 + row) * 8 + g * 4);
            const float x0[4] = {s0.x, s0.y, s0.z, s0.w}, x1[4] = {s1.x, s1.y, s1.z, s1.w};
            if (k < K) {
                const float sup = support_at(net.support_min, net.support_step, k);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    if (g * 4 + q >= nvalid) continue;
                    softmax_push(m[0][q], sm[0][q], ws[0][q], fmaf(x0[q], inv0, bias0), sup);
                    softmax_push(m[1][q], sm[1][q], ws[1][q], fmaf(x1[q], inv1, bias1), sup);
                }
            }
        }
        tile = 2 * nblk; boff = 2 * K; hdone = 3;
    }
#endif
#pragma unroll
    for (int h = 0; h < 3; ++h) {
        if (!((hmask >> h) & 1) || ((hdone >> h) & 1)) continue;
        const Head &H = h == 0 ? net.reward : (h == 1 ? net.value : net.policy);
        const int K = H.K, nblk = (K + 127) >> 7;
        const float inv = net.fc[h].fc2_inv;
        float *glog = h == 0 ? io.reward_logits : (h == 1 ? io.value_logits : io.policy_logits);
        // FC2 bias: the copy staged in shared memory at kernel start (the evaluated heads back to back) or global
        const float *b2 = b2_s ? b2_s + boff : H.b2;
        boff += K;
#pragma unroll 1
        for (int blk = 0; blk < nblk; ++blk, ++tile) {      // rolled: the read-out is a long latency chain, its code must stay small
            const int k = blk * 128 + wg * 32 + lane;
            const float bias = (k < K) ? b2[k] : 0.0f;
            const float4 s0 = *reinterpret_cast<const float4 *>(f2 + ((size_t)tile * 128 + row) * 8 + g * 4);
            const float x[4] = {s0.x, s0.y, s0.z, s0.w};
            if (k < K) {
                const float sup = support_at(net.support_min, net.support_step, k);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int r = g * 4 + q;
                    if (r >= nvalid) continue;
                    const float o = fmaf(x[q], inv, bias);
                    if (glog) glog[(size_t)(root0 + r) * K + k] = o;
                    if (h == 2 && ho && k < 32) ho[r * kHoWords + 4 + k] = o;
                    if (h < 2) softmax_push(m[h & 1][q], sm[h & 1][q], ws[h & 1][q], o, sup);   // running softmax statistics (net6.cuh: the canonical order)
                }
            }
        }
    }
    // block-wide combine per (head, root): max, then rescaled sums (4 warps per root group); both heads at once
    float mg[2][4];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int q = 0; q < 4; ++q) mg[h][q] = m[h][q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int q = 0; q < 4; ++q) mg[h][q] = fmaxf(mg[h][q], __shfl_xor_sync(0xffffffffu, mg[h][q], o));
    auto red_at = [&](int h, int w4, int q) { return red + (((h * 2 + g) * 4 + w4) * 4 + q) * 3; };
    if (lane == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int q = 0; q < 4; ++q) red_at(h, wg, q)[0] = mg[h][q];
    }
    asm volatile("bar.sync 1, %0;\n" ::"n"(kEpiThreads) : "memory");
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            float M = red_at(h, 0, q)[0];
#pragma unroll
            for (int w4 = 1; w4 < 4; ++w4) M = fmaxf(M, red_at(h, w4, q)[0]);
            const float sc = (m[h][q] == -INFINITY) ? 0.0f : expf(m[h][q] - M);
            sm[h][q] *= sc;
            ws[h][q] *= sc;
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                sm[h][q] += __shfl_xor_sync(0xffffffffu, sm[h][q], o);
                ws[h][q] += __shfl_xor_sync(0xffffffffu, ws[h][q], o);
            }
    if (lane == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int q = 0; q < 4; ++q) { red_at(h, wg, q)[1] = sm[h][q]; red_at(h, wg, q)[2] = ws[h][q]; }
    }
    asm volatile("bar.sync 1, %0;\n" ::"n"(kEpiThreads) : "memory");
    if (wg == 0 && lane < 8) {
        const int h = lane >> 2, q = lane & 3, r = g * 4 + q;
        if (r < nvalid && ((hmask >> h) & 1)) {
            float S = 0.0f, W = 0.0f;
#pragma unroll
            for (int w4 = 0; w4 < 4; ++w4) { S += red_at(h, w4, q)[1]; W += red_at(h, w4, q)[2]; }
            const float v = inverse_scalar_transform(W / S);
            float *dst = h == 0 ? io.reward : io.value;
            if (dst) dst[root0 + r] = v;
            if (ho) ho[r * kHoWords + (h == 0 ? 3 : 2)] = v;
        }
    }
}

// ---------------------------------------------------------------------------------------------- kernel
// 32 consecutive channels [32*half, 32*half+32) of pixel p of one root latent of kP pixels.  cl: the kernel-internal layout
// [c / 4][kP][c % 4] (the pool slots this kernel writes in persistent mode, the skip scratch, the action-bias table): a thread's
// float4 j is at ((c0 / 4 + j) * kP + p) * 4, so the lanes of a warp (consecutive pixels) touch consecutive 16-byte chunks --
// coalesced 512-byte warp accesses (a plain channels-last row per lane costs 32 separate sectors per warp instruction).  Else NCHW
// [64][kP] (every tensor that crosses the API).
template <int kP>
__device__ __forceinline__ void load_row32(const float *root, bool cl, int p, int half, float (&v)[32])
{
    if (cl) {
        const float4 *src = reinterpret_cast<const float4 *>(root) + (half * 8) * kP + p;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            // L2-only (the pool / scratch are written by this launch, and allocating these once-read rows in L1 would compete with the
            // tensor core's operand fetch for the shared-memory / L1 data array: measured -1.4 % on the search)
            const float4 q = __ldcg(src + j * kP);
            v[4 * j] = q.x; v[4 * j + 1] = q.y; v[4 * j + 2] = q.z; v[4 * j + 3] = q.w;
        }
    } else {
        const float *src = root + (size_t)(half * 32) * kP + p;
#pragma unroll
        for (int c = 0; c < 32; ++c) v[c] = src[(size_t)c * kP];
    }
}

// 16 consecutive channels [c0, c0 + 16) of pixel p of one root (same layouts)
template <int kP>
__device__ __forceinline__ void store_row16(float *root, bool cl, int p, int c0, const float (&v)[16])
{
    if (cl) {
        float4 *dst = reinterpret_cast<float4 *>(root) + (c0 >> 2) * kP + p;
#pragma unroll
        for (int j = 0; j < 4; ++j) __stcg(dst + j * kP, make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]));
    } else {
        float *dst = root + (size_t)c0 * kP + p;
#pragma unroll
        for (int c = 0; c < 16; ++c) dst[(size_t)c * kP] = v[c];
    }
}

// park / unpark the tree of a warp (kTreeParkWords)
__device__ __forceinline__ void ptree_park(const PTree &T, uint32_t *w, int lane)
{
    if (lane == 0) {
        w[0] = (uint32_t)T.nl; w[1] = (uint32_t)T.plen; w[2] = (uint32_t)T.vtp; w[3] = __float_as_uint(T.mmax); w[4] = __float_as_uint(T.mmin);
        w[5] = (uint32_t)T.root_visit; w[6] = __float_as_uint(T.root_vsum); w[7] = __float_as_uint(T.root_reward);
        w[8] = (uint32_t)T.root_to_play; w[9] = (uint32_t)T.tp0; w[10] = (uint32_t)T.players;
    }
    w[16 + lane] = (uint32_t)T.my_legal; w[48 + lane] = (uint32_t)T.my_pslot; w[80 + lane] = (uint32_t)T.my_pact;
    __syncwarp();
}
__device__ __forceinline__ void ptree_unpark(PTree &T, const uint32_t *w, int lane)
{
    T.nl = (int)w[0]; T.plen = (int)w[1]; T.vtp = (int)w[2]; T.mmax = __uint_as_float(w[3]); T.mmin = __uint_as_float(w[4]);
    T.root_visit = (int)w[5]; T.root_vsum = __uint_as_float(w[6]); T.root_reward = __uint_as_float(w[7]);
    T.root_to_play = (int)w[8]; T.tp0 = (int)w[9]; T.players = (int)w[10];
    T.my_legal = (int)w[16 + lane]; T.my_pslot = (int)w[48 + lane]; T.my_pact = (int)w[80 + lane];
}

// One CTA per SM (~225 KB of shared memory).  Its 12 warps are launched with 168 registers each (three per register-file quarter of
// 16,384); the producer warpgroup drops to kProducerRegs and the consumer warpgroups rise to kConsumerRegs (tc_ptx.cuh), so the
// tree, epilogue and head code keeps its state in registers (at 168 for every thread, ptxas spilled some of it).
// HW: the latent grid (TcGeo); one instantiation per grid, chosen by tc_launch from TcNet::hw.
template <int HW>
__global__ void __launch_bounds__(kTcThreads, 1) k_net_tc(TcNet net, TcIO io, TreeParams tp)
{
    using G = TcGeo<HW>;
    constexpr int kP = G::kPix, kPitch = G::kPitch, kRowsPerRoot = G::kRowsPerRoot, kMargin = G::kMargin;
    constexpr int kPlaneBytes = G::kPlaneBytes, kPartBytes = G::kPartBytes, kActBytes = G::kActBytes;
    constexpr int kSmemMain = G::kSmemMain, kHeadScratch = G::kHeadScratch, kFrBytes = G::kFrBytes;
    constexpr int kRt = G::kMaxRoots, kFbKgBytes = G::kFbKgBytes, kFbBytes = G::kFbBytes;
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char *act = smem;                                   // [2 parts][8 planes][400 rows][16 B]
    unsigned char *ring = smem + kActBytes;                      // [kStages][8 k-groups][128 rows: 64 hi | 64 lo][16 B]
    unsigned char *headw = ring + kStages * kTapBytes;           // [3 heads][hi 2 KB | lo 2 KB]
    TcBars *bars = reinterpret_cast<TcBars *>(headw + kHeadWBytes);
    float *bn_s = reinterpret_cast<float *>(headw + kHeadWBytes + 1024);   // [nlayers][scale 64 | shift 64]
    float *stg = reinterpret_cast<float *>(headw + kHeadWBytes + 1024 + kBnSmemBytes);   // [128 rows][kStgLd] accumulator staging

    // warp index as a warp-UNIFORM value (shuffle broadcast): the role branches below become uniform branches
    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const int R = io.roots_per_cta;
    const int root0 = blockIdx.x * R;
    const int nvalid = min(R, io.B - root0);                     // roots of this CTA that exist
    const int NT = (R * kRowsPerRoot - (HW + 2) + 127) >> 7;
    const int npass = io.npass;
    const int nlayers = net.nlayers;
    const int nsims = io.nsims > 0 ? io.nsims : 1;     // > 1 (or persistent): the whole search loop runs inside this launch
    const bool persistent = io.persistent != 0;

    // ---- one-time setup ----
    if (tid == 0) {
        for (int i = 0; i < kStages; ++i) { mbar_init(&bars->full[i], 1); mbar_init(&bars->empty[i], kEpiWarps); }
        fence_mbar_init();
    }
    // heads whose fully connected parts run in this kernel (EfficientZero: the reward features go to the LSTM kernels instead),
    // streamed through the ring per simulation after the conv taps: FC1 of all heads as one [128 rows][16 P] operand (16 P / 32
    // stages of 2 k-steps), then one stage per 128-output tile of each head's FC2
    const int hmask_fc = ((net.has_reward && !io.ez_feat) ? 1 : 0) | 6;
    // 1x1 head weights (12 KB) and the folded BatchNorm tables of this program's layers: plain copies
    for (int i = tid; i < kHeadWBytes / 16; i += kTcThreads)
        reinterpret_cast<uint4 *>(headw)[i] = __ldg(reinterpret_cast<const uint4 *>(net.headw) + i);
    for (int i = tid; i < nlayers * 128; i += kTcThreads)
        bn_s[i] = __ldg(net.bn + (size_t)net.layer_w[i >> 7] * 128 + (i & 127));
    // persistent search: the exploration-rate table of the PUCT rule next to them when it fits (else it is read from global)
    const bool fast_tree = persistent;      // tree_persist.cuh (A <= 32, checked by tc_launch; larger action spaces use the multi-launch graph)
    const float *pbc_tab = tp.pbc;
    if (fast_tree && (nlayers * 128 + tp.N + 1) * 4 <= kBnSmemBytes) {
        float *pbc_s = bn_s + nlayers * 128;
        for (int i = tid; i <= tp.N; i += kTcThreads) pbc_s[i] = tp.pbc[i];
        pbc_tab = pbc_s;
    }
    // the FC2 bias vectors of the heads this kernel evaluates, back to back behind them when they fit as well
    const float *b2_s = nullptr;
    {
        int nb2 = 0;
        for (int h = 0; h < 3; ++h)
            if ((hmask_fc >> h) & 1) nb2 += net.fc[h].K;
        const int used = nlayers * 128 + ((pbc_tab != tp.pbc) ? tp.N + 1 : 0);
        if ((used + nb2) * 4 <= kBnSmemBytes) {
            float *dst = bn_s + used;
            int off = 0;
            for (int h = 0; h < 3; ++h) {
                if (!((hmask_fc >> h) & 1)) continue;
                const Head &H = h == 0 ? net.reward : (h == 1 ? net.value : net.policy);
                for (int i = tid; i < H.K; i += kTcThreads) dst[off + i] = __ldg(H.b2 + i);
                off += H.K;
            }
            b2_s = dst;
        }
    }
    float *ho = reinterpret_cast<float *>(smem + kSmemMain + kHeadScratch);      // tree <-> network hand-off (persistent search)
    fence_proxy_async();
    __syncthreads();

    if (warp >= kEpiWarps) {
        // ================= weight producer =================
        wg_reg_dealloc<kProducerRegs>();
        if (warp == kEpiWarps && (tid & 31) == 0) {
            uint32_t n = 0;
            auto stage_in = [&](const unsigned char *src, uint32_t bytes = kTapBytes) {      // every stage is released by all consumer warps
                const int st = n % kStages;
                if (n >= (uint32_t)kStages) mbar_wait(&bars->empty[st], ((n / kStages) - 1) & 1);
                mbar_expect_tx(&bars->full[st], bytes);
                bulk_g2s(ring + st * kTapBytes, src, bytes, &bars->full[st]);
                ++n;
            };
            for (int sim = 0; sim < nsims; ++sim) {     // runs ahead of the consumers: the next simulation's first taps are
                for (int L = 0; L < nlayers; ++L) {     // already in the ring while the tree work is going on
                    const unsigned char *src = net.convw + (size_t)net.layer_w[L] * (9 * kTapBytes);
                    for (int tap = 0; tap < 9; ++tap) stage_in(src + (size_t)tap * kTapBytes);
                }
                // the heads: FC1 weights of all heads, then the FC2 tiles of every head this kernel evaluates
                for (int i = 0; i < G::kFc1Stages; ++i) stage_in(net.fcw + (size_t)i * kFc1StageBytes, kFc1StageBytes);
                for (int h = 0; h < 3; ++h) {
                    if (!((hmask_fc >> h) & 1)) continue;
                    const int nblk = (net.fc[h].K + 127) >> 7;
                    for (int blk = 0; blk < nblk; ++blk) stage_in(net.fcw + net.fc[h].fc2_off + (size_t)blk * kTapBytes);
                }
            }
        }
        return;
    }

    // ================= consumer warpgroups: warpgroup wg issues the MMAs of rows [64 wg, 64 wg + 64) of every tile; for the
    // read-outs warp w owns staged rows 32*(w%4).. and the 32-column half w/4 =================
    wg_reg_alloc<kConsumerRegs>();
    const int lane = lane_id();          // read after the reallocation: a value live across it is kept in local memory by ptxas
    const int wg = warp >> 2;
    const int q4 = warp & 3, half = warp >> 2, rowid = q4 * 32 + lane;
    const uint32_t act_s = smem_u32(act), ring_s = smem_u32(ring), headw_s = smem_u32(headw);
    const uint32_t a_lbo = kPlaneBytes >> 4;
    const uint64_t a_desc0 = make_desc(act_s + (kMargin + wg * 64) * 16, a_lbo, 8);   // this warpgroup's row 0, hi part, k-step 0
    const uint64_t b_desc0 = make_desc(ring_s, kTapKgBytes >> 4, 8);                  // stage 0, k-group 0: rows 0-63 hi, 64-127 lo
    uint32_t n = 0;                 // position in the weight stream (the producer's sequence)
    auto ring_wait = [&](uint32_t pos) { mbar_wait(&bars->full[pos % kStages], (pos / kStages) & 1); };
    auto ring_release = [&](uint32_t pos) {       // this warp's MMAs reading the slot have completed
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars->empty[pos % kStages]);
    };
    unsigned char *fr = smem + kSmemMain;      // reward features (fp16 hi / lo, FC1's B-operand rows 0-7), parked from their hook
    unsigned long long *dbg = (io.dbg && blockIdx.x == 0 && tid == 0) ? io.dbg : nullptr;
    if (dbg) dbg[0] = clock64();
    // this warp's tree (tree_persist.cuh): its scalars / first path entries live in registers during the tree phase and are
    // parked in shared memory while the warp does network work
    uint32_t *tree_park = reinterpret_cast<uint32_t *>(smem + kSmemMain + kFrBytes) + warp * kTreeParkWords;
    if (fast_tree && warp < nvalid) {
        PTree T;
        ptree_init(tp, T, root0 + warp, lane);
        ptree_park(T, tree_park, lane);
    }
    // row bookkeeping of this thread (simulation-invariant): per tile (root slot in the CTA) << 8 | pixel, or -1 for pad rows
    int rowc[kMaxTiles];
#pragma unroll
    for (int t = 0; t < kMaxTiles; ++t) {
        int r, p;
        const bool valid = row_decode<HW>(R, nvalid, t * 128 + rowid, r, p) && (t < NT);
        rowc[t] = valid ? ((r << 8) | p) : -1;
    }
    for (int sim = 0; sim <= nsims; ++sim) {        // iteration nsims: only the back-up of the last simulation (mcts_ctree.py:365-368)
        if (sim == nsims && !persistent) break;
        if (dbg && sim < nsims) dbg[50] = clock64();
        if (persistent) {
            // ---- tree phase: one warp per root of this CTA (roots never interact, so the whole search of these roots
            // lives in this CTA): back up the previous simulation, then descend to the next leaf.  cnode.cpp:480-500,754-825
            if (warp < nvalid) {
                const int b = root0 + warp;
                PTree T;
                ptree_unpark(T, tree_park, lane);
                float *my_ho = ho + warp * kHoWords;
                if (sim > 0)       // network outputs of the previous simulation: from the hand-off (written by this CTA's read-out)
                    ptree_backprop(tp, T, b, lane, io.sim0 + sim, my_ho[3], my_ho[2], my_ho + 4);
                if (dbg && sim < nsims) dbg[56] = clock64();
                if (sim < nsims) {
                    ptree_traverse(tp, T, b, lane, io.deterministic, (unsigned)(io.sim0 + sim), pbc_tab, io.ix_rw, io.action_rw,
                                   reinterpret_cast<int *>(my_ho), reinterpret_cast<int *>(my_ho) + 1);
                    ptree_park(T, tree_park, lane);
                }
            }
            if (sim == nsims) break;
            __threadfence_block();
            epi_sync();
        }
        if (dbg) dbg[51] = clock64();
        float *latent_out = persistent ? (io.latent_pool_rw + (size_t)(io.sim0 + sim + 1) * io.slot_stride) : io.latent_out;
        // zero the margins (the head scratch of the previous simulation overlays them; pad rows inside the tiles are
        // rewritten as zeros by every load / epilogue)
        for (int i = tid; i < 2 * 8 * 2 * kMargin; i += kEpiThreads) {
            int part = i / (8 * 2 * kMargin), rem = i % (8 * 2 * kMargin), plane = rem / (2 * kMargin), r = rem % (2 * kMargin);
            int row = r < kMargin ? r : kMargin + kMaxTiles * 128 + (r - kMargin);
            *reinterpret_cast<uint4 *>(act + part * kPartBytes + plane * kPlaneBytes + row * 16) = make_uint4(0, 0, 0, 0);
        }
        // the pool slot holding the input latent of each of this thread's rows (tree -> network hand-off)
        int slot[kMaxTiles];
#pragma unroll
        for (int t = 0; t < kMaxTiles; ++t)
            slot[t] = rowc[t] < 0 ? 0 : (persistent ? reinterpret_cast<const int *>(ho)[(rowc[t] >> 8) * kHoWords] : (io.ix ? io.ix[root0 + (rowc[t] >> 8)] : 0));
        auto in_ptr = [&](int t) { return io.latent_base + (size_t)slot[t] * io.slot_stride + (size_t)(root0 + (rowc[t] >> 8)) * (kC * kP); };
        auto in_is_cl = [&](int t) { return io.pool_cl != 0 && slot[t] > 0; };      // slot 0: root latents as the API delivered them (NCHW)
        // ---- load the input activation: gather the latents, split to fp16 hi/lo ----
#pragma unroll
        for (int t = 0; t < kMaxTiles; ++t) {
            if (t >= NT) continue;
            float va[32];
            if (rowc[t] >= 0) load_row32<kP>(in_ptr(t), in_is_cl(t), rowc[t] & 255, half, va);
            else {
#pragma unroll
                for (int c = 0; c < 32; ++c) va[c] = 0.0f;
            }
            const int m = t * 128 + rowid;
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                unsigned char *p = act + (half * 4 + g) * kPlaneBytes + (kMargin + m) * 16;
                store_split8(p, p + kPartBytes, va + 8 * g);
            }
        }
        fence_proxy_async();          // generic-proxy writes -> the MMAs' operand reads
        epi_sync();
        if (dbg) dbg[1] = clock64();

        bool skip_in_scratch = false;      // the residual operand: the input latent until a layer has parked its output
        for (int L = 0; L < nlayers; ++L) {
            const int flags = net.layer_flags[L];
            // ---- the layer's MMAs: 9 taps x 4 k-steps x npass wgmma per tile, all tiles' accumulators in registers
            float acc[kMaxTiles][32];
#pragma unroll
            for (int t = 0; t < kMaxTiles; ++t)
#pragma unroll
                for (int i = 0; i < 32; ++i) acc[t][i] = 0.0f;
#pragma unroll
            for (int t = 0; t < kMaxTiles; ++t) wg_fence_acc(acc[t]);
            const uint32_t kA = (2 * kPlaneBytes) >> 4, kB = (2 * kTapKgBytes) >> 4, kLo = kPartBytes >> 4, kBLo = (64 * 16) >> 4;
            for (int tap = 0; tap < 9; ++tap) {
                const uint32_t pos = n++;
                ring_wait(pos);
                const int shift = (tap / 3 - 1) * kPitch + (tap % 3 - 1);
                const uint64_t b0 = b_desc0 + (uint64_t)(((pos % kStages) * kTapBytes) >> 4);
                // straight-line issue blocks: all three tiles (rows past the loaded ones are never read back) and the pass count
                // hoisted out, so that no branch separates the wgmma of a commit group (ptxas would serialise them)
                wg_fence();
                if (npass == 3) {
#pragma unroll
                    for (int t = 0; t < kMaxTiles; ++t)
#pragma unroll
                        for (int ks = 0; ks < 4; ++ks) {
                            const uint64_t a0 = a_desc0 + (uint64_t)(t * 128 + shift) + ks * kA;
                            wgmma_n64(acc[t], a0, b0 + ks * kB);
                            wgmma_n64(acc[t], a0, b0 + kBLo + ks * kB);
                            wgmma_n64(acc[t], a0 + kLo, b0 + ks * kB);
                        }
                } else {
#pragma unroll
                    for (int t = 0; t < kMaxTiles; ++t)
#pragma unroll
                        for (int ks = 0; ks < 4; ++ks)
                            wgmma_n64(acc[t], a_desc0 + (uint64_t)(t * 128 + shift) + ks * kA, b0 + ks * kB);
                }
                wg_commit();
                if (tap > 0) {
                    wg_wait<1>();
                    ring_release(pos - 1);
                }
            }
            wg_wait<0>();
#pragma unroll
            for (int t = 0; t < kMaxTiles; ++t) wg_fence_acc(acc[t]);
            ring_release(n - 1);
            epi_sync();                                   // every MMA of the layer has read the buffer: it may be rewritten
            if (dbg) dbg[2 + 2 * L] = clock64();
            // ---- epilogue, one tile at a time through the staging rows: BN (+ residual / action bias) + ReLU -> the buffer in place
            const float4 *bn4 = reinterpret_cast<const float4 *>(bn_s + L * 128 + half * 32);   // scale; shift 16 float4 further
            const bool park = (flags & LF_STORE_RES) && (L + 1 < nlayers);
            const bool has_res = (flags & LF_RES) != 0, has_ab = (flags & LF_ACT_BIAS) != 0;
#pragma unroll
            for (int t = 0; t < kMaxTiles; ++t) {
                if (t >= NT) continue;
                wg_stage<64>(stg, kStgLd, wg * 64, 0, acc[t]);
                epi_sync();
                const int m = t * 128 + rowid;
                const bool valid = rowc[t] >= 0;
                const int p = rowc[t] & 255, b = root0 + (rowc[t] >> 8);
                // residual operand (skip + action bias, in that association): thread-private global rows (L2-resident)
                float rs[32];
                if (has_res && valid) {
                    if (skip_in_scratch) load_row32<kP>(io.skip_scratch + (size_t)b * (kC * kP), true, p, half, rs);
                    else load_row32<kP>(in_ptr(t), in_is_cl(t), p, half, rs);
                    if (has_ab) {
                        const int action_raw = persistent ? reinterpret_cast<const int *>(ho)[(rowc[t] >> 8) * kHoWords + 1] : io.action[b];
                        const int action = min(max(action_raw, 0), net.A - 1);
                        const float4 *ab = reinterpret_cast<const float4 *>(net.abias) + ((size_t)action * 16 + half * 8) * kP + p;
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const float4 q = __ldcg(ab + j * kP);      // action-bias table (A x 9 KB on 6x6, A x 16 KB on 8x8), one row per (root, action): L2-only like the skip rows
                            rs[4 * j] += q.x; rs[4 * j + 1] += q.y; rs[4 * j + 2] += q.z; rs[4 * j + 3] += q.w;
                        }
                    }
                }
                // the thread's 32 channels in two halves of 16
#pragma unroll
                for (int hs = 0; hs < 2; ++hs) {
                    float v[16];
                    const float4 *srow = reinterpret_cast<const float4 *>(stg + (size_t)rowid * kStgLd + half * 32 + hs * 16);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float4 q = srow[j];
                        v[4 * j] = q.x; v[4 * j + 1] = q.y; v[4 * j + 2] = q.z; v[4 * j + 3] = q.w;
                    }
                    if (valid) {
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const float4 sc = bn4[hs * 4 + j], sh = bn4[16 + hs * 4 + j];
                            v[4 * j] = fmaf(v[4 * j], sc.x, sh.x); v[4 * j + 1] = fmaf(v[4 * j + 1], sc.y, sh.y);
                            v[4 * j + 2] = fmaf(v[4 * j + 2], sc.z, sh.z); v[4 * j + 3] = fmaf(v[4 * j + 3], sc.w, sh.w);
                        }
                        if (has_res) {
#pragma unroll
                            for (int c = 0; c < 16; ++c) v[c] += rs[hs * 16 + c];
                        }
#pragma unroll
                        for (int c = 0; c < 16; ++c) v[c] = fmaxf(v[c], 0.0f);       // every layer of these programs ends in ReLU
                        if (park) store_row16<kP>(io.skip_scratch + (size_t)b * (kC * kP), true, p, half * 32 + hs * 16, v);
                        if (flags & LF_WRITE_LATENT) {
                            if (latent_out) store_row16<kP>(latent_out + (size_t)b * (kC * kP), io.pool_cl != 0, p, half * 32 + hs * 16, v);
                            if (io.latent_out2) store_row16<kP>(io.latent_out2 + (size_t)b * (kC * kP), false, p, half * 32 + hs * 16, v);
                        }
                    } else {
#pragma unroll
                        for (int c = 0; c < 16; ++c) v[c] = 0.0f;          // pad rows / absent roots: the conv padding of the next layer
                    }
#pragma unroll
                    for (int g = 0; g < 2; ++g) {
                        unsigned char *pp = act + (half * 4 + hs * 2 + g) * kPlaneBytes + (kMargin + m) * 16;
                        store_split8_pos(pp, pp + kPartBytes, v + 8 * g);
                    }
                }
                epi_sync();                               // the staging rows are refilled by the next tile
            }
            if (park) skip_in_scratch = true;
            fence_proxy_async();
            epi_sync();                                   // the layer's output is visible to the next MMAs
            if (dbg) dbg[3 + 2 * L] = clock64();

            // ---- 1x1 head convolutions on this layer's output (reward hook: dynamics output; value / policy hook: the last layer)
            const bool hook_rew = (flags & LF_HOOK_REWARD) && net.has_reward, hook_vp = (flags & LF_HOOK_VALPOL) != 0;
            if (hook_rew || hook_vp) {
                float hr[kMaxTiles][8], hv[kMaxTiles][16];
#pragma unroll
                for (int t = 0; t < kMaxTiles; ++t) {
#pragma unroll
                    for (int i = 0; i < 8; ++i) hr[t][i] = 0.0f;
#pragma unroll
                    for (int i = 0; i < 16; ++i) hv[t][i] = 0.0f;
                    wg_fence_acc(hr[t]);
                    wg_fence_acc(hv[t]);
                }
                // straight-line issue blocks, as in the 3x3 loop: all three tiles (rows past the loaded ones are never read back), the
                // heads and the pass count hoisted out, so that no branch separates the wgmma of the commit group
                auto hook_mma = [&](auto rew, auto vp, auto np) {
#pragma unroll
                    for (int t = 0; t < kMaxTiles; ++t) {
                        const uint32_t arow = act_s + (uint32_t)(kMargin + t * 128 + wg * 64) * 16u;
#pragma unroll
                        for (int ps = 0; ps < decltype(np)::value; ++ps) {
                            const uint32_t apart = (ps == 2) ? kPartBytes : 0;
#pragma unroll
                            for (int ks = 0; ks < 4; ++ks) {
                                const uint64_t ad = make_desc(arow + apart + ks * 2 * kPlaneBytes, a_lbo, 8);
                                if constexpr (decltype(rew)::value)      // reward head: N = 16, [kg][16 co][8]
                                    wgmma_n16(hr[t], ad, make_desc(headw_s + ((ps == 1) ? 2048 : 0) + ks * 512, 16, 8));
                                if constexpr (decltype(vp)::value)       // value + policy heads as one N = 32 matrix, [kg][32 co][8]
                                    wgmma_n32(hv[t], ad, make_desc(headw_s + 4096 + ((ps == 1) ? 4096 : 0) + ks * 1024, 32, 8));
                            }
                        }
                    }
                };
                auto hook_heads = [&](auto np) {
                    if (hook_rew && hook_vp) hook_mma(std::true_type(), std::true_type(), np);
                    else if (hook_rew) hook_mma(std::true_type(), std::false_type(), np);
                    else hook_mma(std::false_type(), std::true_type(), np);
                };
                wg_fence();
                if (npass == 3) hook_heads(std::integral_constant<int, 3>());
                else hook_heads(std::integral_constant<int, 1>());
                wg_commit();
                wg_wait<0>();
#pragma unroll
                for (int t = 0; t < kMaxTiles; ++t) { wg_fence_acc(hr[t]); wg_fence_acc(hv[t]); }
                epi_sync();              // all reads of the buffer are complete: the value / policy features overlay it (fb)
                const int hm = (hook_rew ? 1 : 0) | (hook_vp ? 6 : 0);
#pragma unroll
                for (int t = 0; t < kMaxTiles; ++t) {
                    if (t >= NT) continue;
                    if (hook_rew) wg_stage<16>(stg, kStgLd, wg * 64, 0, hr[t]);
                    if (hook_vp) wg_stage<32>(stg, kStgLd, wg * 64, 16, hv[t]);
                    epi_sync();
                    if (hook_rew && io.ez_feat) {
                        // EfficientZero (efficientzero_model.py:556-562): the features are the input of the LSTM that the next kernel
                        // evaluates as one batched GEMM over all roots (ez.cu)
                        if (half == 0 && rowc[t] >= 0) {
                            const int nin = net.hc[0] * kP;
                            const float *v = stg + (size_t)rowid * kStgLd;
                            for (int c = 0; c < net.hc[0]; ++c)
                                io.ez_feat[(size_t)(root0 + (rowc[t] >> 8)) * nin + c * kP + (rowc[t] & 255)] =
                                    fmaxf(fmaf(v[c], __ldg(net.head_bn + c), __ldg(net.head_bn + 16 + c)), 0.0f);
                        }
                        head_scatter<HW>(net, hm & 6, fr, act, stg, t, R, nvalid);
                    } else {
                        head_scatter<HW>(net, hm, fr, act, stg, t, R, nvalid);
                    }
                    epi_sync();
                }
            }
        }
        if (dbg) dbg[24] = clock64();

        // ---- heads: FC1 -> FC2 -> softmax expectation -> h^-1 for all heads with the weights streamed through the ring.  The
        // scratch overlays the activation buffer (every conv MMA of this simulation has completed)
        {
            unsigned char *fb = act, *hb = act + kFbBytes;
            float *red = reinterpret_cast<float *>(hb + 3 * kHbHeadBytes);
            float *f2 = reinterpret_cast<float *>(act);           // FC2 accumulators [tile][128][8], over the dead FC1 operand
            // the parked reward features become rows 0..kMaxRoots-1 (hi) / 4 kMaxRoots.. (lo) of the B operand.  FC1 multiplies all
            // 16 P inputs of every head: the host packs zero weights past hc * P, but 0 x an Inf / NaN bit pattern that an earlier
            // simulation (the FC2 staging overlays these rows) or kernel left there is NaN, so a head of hc < 16 channels gets zeros there
            for (int h = 0; h < 3; ++h) {
                const int nin = net.hc[h] * kP;
                if (!((hmask_fc >> h) & 1) || (h > 0 && nin == 16 * kP)) continue;
                for (int i = tid; i < 2 * G::kFc1Kg * kRt; i += kEpiThreads) {
                    const int part = i / (G::kFc1Kg * kRt), rem = i - part * (G::kFc1Kg * kRt), kg = rem >> G::kRootsLog2, r = rem & (kRt - 1);
                    unsigned char *dst = fb + kg * kFbKgBytes + (part * 4 * kRt + h * kRt + r) * 16;
                    const int keep = nin - kg * 8;                // inputs of this k-group that exist
                    if (h > 0 && keep >= 8) continue;
                    uint4 q = make_uint4(0, 0, 0, 0);
                    if (keep > 0) {
                        q = *reinterpret_cast<const uint4 *>(h == 0 ? fr + part * (kFrBytes / 2) + (kg * kRt + r) * 16 : dst);
                        if (keep < 8) {                           // hc * 36 = 4 (mod 8) for odd hc: keep the first 4 halves
                            q.z = 0; q.w = 0;
                        }
                    }
                    *reinterpret_cast<uint4 *>(dst) = q;
                }
            }
            fence_proxy_async();
            epi_sync();                                           // FC1 may start
            if (dbg) dbg[44] = clock64();
            const uint32_t fb_s = act_s, hb_s = act_s + kFbBytes;
            {
                float f1[G::kFbN / 2];
#pragma unroll
                for (int i = 0; i < G::kFbN / 2; ++i) f1[i] = 0.0f;
                wg_fence_acc(f1);
                for (int i = 0; i < G::kFc1Stages; ++i) {
                    const uint32_t pos = n++;
                    ring_wait(pos);
                    const uint32_t st_s = ring_s + (pos % kStages) * kTapBytes;
                    wg_fence();
#pragma unroll
                    for (int ksi = 0; ksi < 2; ++ksi) {
                        const int kstep = 2 * i + ksi;
                        // [k-step][hi 3 KB | lo 3 KB], [kg 2][96 rows][8]: rows 96-127 of warpgroup 1's M = 64 operand are whatever follows
                        // in the slot (their accumulator rows are never read)
                        const uint64_t a_hi = make_desc(st_s + ksi * (kFc1StageBytes / 2) + wg * 64 * 16, 1536 >> 4, 8), a_lo = a_hi + (3072 >> 4);
                        const uint64_t b = make_desc(fb_s + kstep * 2 * kFbKgBytes, kFbKgBytes >> 4, 8);
                        if constexpr (G::kFbN == 64) {
                            wgmma_n64(f1, a_hi, b);
                            wgmma_n64(f1, a_lo, b);
                        } else {
                            wgmma_n32(f1, a_hi, b);
                            wgmma_n32(f1, a_lo, b);
                        }
                    }
                    wg_commit();
                    if (i > 0) {
                        wg_wait<1>();
                        ring_release(pos - 1);
                    }
                }
                wg_wait<0>();
                wg_fence_acc(f1);
                ring_release(n - 1);
                wg_stage<G::kFbN>(stg, kStgLd, wg * 64, 0, f1);
            }
            epi_sync();
            if (dbg) dbg[45] = clock64();
            heads_hidden<HW>(net, hmask_fc, hb, stg);
            fence_proxy_async();
            epi_sync();                                           // FC2 may start
            if (dbg) dbg[46] = clock64();
            int tile = 0;
            for (int h = 0; h < 3; ++h) {
                if (!((hmask_fc >> h) & 1)) continue;
                const int nblk = (net.fc[h].K + 127) >> 7;
                for (int blk = 0; blk < nblk; ++blk, ++tile) {
                    const uint32_t pos = n++;
                    ring_wait(pos);
                    const uint32_t st_s = ring_s + (pos % kStages) * kTapBytes;
                    float d[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) d[i] = 0.0f;
                    wg_fence_acc(d);
                    wg_fence();
#pragma unroll
                    for (int ks = 0; ks < 2; ++ks) {
                        const uint64_t a_hi = make_desc(st_s + ks * 2 * 2048 + wg * 64 * 16, 2048 >> 4, 8), a_lo = a_hi + (8192 >> 4);
                        const uint64_t b = make_desc(hb_s + h * kHbHeadBytes + ks * 2 * 256, 256 >> 4, 8);
                        wgmma_n16(d, a_hi, b);
                        wgmma_n16(d, a_lo, b);
                    }
                    wg_commit();
                    wg_wait<0>();
                    wg_fence_acc(d);
                    ring_release(pos);
                    // columns [0,8) = roots (hi part of H), [8,16) = the same roots (lo part): added here
                    const int r0 = wg * 64 + 16 * q4 + (lane >> 2), c = 2 * (lane & 3);
                    float *o = f2 + ((size_t)tile * 128 + r0) * 8 + c;
                    *reinterpret_cast<float2 *>(o) = make_float2(d[0] + d[4], d[1] + d[5]);
                    *reinterpret_cast<float2 *>(o + 64) = make_float2(d[2] + d[6], d[3] + d[7]);
                }
            }
            epi_sync();
            if (dbg) dbg[47] = clock64();
            heads_outputs(net, io, hmask_fc, f2, red, nvalid, root0, b2_s, persistent ? ho : nullptr);
        }
        if (dbg) dbg[27] = clock64();
        __threadfence_block();
        epi_sync();
    }
}

// ---------------------------------------------------------------------------------------------- host
// One 3x3 conv -> 9 tap blocks, each [kg = ci/8][co: 64 hi rows | 64 lo rows][ci % 8] fp16.  Returns the power-of-two
// scale applied to the weights (exact), which the caller folds into the BatchNorm scale.
float tc_pack_conv3(const float *w_torch /*[64][cin][3][3]*/, int cin_total, int cin_used, unsigned char *dst)
{
    float mx = 0.0f;
    for (int co = 0; co < 64; ++co)
        for (int ci = 0; ci < cin_used; ++ci)
            for (int t = 0; t < 9; ++t) mx = std::max(mx, fabsf(w_torch[((size_t)co * cin_total + ci) * 9 + t]));
    const float scale = pow2_scale(mx);
    __half *h = reinterpret_cast<__half *>(dst);
    for (int t = 0; t < 9; ++t)
        for (int co = 0; co < 64; ++co)
            for (int ci = 0; ci < 64; ++ci) {
                const size_t off = (size_t)t * (kTapBytes / 2) + ((size_t)(ci / 8) * 128 + co) * 8 + (ci % 8);
                // rows 64-127 of the k-group: the lo parts ([B_hi | B_lo] is one N = 128 operand)
                split_hi_lo(w_torch[((size_t)co * cin_total + ci) * 9 + t] * scale, h[off], h[off + 64 * 8]);
            }
    return scale;
}

// 1x1 head conv [hc][64] -> [hi | lo] with nco rows (zero padded), [kg][co][8].
float tc_pack_conv1(const float *w /*[hc][64]*/, int hc, int nco, int co_offset, unsigned char *dst_hi, unsigned char *dst_lo)
{
    float mx = 0.0f;
    for (int i = 0; i < hc * 64; ++i) mx = std::max(mx, fabsf(w[i]));
    const float scale = pow2_scale(mx);
    __half *hh = reinterpret_cast<__half *>(dst_hi), *hl = reinterpret_cast<__half *>(dst_lo);
    for (int co = 0; co < hc; ++co)
        for (int ci = 0; ci < 64; ++ci) {
            const size_t off = ((size_t)(ci / 8) * nco + co + co_offset) * 8 + (ci % 8);
            split_hi_lo(w[co * 64 + ci] * scale, hh[off], hl[off]);
        }
    return scale;
}

int tc_head_layout_bytes() { return kHeadWBytes; }
int tc_conv_layout_bytes() { return 9 * kTapBytes; }

static unsigned long long *g_dbg = nullptr;     // bring-up instrumentation only (env LZ_TC_DEBUG at model finalize time)
unsigned long long *tc_debug_buffer() { return g_dbg; }

int tc_prepare_launch()
{
    LZ_CUDA_CHECK(cudaFuncSetAttribute(k_net_tc<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcGeo<6>::kSmemBytes));
    LZ_CUDA_CHECK(cudaFuncSetAttribute(k_net_tc<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcGeo<8>::kSmemBytes));
    if (getenv("LZ_TC_DEBUG") && !g_dbg) {      // allocated here (model finalize), never inside a stream capture
        LZ_CUDA_CHECK(cudaMalloc(&g_dbg, 64 * 8));
        LZ_CUDA_CHECK(cudaMemset(g_dbg, 0, 64 * 8));
    }
    return LZ_OK;
}

// roots per CTA: at most one wave of CTAs on the 132 SMs of an H100 SXM (one CTA per SM: ~225 KB of shared memory), at most the
// roots of 3 row tiles: 8 on the 6x6 grid (B = 1024 -> 128 CTAs of 8), 4 on the 8x8 grid (B = 1024 -> 256 CTAs of 4)
static int tc_pick_roots(int hw, int B)
{
    int r = (B + kNumSMs - 1) / kNumSMs;
    return std::min(std::max(r, 1), hw == 8 ? TcGeo<8>::kMaxRoots : TcGeo<6>::kMaxRoots);
}
static int tc_rows_per_root(int hw) { return (hw + 1) * (hw + 1); }
static int tc_f2_max_tiles(int hw) { return hw == 8 ? TcGeo<8>::kF2MaxTiles : TcGeo<6>::kF2MaxTiles; }

// the heads k_net_tc evaluates (the hmask_fc of the kernel) and the FC2 tiles they stream
static int tc_heads_mask(const TcNet &net, const TcIO &io) { return ((net.has_reward && !io.ez_feat) ? 1 : 0) | 6; }
static int tc_fc2_tiles(const TcNet &net, int hmask)
{
    int tiles = 0;
    for (int h = 0; h < 3; ++h)
        if ((hmask >> h) & 1) tiles += (net.fc[h].K + 127) >> 7;
    return tiles;
}

// The plan of a (non-persistent) tc_launch: R, NT, CTAs, roots of the last CTA, layers, passes, whether the FC2 biases are
// staged in shared memory, FC2 tiles.  Mirrors the kernel's set-up code.
void tc_describe(const TcNet &net, const TcIO &io, int32_t *info)
{
    const int R = tc_pick_roots(net.hw, io.B), ctas = (io.B + R - 1) / R, hmask = tc_heads_mask(net, io);
    int nb2 = 0;
    for (int h = 0; h < 3; ++h)
        if ((hmask >> h) & 1) nb2 += net.fc[h].K;
    const int used = net.nlayers * 128;
    info[0] = R;
    info[1] = (R * tc_rows_per_root(net.hw) - (net.hw + 2) + 127) >> 7;
    info[2] = ctas;
    info[3] = io.B - (ctas - 1) * R;
    info[4] = net.nlayers;
    info[5] = io.npass;
    info[6] = (used + nb2) * 4 <= kBnSmemBytes;
    info[7] = tc_fc2_tiles(net, hmask);
}

// The plan of a persistent search launch on a tree of N node slots: R, CTAs, roots of the last CTA, whether pbc[] and the FC2
// biases are staged in shared memory, layers.  Mirrors the kernel's set-up code.
void tc_describe_search(const TcNet &net, const TcIO &io, int N, int32_t *info)
{
    const int R = tc_pick_roots(net.hw, io.B), ctas = (io.B + R - 1) / R, hmask = tc_heads_mask(net, io);
    int nb2 = 0;
    for (int h = 0; h < 3; ++h)
        if ((hmask >> h) & 1) nb2 += net.fc[h].K;
    const bool pbc_smem = (net.nlayers * 128 + N + 1) * 4 <= kBnSmemBytes;
    const int used = net.nlayers * 128 + (pbc_smem ? N + 1 : 0);
    info[0] = R;
    info[1] = ctas;
    info[2] = io.B - (ctas - 1) * R;
    info[3] = pbc_smem;
    info[4] = (used + nb2) * 4 <= kBnSmemBytes;
    info[5] = net.nlayers;
}

int tc_launch(const TcNet &net, const TcIO &io_in, cudaStream_t s, const TreeParams *tp_in)
{
    TcIO io = io_in;
    TreeParams tp;
    memset(&tp, 0, sizeof(tp));
    if (tp_in) tp = *tp_in;
    LZ_REQUIRE(!io.persistent || tp_in, LZ_EINVAL, "tc_launch: persistent search needs tree parameters");
    LZ_REQUIRE(net.A <= 1000, LZ_EINVAL, "tc_launch: action space %d too large for the head scratch of the tensor-core path", net.A);
    LZ_REQUIRE(io.skip_scratch, LZ_EINVAL, "tc_launch: no skip scratch");
    LZ_REQUIRE(net.hw == 6 || net.hw == 8, LZ_EINVAL, "tc_launch: latent grid %dx%d not supported (6x6 or 8x8)", net.hw, net.hw);
    LZ_REQUIRE(tc_fc2_tiles(net, tc_heads_mask(net, io)) <= tc_f2_max_tiles(net.hw), LZ_EINVAL, "tc_launch: %d FC2 tiles exceed the %d of the head scratch",
               tc_fc2_tiles(net, tc_heads_mask(net, io)), tc_f2_max_tiles(net.hw));
    io.dbg = g_dbg;
    io.roots_per_cta = tc_pick_roots(net.hw, io.B);
    LZ_REQUIRE(!io.persistent || tp.A <= 32, LZ_EINVAL, "tc_launch: the persistent search needs A <= 32 (got %d)", tp.A);
    const int grid = (io.B + io.roots_per_cta - 1) / io.roots_per_cta;
    if (net.hw == 8) k_net_tc<8><<<grid, kTcThreads, TcGeo<8>::kSmemBytes, s>>>(net, io, tp);
    else k_net_tc<6><<<grid, kTcThreads, TcGeo<6>::kSmemBytes, s>>>(net, io, tp);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

}  // namespace lz
