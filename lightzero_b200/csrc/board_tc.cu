// board_tc.cu -- tensor-core (wgmma) network of the board-game MuZero models (downsample=False, muzero_model.py:20-272):
// representation conv3x3(obs -> C) + BN + ReLU (common.py:764-787), the dynamics conv over [latent | one-hot action planes] + BN +
// latent + ReLU (muzero_model.py:505-538), ResBlocks, and the 1x1-conv + MLP heads (common.py:1189-1215), all at board resolution.
//
// One launch runs the whole program of recurrent_inference (or initial_inference) for all roots; a CTA owns R roots.  Convolutions
// use the arithmetic of net_tc.cu: 3xFP16 (A_hi B_hi + A_hi B_lo + A_lo B_hi, fp32 accumulators in registers; one pass in tc1),
// weights pre-split on the host and pre-scaled by a power of two that is folded into the BatchNorm scale.  Activations live in
// shared memory in the wgmma K-major no-swizzle layout [k-group of 8 channels][row][8 halves]: rows are the pixels of a padded
// (W + 1)-wide grid, (H + 1)(W + 1) rows per root, so the input row of output row m for tap (dy, dx) is m + (W + 1) dy + dx and
// every tap is the same buffer read through a shifted descriptor; the zero pad column / row of each root is the conv padding, and
// W + 2 zero margin rows sit before and after the tiles.  The roots' rows are cut into NT tiles of 64 (one m64nCk16 wgmma per
// tile and k-step); the single warpgroup keeps every tile's accumulators in registers until the layer's MMAs are done, then the
// epilogue (BN, residual, action planes, ReLU) rewrites the buffer in place straight from the fragments.  ResBlock skip tensors
// stay in shared memory as fp32 rows.  The conv weights stream through a ring of per-tap stages (cp.async.bulk, mbarrier
// complete_tx), refilled by thread 0 as soon as every warp's MMAs have read a stage.
// The heads are plain fp32 FMA on the CUDA cores (~20-60 k MAC per root against 0.1-7.7 M MAC of convolutions); the categorical
// read-out is net6.cuh's canonical categorical_to_scalar.
#include <cuda_fp16.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <array>

#include "board_tc.cuh"
#include "model.cuh"
#include "net6.cuh"
#include "tc_ptx.cuh"

namespace lz {

constexpr int kBoardThreads = 128;                 // one warpgroup: MMA issue, epilogues and heads
constexpr int kBoardKmax = 608;                    // largest support / action count of a head

template <int C>
struct BoardGeo {
    static constexpr int kMaxTiles = C == 64 ? 4 : 8;       // the register accumulator budget: NT * C / 2 <= 128 per thread
    static constexpr int kStages = C == 64 ? 3 : 4;         // weight ring stages of one tap each
    static constexpr int kStageBytes = C * C * 4;           // one tap with cin = C: [C / 8 k-groups][C hi | C lo rows][16 B]
    static constexpr int kSkipLd = C + 8;                   // fp32 skip rows (+8: spreads the fragment stores over the banks)
};

struct BoardSmem {
    int act, skip, ring, feat, hid, lbuf, bars, total;
};

// byte offsets of the shared-memory regions of a CTA with R roots in NT tiles
template <int C>
__host__ __device__ inline BoardSmem board_smem(int NT, int R, int H, int W)
{
    using G = BoardGeo<C>;
    const int P = H * W, rows_alloc = 2 * (W + 2) + NT * 64;
    BoardSmem s;
    s.act = 0;
    s.skip = 2 * (C / 8) * rows_alloc * 16;
    s.ring = (s.skip + NT * 64 * G::kSkipLd * 4 + 127) & ~127;
    s.feat = s.ring + G::kStages * G::kStageBytes;
    s.hid = s.feat + R * 16 * P * 4;
    s.lbuf = s.hid + R * 32 * 4;
    s.bars = (s.lbuf + 4 * kBoardKmax * 4 + 7) & ~7;
    s.total = s.bars + G::kStages * 8;
    return s;
}

// root b is computed: no row mask, or its mask bit selects it
__device__ __forceinline__ bool board_root_on(const BoardIO &io, int b)
{
    return !io.row_mask || (__ldg(io.row_mask + b) & 1) == io.row_mask_on;
}

// row m of a CTA's padded grid -> (root slot r, pixel p); false for pad rows and absent roots (past the batch, or masked off)
__device__ __forceinline__ bool board_row(const BoardIO &io, int m, int root0, int nvalid, int H, int W, int &r, int &p)
{
    const int pitch = W + 1, rpr = (H + 1) * pitch;
    r = m / rpr;
    const int q = m - r * rpr, y = q / pitch, x = q - y * pitch;
    p = y * W + x;
    return r < nvalid && y < H && x < W && board_root_on(io, root0 + r);
}

// one head for the CTA's roots from the fp32 latent rows in skip: 1x1 conv + BN + ReLU -> feat, FC1 + BN1d + ReLU -> hid, FC2 ->
// logits (one warp per root, rows ld apart in glog), the categorical heads' scalar through categorical_to_scalar; masked-off
// roots are computed on their zero rows and not written
template <int C>
__device__ void board_head(const BoardNet &net, const BoardIO &io, const BoardHead &hd, const float *skip, float *feat, float *hidb,
                           float *lbuf, int nvalid, int root0, float *glog, int ld, float *gscal, bool categorical)
{
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int H = net.H, W = net.W, P = H * W, pitch = W + 1, rpr = (H + 1) * pitch;
    const int hc = hd.hc, nin = hc * P, hid = hd.hid, K = hd.K;
    for (int i = tid; i < nvalid * nin; i += kBoardThreads) {
        const int r = i / nin, k = i - r * nin, c = k / P, p = k - c * P;
        const float *x = skip + (size_t)(r * rpr + (p / W) * pitch + p % W) * BoardGeo<C>::kSkipLd;
        const float *w = hd.w1 + c * C;
        float a = 0.0f;
#pragma unroll 8
        for (int ci = 0; ci < C; ++ci) a = fmaf(__ldg(w + ci), x[ci], a);
        feat[i] = fmaxf(fmaf(a, __ldg(hd.s1 + c), __ldg(hd.t1 + c)), 0.0f);
    }
    __syncthreads();
    for (int i = tid; i < nvalid * hid; i += kBoardThreads) {
        const int r = i / hid, j = i - r * hid;
        const float *w = hd.fc1 + (size_t)j * nin, *f = feat + r * nin;
        float a = 0.0f;
        for (int k = 0; k < nin; ++k) a = fmaf(__ldg(w + k), f[k], a);
        hidb[i] = fmaxf(fmaf(a, __ldg(hd.s2 + j), __ldg(hd.t2 + j)), 0.0f);
    }
    __syncthreads();
    float *lrow = lbuf + warp * kBoardKmax;
    for (int r = warp; r < nvalid; r += kBoardThreads / 32) {
        const float *hv = hidb + r * hid;
        const int b = root0 + r;
        if (!board_root_on(io, b)) continue;
        for (int k = lane; k < K; k += 32) {
            const float *w = hd.fc2 + (size_t)k * hid;
            float a = 0.0f;
            for (int j = 0; j < hid; ++j) a = fmaf(__ldg(w + j), hv[j], a);
            a += __ldg(hd.b2 + k);
            lrow[k] = a;
            if (glog) glog[(size_t)b * ld + k] = a;
        }
        __syncwarp();
        if (categorical) {
            const float v = categorical_to_scalar(lrow, K, net.support_min, net.support_step, lane);
            if (lane == 0 && gscal) gscal[b] = v;
        }
        __syncwarp();
    }
    __syncthreads();
}

// The MMAs of one tap for every tile: KS k-steps of 16 input channels, NP passes (3: hi/lo, 1: hi only), straight-line so that no
// branch separates the wgmma of a commit group
template <int C, int NT, int KS, int NP>
__device__ __forceinline__ void board_tap_mma(float (&acc)[NT][C / 2], uint64_t a0, uint64_t b0, uint32_t a_kstep, uint32_t a_lo,
                                              uint32_t b_kstep)
{
#pragma unroll
    for (int t = 0; t < NT; ++t)
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            const uint64_t a = a0 + (uint64_t)(t * 64) + ks * a_kstep, b = b0 + ks * b_kstep;
            wgmma_f16<C>(acc[t], a, b);
            if constexpr (NP == 3) {
                wgmma_f16<C>(acc[t], a, b + C);        // B_lo: the C rows after B_hi (C x 16 B)
                wgmma_f16<C>(acc[t], a + a_lo, b);
            }
        }
}

template <int C, int NT>
__global__ void __launch_bounds__(kBoardThreads, 1) k_board_tc(BoardNet net, BoardIO io, int R)
{
    using G = BoardGeo<C>;
    constexpr int kS = G::kStages, kLd = G::kSkipLd;
    extern __shared__ __align__(128) unsigned char smem[];
    const int H = net.H, W = net.W, P = H * W, pitch = W + 1, margin = W + 2;
    const BoardSmem L = board_smem<C>(NT, R, H, W);
    const int plane_bytes = (2 * margin + NT * 64) * 16, part_bytes = (C / 8) * plane_bytes;
    unsigned char *act = smem;
    float *skip = reinterpret_cast<float *>(smem + L.skip);
    unsigned char *ring = smem + L.ring;
    float *feat = reinterpret_cast<float *>(smem + L.feat), *hidb = reinterpret_cast<float *>(smem + L.hid);
    float *lbuf = reinterpret_cast<float *>(smem + L.lbuf);
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + L.bars);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int root0 = blockIdx.x * R, nvalid = min(R, io.B - root0);
    const int nl = net.nlayers, total = nl * 9;
    if (io.row_mask) {
        bool any = false;
        for (int r = tid; r < nvalid; r += kBoardThreads) any |= board_root_on(io, root0 + r);
        if (!__syncthreads_or(any)) return;    // no selected root in this CTA: no weights streamed, nothing written
    }

    auto issue = [&](int pos) {        // thread 0: tap pos of the program's weight stream into its ring stage
        const int layer = pos / 9, tap = pos - layer * 9;
        const uint32_t bytes = ((net.layer_flags[layer] & BF_OBS) ? 16 : C) * C * 4;
        uint64_t *bar = &full[pos % kS];
        mbar_expect_tx(bar, bytes);
        bulk_g2s(ring + (pos % kS) * G::kStageBytes, net.convw + net.layer_woff[layer] + (size_t)tap * bytes, bytes, bar);
    };
    if (tid == 0) {
        for (int i = 0; i < kS; ++i) mbar_init(&full[i], 1);
        fence_mbar_init();
        for (int i = 0; i < min(kS, total); ++i) issue(i);
    }
    // zero the activation buffer (margins, pad rows, planes the first layer does not fill)
    for (int i = tid; i < 2 * part_bytes / 16; i += kBoardThreads) reinterpret_cast<uint4 *>(act)[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();

    // ---- input: observation planes (initial_inference) or the latents (recurrent_inference), fp16 hi / lo (+ fp32 skip rows)
    {
        const bool obs = (net.layer_flags[0] & BF_OBS) != 0;
        const int ch = obs ? 16 : C;
        for (int i = tid; i < ch * NT * 64; i += kBoardThreads) {
            const int c = i / (NT * 64), m = i - c * (NT * 64);
            int r, p;
            float v = 0.0f;
            if (board_row(io, m, root0, nvalid, H, W, r, p)) {
                const int b = root0 + r;
                if (obs) v = c < io.obs_c ? io.obs[((size_t)b * io.obs_c + c) * P + p] : 0.0f;
                else v = io.latent_base[(io.ix ? (size_t)io.ix[b] * io.slot_stride : 0) + ((size_t)b * C + c) * P + p];
            }
            if (!obs) skip[m * kLd + c] = v;
            const float vc = fminf(fmaxf(v, -65504.0f), 65504.0f);
            const __half hi = __float2half_rn(vc);
            unsigned char *d = act + (c >> 3) * plane_bytes + (margin + m) * 16 + (c & 7) * 2;
            *reinterpret_cast<__half *>(d) = hi;
            *reinterpret_cast<__half *>(d + part_bytes) = __float2half_rn(vc - __half2float(hi));
        }
    }
    fence_proxy_async();
    __syncthreads();

    // rows of this thread's accumulator fragments: tile t, half h -> root slot << 8 | pixel, or -1
    int rinfo[NT][2];
#pragma unroll
    for (int t = 0; t < NT; ++t)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            int r, p;
            rinfo[t][h] = board_row(io, t * 64 + 16 * warp + (lane >> 2) + 8 * h, root0, nvalid, H, W, r, p) ? ((r << 8) | p) : -1;
        }

    const uint32_t act_s = smem_u32(act), ring_s = smem_u32(ring);
    const uint64_t a_base = make_desc(act_s + margin * 16, plane_bytes >> 4, 8);
    const uint64_t b_base = make_desc(ring_s, (2 * C * 16) >> 4, 8);
    const uint32_t a_kstep = (2 * plane_bytes) >> 4, a_lo = part_bytes >> 4, b_kstep = (2 * 2 * C * 16) >> 4;
    int pos = 0;
    for (int layer = 0; layer < nl; ++layer) {
        const int flags = net.layer_flags[layer];
        const bool obs16 = (flags & BF_OBS) != 0;
        float acc[NT][C / 2];
#pragma unroll
        for (int t = 0; t < NT; ++t) {
#pragma unroll
            for (int i = 0; i < C / 2; ++i) acc[t][i] = 0.0f;
            wg_fence_acc(acc[t]);
        }
        for (int tap = 0; tap < 9; ++tap, ++pos) {
            mbar_wait(&full[pos % kS], (pos / kS) & 1);
            const int shift = (tap / 3 - 1) * pitch + (tap % 3 - 1);
            const uint64_t a0 = a_base + (uint64_t)(int64_t)shift, b0 = b_base + (uint64_t)(((pos % kS) * G::kStageBytes) >> 4);
            wg_fence();
            if (io.npass == 3) {
                if (obs16) board_tap_mma<C, NT, 1, 3>(acc, a0, b0, a_kstep, a_lo, b_kstep);
                else board_tap_mma<C, NT, C / 16, 3>(acc, a0, b0, a_kstep, a_lo, b_kstep);
            } else {
                if (obs16) board_tap_mma<C, NT, 1, 1>(acc, a0, b0, a_kstep, a_lo, b_kstep);
                else board_tap_mma<C, NT, C / 16, 1>(acc, a0, b0, a_kstep, a_lo, b_kstep);
            }
            wg_commit();
            if (tap > 0) {
                wg_wait<1>();                       // the previous tap's MMAs have read their stage: refill it
                __syncthreads();
                if (tid == 0 && pos - 1 + kS < total) issue(pos - 1 + kS);
            }
        }
        wg_wait<0>();
#pragma unroll
        for (int t = 0; t < NT; ++t) wg_fence_acc(acc[t]);
        __syncthreads();                            // every MMA of the layer has read the buffer: it may be rewritten
        if (tid == 0 && pos - 1 + kS < total) issue(pos - 1 + kS);

        // ---- epilogue straight from the fragments: BN (+ skip + action planes) + ReLU -> fp16 hi / lo in place (+ skip, latent)
        const float *bn = net.bn + net.layer_bn[layer];
        const bool res = (flags & BF_RES) != 0, ab = (flags & BF_ACT_BIAS) != 0, store = (flags & BF_STORE_RES) != 0;
        const bool wl = (flags & BF_WRITE_LATENT) != 0;
#pragma unroll
        for (int t = 0; t < NT; ++t)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = t * 64 + 16 * warp + (lane >> 2) + 8 * h, info = rinfo[t][h];
                const int r = info >> 8, p = info & 255, b = root0 + r;
                const float *abr = nullptr;
                if (ab && info >= 0) abr = net.abias + (size_t)min(max(io.action[b], 0), net.nopt - 1) * C * P + p;
#pragma unroll
                for (int j = 0; j < C / 8; ++j) {
                    const int c = 8 * j + 2 * (lane & 3);
                    float v0 = acc[t][4 * j + 2 * h], v1 = acc[t][4 * j + 2 * h + 1];
                    if (info >= 0) {
                        v0 = fmaf(v0, __ldg(bn + c), __ldg(bn + C + c));
                        v1 = fmaf(v1, __ldg(bn + c + 1), __ldg(bn + C + c + 1));
                        if (res) {
                            float2 s = *reinterpret_cast<const float2 *>(skip + m * kLd + c);
                            if (abr) { s.x += __ldg(abr + (size_t)c * P); s.y += __ldg(abr + (size_t)(c + 1) * P); }
                            v0 += s.x; v1 += s.y;
                        }
                        v0 = fmaxf(v0, 0.0f); v1 = fmaxf(v1, 0.0f);
                        if (store) *reinterpret_cast<float2 *>(skip + m * kLd + c) = make_float2(v0, v1);
                        if (wl) {
                            const size_t o = ((size_t)b * C + c) * P + p;
                            if (io.latent_out) { io.latent_out[o] = v0; io.latent_out[o + P] = v1; }
                            if (io.latent_out2) { io.latent_out2[o] = v0; io.latent_out2[o + P] = v1; }
                        }
                    } else {
                        v0 = v1 = 0.0f;                 // pad rows / absent roots: the next layer's conv padding
                    }
                    const __half2 hi = __floats2half2_rn(fminf(v0, 65504.0f), fminf(v1, 65504.0f));
                    const float2 back = __half22float2(hi);
                    unsigned char *d = act + (c >> 3) * plane_bytes + (margin + m) * 16 + (c & 7) * 2;
                    *reinterpret_cast<__half2 *>(d) = hi;
                    *reinterpret_cast<__half2 *>(d + part_bytes) = __floats2half2_rn(v0 - back.x, v1 - back.y);
                }
            }
        fence_proxy_async();
        __syncthreads();                            // the layer's output is visible to the next MMAs and to the heads

        if (flags & BF_HOOK_REWARD) {
            if (io.reward_logits || io.reward)
                board_head<C>(net, io, net.head[0], skip, feat, hidb, lbuf, nvalid, root0, io.reward_logits, net.head[0].K, io.reward, true);
        }
        if (flags & BF_HOOK_VALPOL) {
            if (io.value_logits || io.value)
                board_head<C>(net, io, net.head[1], skip, feat, hidb, lbuf, nvalid, root0, io.value_logits, net.head[1].K, io.value, true);
            if (io.policy_logits)
                board_head<C>(net, io, net.head[2], skip, feat, hidb, lbuf, nvalid, root0, io.policy_logits,
                              io.policy_stride ? io.policy_stride : net.head[2].K, nullptr, false);
        }
    }
}

// ---------------------------------------------------------------------------------------------- host
static int board_max_tiles(int C) { return C == 64 ? BoardGeo<64>::kMaxTiles : (C == 32 ? BoardGeo<32>::kMaxTiles : BoardGeo<16>::kMaxTiles); }

static int board_smem_total(int C, int NT, int R, int H, int W)
{
    return C == 64 ? board_smem<64>(NT, R, H, W).total : (C == 32 ? board_smem<32>(NT, R, H, W).total : board_smem<16>(NT, R, H, W).total);
}

// Roots per CTA: B / 132 rounded up (small collector batches spread over the SMs, a reanalyze batch of ~1000-1500 roots fills
// about one wave), capped by the rows the accumulator tiles hold; the tile count is the fewest 64-row tiles that hold R roots.
BoardPlan board_plan(const BoardNet &net, int B)
{
    const int rpr = (net.H + 1) * (net.W + 1), pad = net.W + 2, max_rows = board_max_tiles(net.C) * 64;
    const int rmax = std::max(1, (max_rows + pad) / rpr);
    BoardPlan p;
    p.R = std::min(rmax, std::max(1, ceil_div(B, kNumSMs)));
    const int rows = p.R * rpr - pad;
    p.NT = std::max(1, ceil_div(rows, 64));
    p.ctas = ceil_div(B, p.R);
    p.last = B - (p.ctas - 1) * p.R;
    p.smem = board_smem_total(net.C, p.NT, p.R, net.H, net.W);
    return p;
}

// one instantiation per tile count NT = 1 .. kMaxTiles of each channel count
template <int C, int NT = 1>
static bool board_go(const BoardNet &net, const BoardIO &io, const BoardPlan &p, cudaStream_t s)
{
    if constexpr (NT > BoardGeo<C>::kMaxTiles) {
        return false;
    } else {
        if (p.NT != NT) return board_go<C, NT + 1>(net, io, p, s);
        k_board_tc<C, NT><<<p.ctas, kBoardThreads, p.smem, s>>>(net, io, p.R);
        return true;
    }
}

template <int C, int NT = 1>
static int board_attr()
{
    if constexpr (NT > BoardGeo<C>::kMaxTiles) {
        return LZ_OK;
    } else {
        LZ_CUDA_CHECK(cudaFuncSetAttribute(k_board_tc<C, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        return board_attr<C, NT + 1>();
    }
}

int board_prepare_launch()
{
    int rc = board_attr<16>();
    if (rc == LZ_OK) rc = board_attr<32>();
    if (rc == LZ_OK) rc = board_attr<64>();
    return rc;
}

int board_launch(const BoardNet &net, const BoardIO &io, cudaStream_t s)
{
    LZ_REQUIRE(io.B > 0 && (io.npass == 1 || io.npass == 3), LZ_EINVAL, "board_launch: bad argument");
    const BoardPlan p = board_plan(net, io.B);
    LZ_REQUIRE(p.smem <= 227 * 1024, LZ_EINVAL, "board_launch: %d B of shared memory needed", p.smem);
    const bool ok = net.C == 16 ? board_go<16>(net, io, p, s) : (net.C == 32 ? board_go<32>(net, io, p, s) : (net.C == 64 && board_go<64>(net, io, p, s)));
    LZ_REQUIRE(ok, LZ_EINVAL, "board_launch: no kernel for C = %d with %d tiles", net.C, p.NT);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

float board_pack_conv3(const float *w, int C, int cin_total, int cin_used, int cin_pad, unsigned char *dst)
{
    float mx = 0.0f;
    for (int co = 0; co < C; ++co)
        for (int ci = 0; ci < cin_used; ++ci)
            for (int t = 0; t < 9; ++t) mx = std::max(mx, fabsf(w[((size_t)co * cin_total + ci) * 9 + t]));
    const float scale = pow2_scale(mx);
    __half *h = reinterpret_cast<__half *>(dst);
    const size_t tap_halves = (size_t)cin_pad * C * 2;
    for (int t = 0; t < 9; ++t)
        for (int co = 0; co < C; ++co)
            for (int ci = 0; ci < cin_pad; ++ci) {
                const float v = ci < cin_used ? w[((size_t)co * cin_total + ci) * 9 + t] * scale : 0.0f;
                const size_t off = t * tap_halves + ((size_t)(ci / 8) * 2 * C + co) * 8 + ci % 8;
                split_hi_lo(v, h[off], h[off + (size_t)C * 8]);
            }
    return scale;
}

// The encoding planes' share of a dynamics conv (torch [C][C + planes][3][3]) for each of n options: border-aware tap sums of the
// option's plane, times its plane value, times the BN scale.  One-hot encoding (muzero_model.py:341-369): option o is plane o at
// value 1.  Scalar plane (stochastic_muzero_model.py:354-377, 408-431): option o is plane 0 at value o / n in fp32, as the
// reference computes it.  The tap sum accumulates in double and is rounded once.
static void board_option_table(const std::vector<float> &w, int C, int cin_total, int H, int W, int n, bool onehot,
                               const std::vector<float> &scale, float *dst)
{
    const int P = H * W;
    for (int o = 0; o < n; ++o) {
        const int plane = onehot ? o : 0;
        const double v = onehot ? 1.0 : (double)((float)o / (float)n);
        for (int co = 0; co < C; ++co)
            for (int y = 0; y < H; ++y)
                for (int x = 0; x < W; ++x) {
                    double acc = 0.0;
                    for (int t = 0; t < 9; ++t) {
                        const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
                        if (yy >= 0 && yy < H && xx >= 0 && xx < W) acc += w[((size_t)co * cin_total + C + plane) * 9 + t];
                    }
                    dst[((size_t)o * C + co) * P + y * W + x] = (float)(acc * v) * scale[co];
                }
    }
}

// ---- the Board family (lz_model::board) ----------------------------------------------------------------------------------
// tables of the board network: fp16 hi/lo conv weights, folded BN, option planes, fp32 heads.  MuZeroModel has two programs,
// StochasticMuZeroModel (m->chance != 0, stochastic_muzero_model.py) three: `init` (representation + prediction), `rec`
// (dynamics_network over [afterstate | chance plane] + prediction_network, recurrent_inference(afterstate=True)) and `after`
// (afterstate_dynamics_network over [latent | action plane] + afterstate_prediction_network with chance_space_size policy
// outputs, recurrent_inference(afterstate=False)).  Its dynamics networks name their BNs bn / bn_reward where MuZeroModel's
// has norm_common / norm_reward, and its afterstate prediction network bn_value / bn_policy where prediction_network has
// norm_value / norm_policy.
int board_finalize(lz_model *m)
{
    const lz_model_config &c = m->board.cfg;
    const int C = c.num_channels, A = c.action_space_size, n = c.num_res_blocks, H = c.obs_h, W = c.obs_w, P = H * W;
    const int NC = m->chance;
    const bool stoch = NC != 0;
    const std::string D = "dynamics_network.", Q = "prediction_network.", R = "representation_network.";
    const std::string AD = "afterstate_dynamics_network.", AQ = "afterstate_prediction_network.";
    const std::string dyn_bn = stoch ? "bn" : "norm_common", rew_bn = stoch ? "bn_reward" : "norm_reward";
    struct Conv { std::string w, bn; int cin_total, cin_used, cin_pad; };
    // conv indices: 0 dyn conv | 1..2n dyn blocks | 2n+1..4n pred blocks | 4n+1..6n rep blocks | 6n+1 rep conv, and for
    // StochasticMuZeroModel 6n+2 afterstate dyn conv | 6n+3..8n+2 its blocks | 8n+3..10n+2 afterstate pred blocks
    std::vector<Conv> convs;
    auto blocks_of = [&](const std::string &pre) {
        for (int i = 0; i < n; ++i) {
            const std::string b = pre + "resblocks." + std::to_string(i);
            convs.push_back({b + ".conv1.0.weight", b + ".conv1.1", C, C, C});
            convs.push_back({b + ".conv2.0.weight", b + ".conv2.1", C, C, C});
        }
    };
    convs.push_back({D + "conv.weight", D + dyn_bn, C + (stoch ? 1 : A), C, C});
    for (const std::string &pre : {D, Q, R}) blocks_of(pre);
    convs.push_back({R + "conv.weight", R + "norm", c.obs_c, c.obs_c, 16});   // observation planes padded to 16 with zero weights
    const int after_conv = 6 * n + 2;
    if (stoch) {
        convs.push_back({AD + "conv.weight", AD + "bn", C + 1, C, C});
        blocks_of(AD);
        blocks_of(AQ);
    }
    // option tables of the recurrent programs' dynamics convs: rec (actions one-hot, or chance outcomes on a scalar plane),
    // after (actions on a scalar plane)
    struct OptTable { int conv, n; bool onehot; size_t off; };
    std::vector<OptTable> tables = {{0, stoch ? NC : A, !stoch, 0}};
    if (stoch) tables.push_back({after_conv, A, false, (size_t)NC * C * P});
    const size_t ab_floats = tables.back().off + (size_t)tables.back().n * C * P;
    const int nconv = (int)convs.size();
    auto align = [](size_t v) { return (v + 127) & ~(size_t)127; };
    std::vector<size_t> woff(nconv);
    size_t off = 0;
    for (int i = 0; i < nconv; ++i) { woff[i] = off; off += (size_t)9 * convs[i].cin_pad * C * 4; }
    const size_t off_bn = align(off), off_ab = align(off_bn + (size_t)nconv * 2 * C * 4), off_heads = align(off_ab + ab_floats * 4);
    std::vector<unsigned char> host(off_heads, 0);
    float *bn = reinterpret_cast<float *>(host.data() + off_bn), *ab = reinterpret_cast<float *>(host.data() + off_ab);
    for (int ci = 0; ci < nconv; ++ci) {
        const Conv &cv = convs[ci];
        auto w = find_tensor(m, cv.w, (size_t)C * cv.cin_total * 9);
        std::vector<float> scale, shift;
        if (!w || !fold_bn(m, cv.bn, C, scale, shift)) return LZ_EINVAL;
        const float ws = board_pack_conv3(w->data(), C, cv.cin_total, cv.cin_used, cv.cin_pad, host.data() + woff[ci]);
        for (int k = 0; k < C; ++k) { bn[ci * 2 * C + k] = scale[k] / ws; bn[ci * 2 * C + C + k] = shift[k]; }
        for (const OptTable &t : tables)
            if (t.conv == ci) board_option_table(*w, C, cv.cin_total, H, W, t.n, t.onehot, scale, ab + t.off);
    }
    // heads: fp32 tables (conv bias folded into the 1x1 BN shift, Linear bias into the BN1d shift); reward, value, policy of
    // rec and init, then of after
    struct HD { std::string conv, norm, fc; int hc, hid, K; };
    std::vector<HD> heads = {{D + "conv1x1_reward", D + rew_bn, D + "fc_reward_head", c.reward_head_channels, c.reward_hidden, m->K},
                             {Q + "conv1x1_value", Q + "norm_value", Q + "fc_value", c.value_head_channels, c.value_hidden, m->K},
                             {Q + "conv1x1_policy", Q + "norm_policy", Q + "fc_policy", c.policy_head_channels, c.policy_hidden, A}};
    if (stoch) {
        heads.push_back({AD + "conv1x1_reward", AD + "bn_reward", AD + "fc_reward_head", c.reward_head_channels, c.reward_hidden, m->K});
        heads.push_back({AQ + "conv1x1_value", AQ + "bn_value", AQ + "fc_value", c.value_head_channels, c.value_hidden, m->K});
        heads.push_back({AQ + "conv1x1_policy", AQ + "bn_policy", AQ + "fc_policy", c.policy_head_channels, c.policy_hidden, NC});
    }
    const int nheads = (int)heads.size();
    TablePacker hp;
    std::vector<std::array<size_t, 8>> hoff(nheads);
    for (int h = 0; h < nheads; ++h) {
        const HD &d = heads[h];
        const int nin = d.hc * P;
        auto w1 = find_tensor(m, d.conv + ".weight", (size_t)d.hc * C), b1 = find_tensor(m, d.conv + ".bias", d.hc);
        auto W0 = find_tensor(m, d.fc + ".0.weight", (size_t)d.hid * nin), B0 = find_tensor(m, d.fc + ".0.bias", d.hid);
        auto W3 = find_tensor(m, d.fc + ".3.weight", (size_t)d.K * d.hid), B3 = find_tensor(m, d.fc + ".3.bias", d.K);
        std::vector<float> s1, t1, s2, t2;
        if (!w1 || !b1 || !W0 || !B0 || !W3 || !B3 || !fold_bn(m, d.norm, d.hc, s1, t1) || !fold_bn(m, d.fc + ".1", d.hid, s2, t2))
            return LZ_EINVAL;
        for (int i = 0; i < d.hc; ++i) t1[i] += s1[i] * (*b1)[i];
        for (int j = 0; j < d.hid; ++j) t2[j] += s2[j] * (*B0)[j];
        const std::vector<float> *parts[8] = {w1, &s1, &t1, W0, &s2, &t2, W3, B3};
        for (int k = 0; k < 8; ++k) hoff[h][k] = hp.add(*parts[k]);
    }
    host.resize(off_heads + hp.host.size() * sizeof(float));
    memcpy(host.data() + off_heads, hp.host.data(), hp.host.size() * sizeof(float));
    int rc = upload(&m->board.d_board, host.data(), host.size());
    if (rc != LZ_OK) return rc;
    BoardNet base;
    memset(&base, 0, sizeof(base));
    base.convw = m->board.d_board;
    base.bn = reinterpret_cast<const float *>(m->board.d_board + off_bn);
    const float *abd = reinterpret_cast<const float *>(m->board.d_board + off_ab);
    const float *hb = reinterpret_cast<const float *>(m->board.d_board + off_heads);
    base.C = C; base.H = H; base.W = W;
    base.support_min = c.support_min; base.support_step = c.support_step;
    // a program's three heads from heads[h0 ..], its option table from tables[t]
    auto program = [&](int h0, int t) {
        BoardNet net = base;
        for (int h = 0; h < 3; ++h) {
            BoardHead &o = net.head[h];
            const std::array<size_t, 8> &q = hoff[h0 + h];
            o.w1 = hb + q[0]; o.s1 = hb + q[1]; o.t1 = hb + q[2];
            o.fc1 = hb + q[3]; o.s2 = hb + q[4]; o.t2 = hb + q[5];
            o.fc2 = hb + q[6]; o.b2 = hb + q[7];
            o.hc = heads[h0 + h].hc; o.hid = heads[h0 + h].hid; o.K = heads[h0 + h].K;
        }
        net.abias = abd + tables[t].off;
        net.nopt = tables[t].n;
        return net;
    };
    BoardNet rec = program(0, 0), init = program(0, 0), after = stoch ? program(3, 1) : base;
    auto add = [&](BoardNet &net, int ci, int flags) {
        net.layer_woff[net.nlayers] = (uint32_t)woff[ci];
        net.layer_bn[net.nlayers] = ci * 2 * C;
        net.layer_flags[net.nlayers++] = flags;
    };
    auto blocks = [&](BoardNet &net, int first, int last_flags) {
        for (int i = 0; i < n; ++i) {
            add(net, first + 2 * i, 0);
            add(net, first + 2 * i + 1, BF_RES | BF_STORE_RES | (i == n - 1 ? last_flags : 0));
        }
    };
    add(rec, 0, BF_RES | BF_STORE_RES | BF_ACT_BIAS);
    blocks(rec, 1, BF_WRITE_LATENT | BF_HOOK_REWARD);
    blocks(rec, 2 * n + 1, BF_HOOK_VALPOL);
    add(init, 6 * n + 1, BF_OBS | BF_STORE_RES);
    blocks(init, 4 * n + 1, BF_WRITE_LATENT);
    blocks(init, 2 * n + 1, BF_HOOK_VALPOL);
    if (stoch) {
        add(after, after_conv, BF_RES | BF_STORE_RES | BF_ACT_BIAS);
        blocks(after, after_conv + 1, BF_WRITE_LATENT | BF_HOOK_REWARD);
        blocks(after, after_conv + 1 + 2 * n, BF_HOOK_VALPOL);
    }
    m->board.rec = rec; m->board.init = init; m->board.after = after;
    return board_prepare_launch();
}

static BoardIO board_io(const lz_model *m, int B)
{
    BoardIO b;
    memset(&b, 0, sizeof(b));
    b.B = B; b.npass = m->npass; b.obs_c = m->board.cfg.obs_c;
    return b;
}

int board_recurrent(lz_model *m, const RecIO &io, cudaStream_t s)
{
    BoardIO b = board_io(m, io.B);
    b.latent_base = io.latent_base; b.ix = io.ix; b.slot_stride = io.slot_stride; b.action = io.action;
    b.latent_out = io.next_latent; b.reward = io.reward; b.value = io.value; b.policy_logits = io.policy_logits;
    b.reward_logits = io.reward_logits; b.value_logits = io.value_logits;
    b.policy_stride = io.policy_stride; b.row_mask = io.row_mask; b.row_mask_on = io.row_mask_on;
    return board_launch(io.after_program ? m->board.after : m->board.rec, b, s);
}

int board_initial(lz_model *m, int B, const float *d_obs, const TailIO &io_in, cudaStream_t s)
{
    BoardIO b = board_io(m, B);
    b.obs = d_obs; b.latent_out = io_in.latent; b.latent_out2 = io_in.latent2;
    b.value = io_in.value; b.policy_logits = io_in.policy_logits; b.value_logits = io_in.value_logits;
    b.policy_stride = io_in.policy_stride;
    return board_launch(m->board.init, b, s);
}

// lz_model_debug_net_stage of the board network: which 1 is the whole initial_inference program, d_latent the observations;
// which 2 StochasticMuZeroModel's afterstate program (policy logits chance_space_size wide)
int board_debug_stage(lz_model *m, int which, int B, const float *d_in, const int32_t *d_action, int stage, void *d_out,
                             size_t out_bytes, int32_t *h_info, cudaStream_t st)
{
    // a copy: the model's programs stay as they are
    BoardNet net = which == 2 ? m->board.after : which ? m->board.init : m->board.rec;
    const int nl = net.nlayers, K = m->K, A = net.head[2].K;
    const bool obs = which == 1;
    LZ_REQUIRE(stage <= nl, LZ_EINVAL, "lz_model_debug_net_stage: stage %d past the %d layers of the program", stage, nl);
    const size_t nfl = stage < nl ? (size_t)B * m->latent_floats : (size_t)B * (2 * K + 2 * A + 4);
    LZ_REQUIRE(out_bytes >= nfl * sizeof(float), LZ_EINVAL, "lz_model_debug_net_stage: stage %d needs %zu bytes, got %zu", stage,
               nfl * sizeof(float), out_bytes);
    const BoardPlan p = board_plan(net, B);
    const int32_t info[8] = {p.R, p.NT, p.ctas, p.last, stage < nl ? stage + 1 : nl, m->npass, p.smem, 0};
    memcpy(h_info, info, sizeof(info));
    float *o = reinterpret_cast<float *>(d_out);
    BoardIO io = board_io(m, B);
    if (obs) io.obs = d_in;
    else { io.latent_base = d_in; io.action = d_action; }
    if (stage < nl) {
        // the program cut after layer `stage`, whose output is the only latent written; no head runs
        net.nlayers = stage + 1;
        for (int L = 0; L <= stage; ++L) net.layer_flags[L] &= ~(BF_WRITE_LATENT | BF_HOOK_REWARD | BF_HOOK_VALPOL);
        net.layer_flags[stage] |= BF_WRITE_LATENT;
        io.latent_out = o;
        return board_launch(net, io, st);
    }
    // the whole program with the raw logits, then without them (the scalars alone, as a search asks for them)
    LZ_CUDA_CHECK(cudaMemsetAsync(d_out, 0, nfl * sizeof(float), st));
    float *rl = o, *vl = rl + (size_t)B * K, *pl = vl + (size_t)B * K, *r = pl + (size_t)B * A, *v = r + B;
    float *pl2 = v + B, *r2 = pl2 + (size_t)B * A, *v2 = r2 + B;
    io.policy_logits = pl; io.value_logits = vl; io.value = v;
    if (!obs) { io.reward_logits = rl; io.reward = r; }
    int rc = board_launch(net, io, st);
    if (rc) return rc;
    io.policy_logits = pl2; io.value_logits = nullptr; io.value = v2;
    io.reward_logits = nullptr; io.reward = obs ? nullptr : r2;
    return board_launch(net, io, st);
}

}  // namespace lz
