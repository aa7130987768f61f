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

#include "board_tc.cuh"
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

// row m of a CTA's padded grid -> (root slot r, pixel p); false for pad rows and absent roots
__device__ __forceinline__ bool board_row(int m, int nvalid, int H, int W, int &r, int &p)
{
    const int pitch = W + 1, rpr = (H + 1) * pitch;
    r = m / rpr;
    const int q = m - r * rpr, y = q / pitch, x = q - y * pitch;
    p = y * W + x;
    return r < nvalid && y < H && x < W;
}

// one head for the CTA's roots from the fp32 latent rows in skip: 1x1 conv + BN + ReLU -> feat, FC1 + BN1d + ReLU -> hid, FC2 ->
// logits (one warp per root), the categorical heads' scalar through categorical_to_scalar
template <int C>
__device__ void board_head(const BoardNet &net, const BoardHead &hd, const float *skip, float *feat, float *hidb, float *lbuf, int nvalid,
                           int root0, float *glog, float *gscal, bool categorical)
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
        for (int k = lane; k < K; k += 32) {
            const float *w = hd.fc2 + (size_t)k * hid;
            float a = 0.0f;
            for (int j = 0; j < hid; ++j) a = fmaf(__ldg(w + j), hv[j], a);
            a += __ldg(hd.b2 + k);
            lrow[k] = a;
            if (glog) glog[(size_t)b * K + k] = a;
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
            if (board_row(m, nvalid, H, W, r, p)) {
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
            rinfo[t][h] = board_row(t * 64 + 16 * warp + (lane >> 2) + 8 * h, nvalid, H, W, r, p) ? ((r << 8) | p) : -1;
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
                if (ab && info >= 0) abr = net.abias + (size_t)min(max(io.action[b], 0), net.A - 1) * C * P + p;
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
                board_head<C>(net, net.head[0], skip, feat, hidb, lbuf, nvalid, root0, io.reward_logits, io.reward, true);
        }
        if (flags & BF_HOOK_VALPOL) {
            if (io.value_logits || io.value)
                board_head<C>(net, net.head[1], skip, feat, hidb, lbuf, nvalid, root0, io.value_logits, io.value, true);
            if (io.policy_logits)
                board_head<C>(net, net.head[2], skip, feat, hidb, lbuf, nvalid, root0, io.policy_logits, nullptr, false);
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
    int e = 0;
    if (mx > 0.0f) frexpf(mx, &e);
    const float scale = ldexpf(1.0f, 13 - e);       // largest |w| lands in [4096, 8192): the lo parts stay in fp16's normal range
    __half *h = reinterpret_cast<__half *>(dst);
    const size_t tap_halves = (size_t)cin_pad * C * 2;
    for (int t = 0; t < 9; ++t)
        for (int co = 0; co < C; ++co)
            for (int ci = 0; ci < cin_pad; ++ci) {
                const float v = ci < cin_used ? w[((size_t)co * cin_total + ci) * 9 + t] * scale : 0.0f;
                const __half hi = __float2half_rn(v), lo = __float2half_rn(v - __half2float(hi));
                const size_t off = t * tap_halves + ((size_t)(ci / 8) * 2 * C + co) * 8 + ci % 8;
                h[off] = hi;
                h[off + (size_t)C * 8] = lo;
            }
    return scale;
}

}  // namespace lz
