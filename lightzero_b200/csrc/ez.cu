// ez.cu -- EfficientZero value-prefix head for sm_90a: LSTM step + BatchNorm1d/ReLU/MLP/categorical expectation.
//
// k_ez_lstm: gates[B][4H] = [feat | h_in] (B x (nin+H)) * wcat ((nin+H) x 4H) + bias as a tiled fp32 GEMM over ALL roots
// (the weights, 8.9 MB at nin = 576 / H = 512, are read once per 64-row tile instead of once per root), with the LSTM cell
// update fused into the epilogue: the weight columns are ordered unit-major / gate-minor so that the 4 x 4 register tile
// of a thread holds (i, f, g, o) of one hidden unit for 4 roots.  torch.nn.LSTM gate order i, f, g, o; c' = sig(f) c +
// sig(i) tanh(g); h' = sig(o) tanh(c').
// k_ez_head: per root relu(bn(h')) (h' alone for EfficientZeroModelMLP) -> Linear(H, hid) + BN + ReLU -> Linear(hid, K) -> softmax expectation -> h^-1.
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "ez.cuh"
#include "model.cuh"
#include "tc_ptx.cuh"

namespace lz {

constexpr int kGM = 64, kGN = 32, kGK = 16;      // 64 roots x 32 gate columns (= 8 hidden units) per CTA: 64 x ceil(B/64) CTAs
constexpr int kGThreads = 128;                   // thread = 4 roots x 4 gates of one hidden unit

__global__ void __launch_bounds__(kGThreads) k_ez_lstm(EzNet net, EzIO io)
{
    __shared__ float As[kGK][kGM + 4];
    __shared__ float Bs[kGK][kGN];
    const int tid = threadIdx.x, tx = tid & 7, ty = tid >> 3;          // tx: hidden unit within the tile, ty: 4-row group
    const int n0 = blockIdx.x * kGN, m0 = blockIdx.y * kGM;
    const int H = net.H, nin = net.nin, KT = nin + H, N = 4 * H;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
    // A-tile loader: thread -> (row = tid / 2, 8 consecutive k); B-tile loader: thread -> (k = tid / 8, 4 consecutive n)
    const int ar = tid >> 1, ak = (tid & 1) * 8;
    const int arow = m0 + ar;
    const bool arow_on = arow < io.B;
    const float *hsrc = io.h_base + (arow_on && io.ix ? (size_t)io.ix[arow] * io.slot_stride : 0) + (size_t)(arow_on ? arow : 0) * H;
    const float *fsrc = io.feat + (size_t)(arow_on ? arow : 0) * nin;
    const int bk = tid >> 3, bn = (tid & 7) * 4;
    float4 a4[2];
    float4 b4;
    auto fetch = [&](int k0) {       // global -> registers (in flight while the previous tile is being multiplied)
#pragma unroll
        for (int v = 0; v < 2; ++v) {        // nin and H are multiples of 4, so a 16-byte load never straddles feat | h
            const int k = k0 + ak + 4 * v;
            a4[v] = (arow_on && k < KT) ? *reinterpret_cast<const float4 *>(k < nin ? fsrc + k : hsrc + (k - nin)) : make_float4(0, 0, 0, 0);
        }
        b4 = (k0 + bk < KT) ? __ldg(reinterpret_cast<const float4 *>(net.wcat + (size_t)(k0 + bk) * N + n0 + bn)) : make_float4(0, 0, 0, 0);
    };
    fetch(0);
    for (int k0 = 0; k0 < KT; k0 += kGK) {
        __syncthreads();
#pragma unroll
        for (int v = 0; v < 2; ++v) {
            As[ak + 4 * v + 0][ar] = a4[v].x; As[ak + 4 * v + 1][ar] = a4[v].y;
            As[ak + 4 * v + 2][ar] = a4[v].z; As[ak + 4 * v + 3][ar] = a4[v].w;
        }
        *reinterpret_cast<float4 *>(&Bs[bk][bn]) = b4;
        __syncthreads();
        if (k0 + kGK < KT) fetch(k0 + kGK);
#pragma unroll
        for (int k = 0; k < kGK; ++k) {
            const float4 a = *reinterpret_cast<const float4 *>(&As[k][ty * 4]);
            const float4 b = *reinterpret_cast<const float4 *>(&Bs[k][tx * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
    }
    // epilogue: this thread owns hidden unit `unit` for rows m0 + ty*4 .. +3
    const int unit = (n0 >> 2) + tx;
    const float4 bias = *reinterpret_cast<const float4 *>(net.bias + n0 + tx * 4);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int b = m0 + ty * 4 + i;
        if (b >= io.B) continue;
        const float gi = acc[i][0] + bias.x, gf = acc[i][1] + bias.y, gg = acc[i][2] + bias.z, go = acc[i][3] + bias.w;
        const float c_in = io.c_base[(io.ix ? (size_t)io.ix[b] * io.slot_stride : 0) + (size_t)b * H + unit];
        const float si = 1.0f / (1.0f + expf(-gi)), sf = 1.0f / (1.0f + expf(-gf)), so = 1.0f / (1.0f + expf(-go));
        const float c_new = sf * c_in + si * tanhf(gg);
        const float h_new = so * tanhf(c_new);
        const bool reset = io.is_reset && io.is_reset[b] != 0;
        io.h_tmp[(size_t)b * H + unit] = h_new;
        if (io.h_out) io.h_out[(size_t)b * H + unit] = reset ? 0.0f : h_new;
        if (io.c_out) io.c_out[(size_t)b * H + unit] = reset ? 0.0f : c_new;
    }
}

constexpr int kHR = 2;        // roots per CTA of the head kernel (the FC weights are 64 KB + 77 KB, L2-resident)
constexpr int kHMaxH = 512, kHMaxHid = 32, kHLd = 608;

__global__ void __launch_bounds__(256) k_ez_head(EzNet net, EzIO io)
{
    __shared__ float x[kHR][kHMaxH];
    __shared__ float part[8][kHR][kHMaxHid];
    __shared__ float hidden[kHR][kHMaxHid];
    __shared__ float logits[kHR][kHLd];
    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;   // warp-uniform value: uniform role branches (see net_tc.cu)
    const int r0 = blockIdx.x * kHR, nr = min(kHR, io.B - r0);
    const int H = net.H, hid = net.hid, K = net.K;
    for (int i = tid; i < kHR * H; i += 256) {                       // norm_value_prefix + ReLU (efficientzero_model.py:565-566)
        const int r = i / H, u = i - r * H;
        float v = 0.0f;
        if (r < nr) {
            v = io.h_tmp[(size_t)(r0 + r) * H + u];
            if (!net.no_vp_norm) v = fmaxf(fmaf(v, net.vp_s[u], net.vp_t[u]), 0.0f);
        }
        x[r][u] = v;
    }
    __syncthreads();
    {   // Linear(H -> hid): warp w sums its eighth of the inputs, lane = hidden unit; 16 weight rows in flight per batch
        const int per = (H + 7) / 8, i0 = warp * per, i1 = min(H, i0 + per);
        float a[kHR];
#pragma unroll
        for (int r = 0; r < kHR; ++r) a[r] = 0.0f;
        const bool lane_on = lane < hid;
        for (int i = i0; i < i1; i += 16) {
            float w[16];
#pragma unroll
            for (int u = 0; u < 16; ++u) w[u] = (lane_on && i + u < i1) ? __ldg(net.fc1 + (size_t)(i + u) * hid + lane) : 0.0f;
#pragma unroll
            for (int u = 0; u < 16; ++u) {
                const int ii = min(i + u, H - 1);
#pragma unroll
                for (int r = 0; r < kHR; ++r) a[r] = fmaf(x[r][ii], w[u], a[r]);
            }
        }
#pragma unroll
        for (int r = 0; r < kHR; ++r) part[warp][r][lane] = a[r];
    }
    __syncthreads();
    if (tid < kHR * 32) {
        const int r = tid >> 5, j = tid & 31;      // kHR roots x 32 hidden units
        float v = 0.0f;
#pragma unroll
        for (int w = 0; w < 8; ++w) v += part[w][r][j];
        hidden[r][j] = j < hid ? fmaxf(fmaf(v, net.s2[j], net.t2[j]), 0.0f) : 0.0f;
    }
    __syncthreads();
    for (int k = tid; k < K; k += 256) {           // Linear(hid -> K)
        float o[kHR];
        const float bias = __ldg(net.b2 + k);
#pragma unroll
        for (int r = 0; r < kHR; ++r) o[r] = bias;
        float w[kHMaxHid];
#pragma unroll
        for (int j = 0; j < kHMaxHid; ++j) w[j] = j < hid ? __ldg(net.fc2 + (size_t)j * K + k) : 0.0f;     // all rows in flight
#pragma unroll
        for (int j = 0; j < kHMaxHid; ++j) {
#pragma unroll
            for (int r = 0; r < kHR; ++r) o[r] = fmaf(hidden[r][j], w[j], o[r]);
        }
#pragma unroll
        for (int r = 0; r < kHR; ++r) logits[r][k] = o[r];
    }
    __syncthreads();
    if (warp < nr) {
        const int b = r0 + warp;
        const float vp = categorical_to_scalar(logits[warp], K, net.support_min, net.support_step, lane);
        if (lane == 0 && io.value_prefix) io.value_prefix[b] = vp;
        if (io.vp_logits)
            for (int k = lane; k < K; k += 32) io.vp_logits[(size_t)b * K + k] = logits[warp][k];
    }
}

// ---------------------------------------------------------------------------------------------- wgmma LSTM step
// gates = [feat | h] * W as a wgmma GEMM with fp32 accuracy ("3xFP16": A_hi*W_hi + A_hi*W_lo + A_lo*W_hi, fp32 accumulation in
// registers).  CTA tile: 128 roots x 64 gate columns (16 hidden units), K = nin + H in chunks of 64 through a 3-stage ring.  Two
// warpgroups: each gathers the fp32 A rows of every other chunk (features, then the leaf parent's h through ix), splits them to fp16
// hi / lo into the wgmma K-major layout [k-group][row][8 halves], issues the MMAs of its 64 rows of every chunk and runs the
// epilogue (LSTM cell update, reset) from its accumulators.  Warp 8 lane 0 bulk-copies the pre-split weight chunks.
constexpr int kTM = 128, kTN = 64, kTK = 64, kTStages = 3;
constexpr int kTAPart = 8 * kTM * 16;            // one hi or lo part of an A stage: [8 k-groups][128 rows][16 B] = 16 KB
constexpr int kTWPart = 8 * kTN * 16;            // one hi or lo part of a W stage: 8 KB
constexpr int kTStageBytes = 2 * kTAPart + 2 * kTWPart;     // 48 KB
constexpr int kTSmem = kTStages * kTStageBytes + 256;
constexpr int kTThreads = 256 + 32;

struct EzTcBars {
    uint64_t full_a[kTStages], full_w[kTStages], empty[kTStages];
};

__global__ void __launch_bounds__(kTThreads, 1) k_ez_lstm_tc(EzNet net, EzIO io)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    EzTcBars *bars = reinterpret_cast<EzTcBars *>(smem + kTStages * kTStageBytes);
    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;   // warp-uniform value: uniform role branches
    const int nt = blockIdx.x, m0 = blockIdx.y * kTM;
    const int H = net.H, nin = net.nin, KT = nin + H, nchunks = KT / kTK;

    if (tid == 0) {
        for (int i = 0; i < kTStages; ++i) { mbar_init(&bars->full_a[i], 128); mbar_init(&bars->full_w[i], 1); mbar_init(&bars->empty[i], 8); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            const unsigned char *src = net.wtc + (size_t)nt * nchunks * (2 * kTWPart);
            for (int c = 0; c < nchunks; ++c) {
                const int st = c % kTStages;
                if (c >= kTStages) mbar_wait(&bars->empty[st], ((c / kTStages) - 1) & 1);
                mbar_expect_tx(&bars->full_w[st], 2 * kTWPart);
                bulk_g2s(smem + st * kTStageBytes + 2 * kTAPart, src + (size_t)c * (2 * kTWPart), 2 * kTWPart, &bars->full_w[st]);
            }
        }
        return;
    }
    // ---- A production: warpgroup grp converts chunks grp, grp + 2, ...  Per pass a warp covers 8 rows x 8 k-groups: lane -> (row =
    // lane % 8, k-groups lane / 8 and lane / 8 + 4), so one load instruction touches 8 lines (one per row) instead of 32 and each
    // quarter-warp stores 8 consecutive rows of one k-group plane (conflict-free).
    const int grp = warp >> 2, tg = tid & 127;
    const int pw = tg >> 5, pl = tg & 31, prow0 = pw * 8 + (pl & 7), pkg = pl >> 3;
    const float *fsrc[4], *hsrc[4];
    bool pon[4];
#pragma unroll
    for (int ps = 0; ps < 4; ++ps) {
        const int bb = m0 + ps * 32 + prow0;
        pon[ps] = bb < io.B;
        fsrc[ps] = io.feat + (size_t)(pon[ps] ? bb : 0) * nin;
        hsrc[ps] = io.h_base + (pon[ps] && io.ix ? (size_t)io.ix[bb] * io.slot_stride : 0) + (size_t)(pon[ps] ? bb : 0) * H;
    }
    auto produce = [&](int c) {
        const int st = c % kTStages;
        const int k0 = c * kTK;                                             // nin is a multiple of 64: a chunk never straddles feat | h
        float4 v[16];
#pragma unroll
        for (int ps = 0; ps < 4; ++ps) {
            const float *src = (k0 < nin ? fsrc[ps] + k0 : hsrc[ps] + (k0 - nin)) + pkg * 8;
#pragma unroll
            for (int u = 0; u < 4; ++u)      // u: 0,1 = k-group pkg, 2,3 = k-group pkg + 4
                v[ps * 4 + u] = pon[ps] ? *reinterpret_cast<const float4 *>(src + (u >> 1) * 32 + (u & 1) * 4) : make_float4(0, 0, 0, 0);
        }
        if (c >= kTStages) mbar_wait(&bars->empty[st], ((c / kTStages) - 1) & 1);
#pragma unroll
        for (int ps = 0; ps < 4; ++ps) {
            unsigned char *a_hi = smem + st * kTStageBytes + (ps * 32 + prow0) * 16;
#pragma unroll
            for (int h2 = 0; h2 < 2; ++h2) {
                const float4 x = v[ps * 4 + 2 * h2], y = v[ps * 4 + 2 * h2 + 1];
                const float f[8] = {x.x, x.y, x.z, x.w, y.x, y.y, y.z, y.w};
                const int kg = pkg + 4 * h2;
                store_split8(a_hi + kg * (kTM * 16), a_hi + kTAPart + kg * (kTM * 16), f);
            }
        }
        fence_proxy_async();
        mbar_arrive(&bars->full_a[st]);
    };
    for (int c = grp; c < kTStages && c < nchunks; c += 2) produce(c);
    // ---- MMAs of this warpgroup's 64 rows; a chunk's slot is refilled (A by its producing warpgroup) once both have read it
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.0f;
    for (int c = 0; c < nchunks; ++c) {
        const int st = c % kTStages;
        mbar_wait(&bars->full_a[st], (c / kTStages) & 1);
        mbar_wait(&bars->full_w[st], (c / kTStages) & 1);
        const uint32_t a_s = smem_u32(smem + st * kTStageBytes) + grp * 64 * 16, w_s = smem_u32(smem + st * kTStageBytes) + 2 * kTAPart;
        const uint64_t a_hi = make_desc(a_s, (kTM * 16) >> 4, 8), a_lo = make_desc(a_s + kTAPart, (kTM * 16) >> 4, 8);
        const uint64_t w_hi = make_desc(w_s, (kTN * 16) >> 4, 8), w_lo = make_desc(w_s + kTWPart, (kTN * 16) >> 4, 8);
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < kTK / 16; ++ks) {
            const uint64_t ao = (uint64_t)(ks * 2 * kTM * 16 >> 4), wo = (uint64_t)(ks * 2 * kTN * 16 >> 4);
            wgmma_n64(acc, a_hi + ao, w_hi + wo);
            wgmma_n64(acc, a_hi + ao, w_lo + wo);
            wgmma_n64(acc, a_lo + ao, w_hi + wo);
        }
        wg_commit();
        wg_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars->empty[st]);
        if (c + kTStages < nchunks && ((c + kTStages) & 1) == grp) produce(c + kTStages);
    }
    // ---- epilogue from the fragment: columns 8 j + 2 (lane % 4) + {0, 1} are gates (i, f) (even lane % 4) or (g, o) (odd) of hidden
    // unit 2 j + (lane % 4) / 2; lane pairs swap one row's half so the even lane updates its first row, the odd lane its second.
    // sigmoid / tanh through __expf + __fdividef: abs error ~1e-6 on values in (-1, 1).
    {
        const bool odd = (lane & 1) != 0;
        const int row = grp * 64 + 16 * (warp & 3) + (lane >> 2) + (odd ? 8 : 0), b = m0 + row;
        const bool on = b < io.B;
        const size_t hoff = (on && io.ix ? (size_t)io.ix[b] * io.slot_stride : 0) + (size_t)(on ? b : 0) * H;
        const float inv = net.wtc_inv_scale;
        const float *c_in = io.c_base + hoff;
        const bool reset = on && io.is_reset && io.is_reset[b] != 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float s0 = odd ? acc[4 * j] : acc[4 * j + 2], s1 = odd ? acc[4 * j + 1] : acc[4 * j + 3];
            const float r0 = __shfl_xor_sync(0xffffffffu, s0, 1), r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
            const float ai = odd ? r0 : acc[4 * j], af = odd ? r1 : acc[4 * j + 1];
            const float ag = odd ? acc[4 * j + 2] : r0, ao = odd ? acc[4 * j + 3] : r1;
            if (!on) continue;
            const int u = nt * 16 + 2 * j + ((lane & 3) >> 1);
            const float4 bias = *reinterpret_cast<const float4 *>(net.bias + (size_t)u * 4);
            const float gi = fmaf(ai, inv, bias.x), gf = fmaf(af, inv, bias.y);
            const float gg = fmaf(ag, inv, bias.z), go = fmaf(ao, inv, bias.w);
            const float si = __fdividef(1.0f, 1.0f + __expf(-gi)), sf = __fdividef(1.0f, 1.0f + __expf(-gf));
            const float so = __fdividef(1.0f, 1.0f + __expf(-go));
            const float tg_ = 1.0f - __fdividef(2.0f, __expf(2.0f * gg) + 1.0f);
            const float cn = sf * c_in[u] + si * tg_;
            const float hn = so * (1.0f - __fdividef(2.0f, __expf(2.0f * cn) + 1.0f));
            io.h_tmp[(size_t)b * H + u] = hn;
            if (io.h_out) io.h_out[(size_t)b * H + u] = reset ? 0.0f : hn;
            if (io.c_out) io.c_out[(size_t)b * H + u] = reset ? 0.0f : cn;
        }
    }
}

bool ez_tc_shape(int nin, int H) { return (nin % kTK) == 0 && (H % kTK) == 0; }

size_t ez_wtc_bytes(int nin, int H) { return (size_t)(4 * H / kTN) * ((nin + H) / kTK) * (2 * kTWPart); }

// W_ih [4H][nin], W_hh [4H][H] (torch gate order i, f, g, o along dim 0) -> per (n-tile, k-chunk) [hi | lo] blocks of
// [k-group][n][8 halves]; column n = unit * 4 + gate as in the fp32 path.  Returns the power-of-two scale applied.
float ez_pack_wtc(const float *w_ih, const float *w_hh, int nin, int H, unsigned char *dst)
{
    const int KT = nin + H, N = 4 * H, nchunks = KT / kTK;
    float mx = 0.0f;
    for (size_t i = 0; i < (size_t)N * nin; ++i) mx = std::max(mx, fabsf(w_ih[i]));
    for (size_t i = 0; i < (size_t)N * H; ++i) mx = std::max(mx, fabsf(w_hh[i]));
    const float scale = pow2_scale(mx);
    __half *h = reinterpret_cast<__half *>(dst);
    for (int n = 0; n < N; ++n) {
        const int unit = n >> 2, gate = n & 3, row = gate * H + unit, nt = n / kTN, nn = n % kTN;
        for (int k = 0; k < KT; ++k) {
            const float w = (k < nin ? w_ih[(size_t)row * nin + k] : w_hh[(size_t)row * H + (k - nin)]) * scale;
            const int c = k / kTK, kk = k % kTK;
            const size_t blk = ((size_t)nt * nchunks + c) * (2 * kTWPart / 2);      // in halves
            const size_t off = blk + ((size_t)(kk / 8) * kTN + nn) * 8 + (kk % 8);
            split_hi_lo(w, h[off], h[off + kTWPart / 2]);
        }
    }
    return scale;
}

int ez_prepare_launch()
{
    LZ_CUDA_CHECK(cudaFuncSetAttribute(k_ez_lstm_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, kTSmem));
    return LZ_OK;
}

int ez_launch(const EzNet &net, const EzIO &io, cudaStream_t s)
{
    LZ_REQUIRE(net.H <= kHMaxH && net.hid <= kHMaxHid && net.K <= kHLd && (net.H % 8) == 0, LZ_EINVAL,
               "ez_launch: unsupported LSTM / head size (H=%d hid=%d K=%d)", net.H, net.hid, net.K);
    const bool tc_ok = net.wtc && ez_tc_shape(net.nin, net.H);
    if (tc_ok) {
        dim3 grid(4 * net.H / kTN, (io.B + kTM - 1) / kTM);
        k_ez_lstm_tc<<<grid, kTThreads, kTSmem, s>>>(net, io);
    } else {
        dim3 grid(4 * net.H / kGN, (io.B + kGM - 1) / kGM);
        k_ez_lstm<<<grid, kGThreads, 0, s>>>(net, io);
    }
    LZ_KERNEL_CHECK();
    k_ez_head<<<(io.B + kHR - 1) / kHR, 256, 0, s>>>(net, io);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

// ---- the value-prefix head of a model (lz_model::ez) ------------------------------------------------------------------------
// Tables of nn.LSTM(nin -> H) (one step) and fc_reward_head (Linear(H -> hid) + BN1d + ReLU + Linear(hid -> K)), preceded by
// norm_value_prefix (BN1d + ReLU, vp_norm) in the conv model (efficientzero_model.py:511-525, 556-569) and by nothing in
// EfficientZeroModelMLP (efficientzero_model_mlp.py:416-429, 466-467): fp32 tables in m->ez.d_tables, the tensor-core copy of
// the LSTM weights in m->ez.d_wtc.
int ez_finalize(lz_model *m, int nin, int hid, bool vp_norm)
{
    const std::string D = "dynamics_network.";
    const int K = m->K, H = m->lstm_hidden;
    auto Wih = find_tensor(m, D + "lstm.weight_ih_l0", (size_t)4 * H * nin), Whh = find_tensor(m, D + "lstm.weight_hh_l0", (size_t)4 * H * H);
    auto bih = find_tensor(m, D + "lstm.bias_ih_l0", (size_t)4 * H), bhh = find_tensor(m, D + "lstm.bias_hh_l0", (size_t)4 * H);
    auto W0 = find_tensor(m, D + "fc_reward_head.0.weight", (size_t)hid * H), B0 = find_tensor(m, D + "fc_reward_head.0.bias", hid);
    auto W3 = find_tensor(m, D + "fc_reward_head.3.weight", (size_t)K * hid), B3 = find_tensor(m, D + "fc_reward_head.3.bias", K);
    std::vector<float> vs, vt, s2, t2;
    if (!Wih || !Whh || !bih || !bhh || !W0 || !B0 || !W3 || !B3 || (vp_norm && !fold_bn(m, D + "norm_value_prefix", H, vs, vt)) ||
        !fold_bn(m, D + "fc_reward_head.1", hid, s2, t2))
        return LZ_EINVAL;
    for (int j = 0; j < hid; ++j) t2[j] += s2[j] * (*B0)[j];
    // torch.nn.LSTM stacks the gates (i, f, g, o) along dim 0; column n = unit * 4 + gate
    std::vector<float> wcat((size_t)(nin + H) * 4 * H), bias((size_t)4 * H), fc1((size_t)H * hid), fc2((size_t)hid * K);
    for (int g = 0; g < 4; ++g)
        for (int u = 0; u < H; ++u) {
            const size_t row = (size_t)g * H + u, col = (size_t)u * 4 + g;
            for (int k = 0; k < nin; ++k) wcat[(size_t)k * 4 * H + col] = (*Wih)[row * nin + k];
            for (int k = 0; k < H; ++k) wcat[(size_t)(nin + k) * 4 * H + col] = (*Whh)[row * H + k];
            bias[col] = (*bih)[row] + (*bhh)[row];
        }
    for (int j = 0; j < hid; ++j)
        for (int i = 0; i < H; ++i) fc1[(size_t)i * hid + j] = (*W0)[(size_t)j * H + i];
    for (int k = 0; k < K; ++k)
        for (int j = 0; j < hid; ++j) fc2[(size_t)j * K + k] = (*W3)[(size_t)k * hid + j];
    EzHead &z = m->ez;
    float scale = 1.0f;
    dev_free(z.d_wtc);
    z.d_wtc = nullptr;
    if (ez_tc_shape(nin, H)) {   // tensor-core copy of the LSTM weights (fp16 hi / lo, power-of-two scaled); other shapes (e.g. 8
                                 // reward-head channels: nin = 288) run the fp32 k_ez_lstm
        std::vector<unsigned char> wtc(ez_wtc_bytes(nin, H));
        scale = ez_pack_wtc(Wih->data(), Whh->data(), nin, H, wtc.data());
        int rc = upload(&z.d_wtc, wtc.data(), wtc.size());
        if (rc != LZ_OK) return rc;
    }
    TablePacker P;
    const size_t o_wcat = P.add(wcat), o_bias = P.add(bias), o_vps = P.add(vs), o_vpt = P.add(vt), o_fc1 = P.add(fc1);
    const size_t o_s2 = P.add(s2), o_t2 = P.add(t2), o_fc2 = P.add(fc2), o_b2 = P.add(*B3);
    int rc = upload(&z.d_tables, P.host.data(), P.host.size() * sizeof(float));
    if (rc != LZ_OK) return rc;
    const float *base = z.d_tables;
    EzNet &e = z.net;
    memset(&e, 0, sizeof(e));
    e.wcat = base + o_wcat; e.bias = base + o_bias; e.vp_s = base + o_vps; e.vp_t = base + o_vpt;
    e.fc1 = base + o_fc1; e.s2 = base + o_s2; e.t2 = base + o_t2; e.fc2 = base + o_fc2; e.b2 = base + o_b2;
    e.nin = nin; e.H = H; e.hid = hid; e.K = K; e.no_vp_norm = vp_norm ? 0 : 1;
    e.support_min = m->support_min; e.support_step = m->support_step;
    e.wtc = z.d_wtc; e.wtc_inv_scale = 1.0f / scale;
    return ez_prepare_launch();
}

// the LSTM input and hidden-state scratch of B roots
int ez_reserve(lz_model *m, int B)
{
    EzHead &z = m->ez;
    if (B <= z.B) return LZ_OK;
    ++m->generation;
    dev_free(z.feat); dev_free(z.htmp);
    z.feat = z.htmp = nullptr;
    int rc = dev_alloc(&z.feat, (size_t)B * z.net.nin);
    if (rc == LZ_OK) rc = dev_alloc(&z.htmp, (size_t)B * m->lstm_hidden);
    if (rc != LZ_OK) return rc;
    z.B = B;
    return LZ_OK;
}

// the head on the LSTM input features in m->ez.feat
int ez_tail(lz_model *m, const RecIO &io, cudaStream_t s)
{
    EzIO e;
    memset(&e, 0, sizeof(e));
    e.B = io.B; e.feat = m->ez.feat; e.h_base = io.h_base; e.c_base = io.c_base; e.ix = io.ix; e.slot_stride = io.hslot_stride;
    e.h_out = io.h_out; e.c_out = io.c_out; e.is_reset = io.is_reset; e.h_tmp = m->ez.htmp;
    e.value_prefix = io.reward; e.vp_logits = io.reward_logits;
    return ez_launch(m->ez.net, e, s);
}

}  // namespace lz
