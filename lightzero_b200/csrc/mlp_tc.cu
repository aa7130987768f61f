// mlp_tc.cu -- tensor-core (wgmma) network of EfficientZeroModelMLP (lzero/model/efficientzero_model_mlp.py:150-300) and
// MuZeroModelMLP (lzero/model/muzero_model_mlp.py:21-442): representation Linear(obs -> L) + BN + GELU(tanh) + Linear(L -> L) +
// LayerNorm (common.py:790-850), the dynamics MLPs over [latent | one-hot action] (fc_dynamics, or fc_dynamics_1 + latent ->
// fc_dynamics_2 with res_connection_in_dynamics, efficientzero_model_mlp.py:440-468, muzero_model_mlp.py:428-438) and the
// prediction MLPs (common.py:1218-1292).  EfficientZeroModelMLP's LSTM value-prefix head that follows the dynamics network runs
// in ez.cu on the LSTM input this kernel writes; MuZeroModelMLP's categorical reward head (fc_reward_head, muzero_model_mlp.py:440)
// runs in the recurrent program itself, the same way as the value head.
//
// One launch runs a whole layer program (initial_inference, or the dense part of recurrent_inference) for all roots; a CTA of one
// warpgroup owns up to 64 roots, the rows of one m64 wgmma tile.  Arithmetic as net_tc.cu / board_tc.cu: 3xFP16 (A_hi B_hi +
// A_hi B_lo + A_lo B_hi, fp32 accumulators in registers; one pass in tc1), weights pre-split on the host and pre-scaled by a power
// of two that is folded into the BN scale.  Activations stay in shared memory in the wgmma K-major no-swizzle layout
// [k-group of 8 features][64 rows][8 halves] (hi plane, then lo plane) in two L-wide slots and one 32-wide buffer (head hidden
// layer, or the current 32-feature chunk of the observation, which is streamed from global memory).  Weights stream in chunks of
// 32 inputs through a ring of stages (cp.async.bulk, mbarrier complete_tx), refilled by thread 0 as soon as the MMAs have read a
// stage.  Every layer accumulates all of its outputs (N <= L <= 256: <= 128 fp32 registers per thread) before its epilogue runs
// straight from the fragments: folded BN / bias, the one-hot action as a gathered fp32 weight row, ReLU or GELU, the residual
// from the fp32 input latent, LayerNorm (a row lives in one lane quad: two quad-shuffle reductions), then the fp16 hi / lo
// rewrite of the next layer's operand and the fp32 outputs.  The last Linear of each head is cut into pieces of <= L outputs
// (K = 32 inputs) that run the same way; the value (and reward) head's softmax expectation is folded online across its pieces.
#include <cuda_fp16.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "model.cuh"
#include "tc_ptx.cuh"

namespace lz {

constexpr int kMezThreads = 128;
constexpr int kMezKgBytes = kMezRows * 16;                 // one k-group plane of 64 rows: 1 KB
constexpr int kMezHidBytes = 2 * 4 * kMezKgBytes;          // 32-wide buffer, hi | lo: 8 KB
constexpr int kMezSmemMax = 227 * 1024;

__host__ __device__ inline int mez_slot_part(int L) { return (L / 8) * kMezKgBytes; }    // hi (or lo) plane of an L-wide slot
__host__ __device__ inline int mez_stage_bytes(int L) { return 128 * L; }               // 32 inputs x <= L outputs, hi | lo

struct MezSmem {
    int slot1, hid, ring, bars, total;
};

__host__ __device__ inline MezSmem mez_smem(int L, int stages)
{
    MezSmem s;
    s.slot1 = 2 * mez_slot_part(L);
    s.hid = 2 * s.slot1;
    s.ring = s.hid + kMezHidBytes;
    s.bars = s.ring + stages * mez_stage_bytes(L);
    s.total = s.bars + stages * 8;
    return s;
}

__device__ __forceinline__ float mez_gelu(float x)
{
    const float k0 = 0.7978845608028654f, k1 = 0.044715f;      // sqrt(2/pi), torch.nn.GELU(approximate='tanh')
    return 0.5f * x * (1.0f + tanhf(k0 * (x + k1 * x * x * x)));
}

// The MMAs of one 32-input chunk: 2 k-steps, W n32 column blocks (as n64 pairs, an odd one as n32), NP passes; straight-line so
// that no branch separates the wgmma of a commit group.  An n64 fragment is the two n32 fragments of its columns back to back.
template <int NC, int W, int NP>
__device__ __forceinline__ void mez_mma(float (&acc)[NC * 16], uint64_t a0, uint64_t b0, uint32_t a_kstep, uint32_t a_lo,
                                        uint32_t b_kstep, uint32_t b_lo)
{
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
        const uint64_t a = a0 + ks * a_kstep, bk = b0 + ks * b_kstep;
#pragma unroll
        for (int p = 0; p < W / 2; ++p) {
            float(&d)[32] = *reinterpret_cast<float(*)[32]>(&acc[32 * p]);
            const uint64_t b = bk + 64 * p;                 // 64 weight rows of 16 B
            wgmma_n64(d, a, b);
            if constexpr (NP == 3) {
                wgmma_n64(d, a, b + b_lo);
                wgmma_n64(d, a + a_lo, b);
            }
        }
        if constexpr (W % 2 == 1) {
            float(&d)[16] = *reinterpret_cast<float(*)[16]>(&acc[16 * (W - 1)]);
            const uint64_t b = bk + 32 * (W - 1);
            wgmma_n32(d, a, b);
            if constexpr (NP == 3) {
                wgmma_n32(d, a, b + b_lo);
                wgmma_n32(d, a + a_lo, b);
            }
        }
    }
}

template <int NC>
__global__ void __launch_bounds__(kMezThreads, 1) k_mez_tc(MezNet net, MezIO io, int R, int kS)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    constexpr int L = 32 * NC;
    const MezSmem S = mez_smem(L, kS);
    unsigned char *ring = smem + S.ring;
    float *part = reinterpret_cast<float *>(smem + S.slot1);    // [NC * 16][128] fp32 partial sums of the observation layer
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + S.bars);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int root0 = blockIdx.x * R, nvalid = min(R, io.B - root0);
    const int sbytes = mez_stage_bytes(L);
    auto sel = [&](int b) { return !io.row_mask || (io.row_mask[b] & 1) == io.row_mask_on; };
    if (io.row_mask) {
        bool any = false;
        for (int m = tid; m < nvalid; m += kMezThreads) any |= sel(root0 + m);
        if (!__syncthreads_or(any)) return;    // no selected row in this CTA: no weights streamed, nothing written
    }

    int il = 0, ic = 0, issued = 0;            // thread 0: the next weight chunk of the program to stream
    auto issue_next = [&]() {
        const uint32_t bytes = 128u * net.layer[il].N;
        uint64_t *bar = &full[issued % kS];
        mbar_expect_tx(bar, bytes);
        bulk_g2s(ring + (issued % kS) * sbytes, net.w + net.layer[il].woff + (size_t)ic * bytes, bytes, bar);
        ++issued;
        if (++ic == net.layer[il].K / 32) { ic = 0; ++il; }
    };
    auto release = [&]() {                     // a stage has been read: it takes the next chunk in program order
        if (tid == 0 && issued < net.nchunks) issue_next();
    };
    if (tid == 0) {
        for (int i = 0; i < kS; ++i) mbar_init(&full[i], 1);
        fence_mbar_init();
        for (int i = 0; i < kS && issued < net.nchunks; ++i) issue_next();
    }

    // rows of this thread's accumulator fragments and their per-root operands
    int brow[2];
    bool on[2];
    const float *zrow[2], *arow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = 16 * warp + (lane >> 2) + 8 * h;
        on[h] = m < nvalid && sel(root0 + m);
        brow[h] = root0 + (on[h] ? m : 0);
        zrow[h] = (io.latent_base && on[h]) ? io.latent_base + (io.ix ? (size_t)io.ix[brow[h]] * io.slot_stride : 0) + (size_t)brow[h] * L : nullptr;
        arow[h] = (io.action && on[h]) ? net.abias + (size_t)min(max(io.action[brow[h]], 0), net.nact - 1) * L : nullptr;
    }

    // ---- input latents (recurrent programs) -> slot 0, fp16 hi / lo
    if (net.layer[0].in == MB_SLOT0) {
        for (int i = tid; i < kMezRows * (L / 8); i += kMezThreads) {
            const int m = i % kMezRows, kg = i / kMezRows;
            float v[8];
            if (m < nvalid && sel(root0 + m)) {
                const int b = root0 + m;
                const float *src = io.latent_base + (io.ix ? (size_t)io.ix[b] * io.slot_stride : 0) + (size_t)b * L + 8 * kg;
                const float4 x = *reinterpret_cast<const float4 *>(src), y = *reinterpret_cast<const float4 *>(src + 4);
                v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w; v[4] = y.x; v[5] = y.y; v[6] = y.z; v[7] = y.w;
            } else {
#pragma unroll
                for (int u = 0; u < 8; ++u) v[u] = 0.0f;
            }
            store_split8(smem + kg * kMezKgBytes + m * 16, smem + mez_slot_part(L) + kg * kMezKgBytes + m * 16, v);
        }
    }
    fence_proxy_async();
    __syncthreads();

    float sm_m[2] = {-INFINITY, -INFINITY}, sm_s[2] = {0.0f, 0.0f}, sm_w[2] = {0.0f, 0.0f};   // value / reward head: online softmax
    int pos = 0;
    for (int l = 0; l < net.nlayers; ++l) {
        const int K = net.layer[l].K, N = net.layer[l].N, in = net.layer[l].in, out = net.layer[l].out;
        const int f = net.layer[l].flags, nch = N / 32, nk = K / 32;
        const bool obs = in == MB_OBS;
        float acc[NC * 16];
#pragma unroll
        for (int i = 0; i < NC * 16; ++i) acc[i] = 0.0f;
        wg_fence_acc(acc);
        const bool narrow = obs || in == MB_HID;              // the 32-wide buffer
        unsigned char *abuf = narrow ? smem + S.hid : smem + (in == MB_SLOT1 ? S.slot1 : 0);
        const uint64_t a_base = make_desc(smem_u32(abuf), kMezKgBytes >> 4, 8);
        const uint32_t a_kstep = (2 * kMezKgBytes) >> 4, a_lo = (narrow ? 4 * kMezKgBytes : mez_slot_part(L)) >> 4;
        const uint32_t b_lo = N, b_kstep = 4 * N;             // 16-B units: N rows; two k-groups of [N hi | N lo] rows
        for (int c = 0; c < nk; ++c, ++pos) {
            uint64_t a0 = a_base;
            if (obs) {      // observation features 32c .. 32c + 31 -> the 32-wide buffer (the previous chunk's MMAs are done)
                const int m = tid % kMezRows, hf = tid / kMezRows;
                float v[16];
#pragma unroll
                for (int u = 0; u < 16; ++u) {
                    const int k = 32 * c + 16 * hf + u;
                    v[u] = (m < nvalid && k < net.obs_dim && sel(root0 + m)) ? io.obs[(size_t)(root0 + m) * net.obs_dim + k] : 0.0f;
                }
#pragma unroll
                for (int g = 0; g < 2; ++g) {
                    unsigned char *d = smem + S.hid + (2 * hf + g) * kMezKgBytes + m * 16;
                    store_split8(d, d + 4 * kMezKgBytes, v + 8 * g);
                }
                fence_proxy_async();
                __syncthreads();
            } else {
                a0 += (uint64_t)((4 * c * kMezKgBytes) >> 4);
            }
            const int st = pos % kS;
            mbar_wait(&full[st], (pos / kS) & 1);
            const uint64_t b0 = make_desc(smem_u32(ring + st * sbytes), (2 * N * 16) >> 4, 8);
            wg_fence();
            if (io.npass == 3) {
                if (nch == NC) mez_mma<NC, NC, 3>(acc, a0, b0, a_kstep, a_lo, b_kstep, b_lo);
                else mez_mma<NC, 1, 3>(acc, a0, b0, a_kstep, a_lo, b_kstep, b_lo);
            } else {
                if (nch == NC) mez_mma<NC, NC, 1>(acc, a0, b0, a_kstep, a_lo, b_kstep, b_lo);
                else mez_mma<NC, 1, 1>(acc, a0, b0, a_kstep, a_lo, b_kstep, b_lo);
            }
            wg_commit();
            if (obs) {
                // each chunk's sums are added into fp32 partials (round to nearest) in the free slot 1: the tensor cores'
                // accumulation truncates, and over the ~270 accumulations of a 2835-wide observation that bias would grow
                // linearly (2e-5 of the latent after the LayerNorm instead of 1e-6)
                wg_wait<0>();
                wg_fence_acc(acc);
#pragma unroll
                for (int i = 0; i < NC * 16; ++i) {
                    const float p = c ? part[i * kMezThreads + tid] : 0.0f;
                    part[i * kMezThreads + tid] = p + acc[i];
                    acc[i] = 0.0f;
                }
                wg_fence_acc(acc);
                __syncthreads();
                release();
            } else if (c > 0) {
                wg_wait<1>();                                 // the previous chunk's MMAs have read their stage: refill it
                __syncthreads();
                release();
            }
        }
        wg_wait<0>();
        wg_fence_acc(acc);
        if (obs) {
#pragma unroll
            for (int i = 0; i < NC * 16; ++i) acc[i] = part[i * kMezThreads + tid];
        }
        __syncthreads();                                      // every MMA of the layer has read its operand: it may be rewritten
        if (!obs) release();

        // ---- epilogue, pass 1 (in place): folded BN / bias, action row, activation, residual
        const float *sc = net.tab + net.layer[l].bn, *sh = sc + N;
#pragma unroll
        for (int j = 0; j < NC; ++j) {
            if (j >= nch) break;
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = 32 * j + 8 * q + 2 * (lane & 3) + e;
                        float v = fmaf(acc[16 * j + 4 * q + 2 * h + e], __ldg(sc + col), __ldg(sh + col));
                        if ((f & MF_ACT) && on[h]) v += __ldg(arow[h] + col);
                        if (f & MF_RELU) v = fmaxf(v, 0.0f);
                        else if (f & MF_GELU) v = mez_gelu(v);
                        if ((f & MF_RES) && on[h]) v += zrow[h][col];
                        acc[16 * j + 4 * q + 2 * h + e] = v;
                    }
        }
        if (f & MF_LN) {     // nn.LayerNorm(L), eps 1e-5, biased variance: a row's L values live in one lane quad
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float s = 0.0f;
#pragma unroll
                for (int j = 0; j < NC; ++j)
#pragma unroll
                    for (int q = 0; q < 4; ++q) s += acc[16 * j + 4 * q + 2 * h] + acc[16 * j + 4 * q + 2 * h + 1];
                s += __shfl_xor_sync(0xffffffffu, s, 1);
                s += __shfl_xor_sync(0xffffffffu, s, 2);
                const float mean = s / (float)L;
                float d2 = 0.0f;
#pragma unroll
                for (int j = 0; j < NC; ++j)
#pragma unroll
                    for (int q = 0; q < 4; ++q)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const float d = acc[16 * j + 4 * q + 2 * h + e] - mean;
                            d2 += d * d;
                        }
                d2 += __shfl_xor_sync(0xffffffffu, d2, 1);
                d2 += __shfl_xor_sync(0xffffffffu, d2, 2);
                const float rstd = rsqrtf(d2 / (float)L + 1e-5f);
#pragma unroll
                for (int j = 0; j < NC; ++j)
#pragma unroll
                    for (int q = 0; q < 4; ++q)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = 32 * j + 8 * q + 2 * (lane & 3) + e;
                            float &v = acc[16 * j + 4 * q + 2 * h + e];
                            v = (v - mean) * rstd * __ldg(net.ln_w + col) + __ldg(net.ln_b + col);
                        }
            }
        }
        if (f & MF_CAT_BEGIN) {
#pragma unroll
            for (int h = 0; h < 2; ++h) { sm_m[h] = -INFINITY; sm_s[h] = 0.0f; sm_w[h] = 0.0f; }
        }

        // ---- pass 2: the fp32 outputs and the next layer's fp16 hi / lo operand
        const bool rew = (f & MF_REWARD) != 0, cat = (f & (MF_VALUE | MF_REWARD)) != 0;   // cat: a categorical head's piece
        const bool head = (f & (MF_VALUE | MF_REWARD | MF_POLICY)) != 0;
        const int ncols = cat ? net.K : net.A, col0 = net.layer[l].col0;
        const int rstride = (cat || !io.policy_stride) ? ncols : io.policy_stride;
        float *lg = rew ? io.reward_logits : (cat ? io.value_logits : io.policy_logits);
        unsigned char *ob = out == MB_NONE ? nullptr : smem + (out == MB_HID ? S.hid : (out == MB_SLOT1 ? S.slot1 : 0));
        const int opart = out == MB_HID ? 4 * kMezKgBytes : mez_slot_part(L);
#pragma unroll
        for (int j = 0; j < NC; ++j) {
            if (j >= nch) break;
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int col = 32 * j + 8 * q + 2 * (lane & 3), m = 16 * warp + (lane >> 2) + 8 * h;
                    float v0 = acc[16 * j + 4 * q + 2 * h], v1 = acc[16 * j + 4 * q + 2 * h + 1];
                    if (on[h]) {
                        const size_t o = (size_t)brow[h] * L + col;
                        if ((f & MF_LATENT) && io.latent_out) *reinterpret_cast<float2 *>(io.latent_out + o) = make_float2(v0, v1);
                        if ((f & MF_LATENT) && io.latent_out2) *reinterpret_cast<float2 *>(io.latent_out2 + o) = make_float2(v0, v1);
                        if ((f & MF_FEAT) && io.feat) *reinterpret_cast<float2 *>(io.feat + o) = make_float2(v0, v1);
                        if (head) {
                            const int k = col0 + col;
                            if (lg && k < ncols) lg[(size_t)brow[h] * rstride + k] = v0;
                            if (lg && k + 1 < ncols) lg[(size_t)brow[h] * rstride + k + 1] = v1;
                            if (cat && k < ncols) softmax_push(sm_m[h], sm_s[h], sm_w[h], v0, support_at(net.support_min, net.support_step, k));
                            if (cat && k + 1 < ncols) softmax_push(sm_m[h], sm_s[h], sm_w[h], v1, support_at(net.support_min, net.support_step, k + 1));
                        }
                    } else {
                        v0 = v1 = 0.0f;
                    }
                    if (ob) {
                        const float c0 = fminf(fmaxf(v0, -65504.0f), 65504.0f), c1 = fminf(fmaxf(v1, -65504.0f), 65504.0f);
                        const __half2 hi = __floats2half2_rn(c0, c1);
                        const float2 back = __half22float2(hi);
                        unsigned char *d = ob + (col >> 3) * kMezKgBytes + m * 16 + (col & 7) * 2;
                        *reinterpret_cast<__half2 *>(d) = hi;
                        *reinterpret_cast<__half2 *>(d + opart) = __floats2half2_rn(c0 - back.x, c1 - back.y);
                    }
                }
        }
        if (f & MF_CAT_END) {      // the quad's partial (max, sum, weighted sum) triples -> softmax . support -> h^-1
            float *sc_out = rew ? io.reward : io.value;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float M = fmaxf(sm_m[h], __shfl_xor_sync(0xffffffffu, sm_m[h], 1));
                M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, 2));
                const float r = sm_m[h] == -INFINITY ? 0.0f : expf(sm_m[h] - M);
                float s = sm_s[h] * r, w = sm_w[h] * r;
                s += __shfl_xor_sync(0xffffffffu, s, 1);
                w += __shfl_xor_sync(0xffffffffu, w, 1);
                s += __shfl_xor_sync(0xffffffffu, s, 2);
                w += __shfl_xor_sync(0xffffffffu, w, 2);
                if (on[h] && (lane & 3) == 0 && sc_out) sc_out[brow[h]] = inverse_scalar_transform(w / s);
            }
        }
        fence_proxy_async();
        __syncthreads();                                      // the layer's output is visible to the next layer's MMAs
    }
}

// ---------------------------------------------------------------------------------------------- host
static int mez_stages(int L)
{
    const int fixed = mez_smem(L, 0).total;
    return std::min(4, (kMezSmemMax - fixed) / (mez_stage_bytes(L) + 8));
}

// Roots per CTA: 64 (one full m64 tile) whenever the batch has them.  Every CTA streams the whole program's weights from L2
// (0.3-2.4 MB in tc3), and that stream, not the MMAs, sets a CTA's time; splitting a batch into more, emptier CTAs would not
// shorten any CTA and would multiply the L2 traffic.  Up to 64 x 132 roots run in one wave.
MezPlan mez_plan(const MezNet &net, int B)
{
    MezPlan p;
    p.R = std::min(kMezRows, std::max(1, B));
    p.ctas = ceil_div(B, p.R);
    p.last = B - (p.ctas - 1) * p.R;
    p.stages = mez_stages(net.L);
    p.smem = mez_smem(net.L, p.stages).total;
    return p;
}

template <int NC = 1>
static void mez_go(const MezNet &net, const MezIO &io, const MezPlan &p, cudaStream_t s)
{
    if constexpr (NC > kMezMaxL / 32) {
        return;
    } else {
        if (net.L != 32 * NC) return mez_go<NC + 1>(net, io, p, s);
        k_mez_tc<NC><<<p.ctas, kMezThreads, p.smem, s>>>(net, io, p.R, p.stages);
    }
}

template <int NC = 1>
static int mez_attr()
{
    if constexpr (NC > kMezMaxL / 32) {
        return LZ_OK;
    } else {
        LZ_CUDA_CHECK(cudaFuncSetAttribute(k_mez_tc<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMezSmemMax));
        return mez_attr<NC + 1>();
    }
}

int mez_prepare_launch() { return mez_attr<1>(); }

int mez_launch(const MezNet &net, const MezIO &io, cudaStream_t s)
{
    LZ_REQUIRE(io.B > 0 && (io.npass == 1 || io.npass == 3), LZ_EINVAL, "mez_launch: bad argument");
    LZ_REQUIRE(net.L % 32 == 0 && net.L >= 32 && net.L <= kMezMaxL, LZ_EINVAL, "mez_launch: latent %d", net.L);
    const MezPlan p = mez_plan(net, io.B);
    LZ_REQUIRE(p.stages >= 2 && p.smem <= kMezSmemMax, LZ_EINVAL, "mez_launch: %d B of shared memory needed", p.smem);
    mez_go(net, io, p, s);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

// ---- weights ----------------------------------------------------------------------------------
namespace {

struct MezPacker {
    lz_model *m;
    std::vector<unsigned char> w;
    TablePacker tab;

    // Linear `lin` (weight [out_total][in_total]) rows row0 .. row0 + N of inputs 0 .. in_used (+ eval BatchNorm1d `bn`) as one
    // program layer of K (>= in_used, a multiple of 32) inputs; rows past out_total are zero.  Input columns in_used ..
    // in_total (the one-hot action) become the [in_total - in_used][N] table `act` times the BN scale.
    bool layer(MezNet &net, const std::string &lin, const std::string &bn, int in_total, int in_used, int out_total, int row0,
               int N, int K, int in, int out, int flags, std::vector<float> *act = nullptr)
    {
        auto W = find_tensor(m, lin + ".weight", (size_t)out_total * in_total), b = find_tensor(m, lin + ".bias", out_total);
        if (!W || !b) return false;
        std::vector<float> fs(out_total, 1.0f), ft(*b), s(N, 0.0f), t(N, 0.0f);
        if (!bn.empty() && !fold_bn_linear(m, bn, *b, fs, ft)) return false;
        float mx = 0.0f;
        for (int n = 0; n < N && row0 + n < out_total; ++n) {
            s[n] = fs[row0 + n];
            t[n] = ft[row0 + n];
            for (int k = 0; k < in_used; ++k) mx = std::max(mx, fabsf((*W)[(size_t)(row0 + n) * in_total + k]));
        }
        const float scale = pow2_scale(mx);
        const size_t woff = w.size(), chunk = (size_t)128 * N;
        w.resize(woff + chunk * (K / 32));
        __half *hp = reinterpret_cast<__half *>(w.data() + woff);
        for (int c = 0; c < K / 32; ++c)
            for (int kg = 0; kg < 4; ++kg)
                for (int n = 0; n < N; ++n)
                    for (int u = 0; u < 8; ++u) {
                        const int k = 32 * c + 8 * kg + u, r = row0 + n;
                        const float v = (r < out_total && k < in_used) ? (*W)[(size_t)r * in_total + k] * scale : 0.0f;
                        const size_t off = c * chunk / 2 + ((size_t)kg * 2 * N + n) * 8 + u;
                        split_hi_lo(v, hp[off], hp[off + (size_t)N * 8]);
                    }
        if (act) {
            const int na = in_total - in_used;
            act->assign((size_t)na * N, 0.0f);
            for (int a = 0; a < na; ++a)
                for (int n = 0; n < N && row0 + n < out_total; ++n)
                    (*act)[(size_t)a * N + n] = (*W)[(size_t)(row0 + n) * in_total + in_used + a] * s[n];
        }
        std::vector<float> st(2 * N);
        for (int n = 0; n < N; ++n) { st[n] = s[n] / scale; st[N + n] = t[n]; }
        LZ_REQUIRE(net.nlayers < kMezMaxLayers, false, "lz_model_finalize: more than %d layers", kMezMaxLayers);
        MezLayer &ly = net.layer[net.nlayers++];
        ly.woff = (uint32_t)woff; ly.K = K; ly.N = N; ly.in = in; ly.out = out; ly.flags = flags; ly.bn = (int)tab.add(st); ly.col0 = row0;
        net.nchunks += K / 32;
        return true;
    }

    // a categorical head (MLP_V2: Linear(L -> hid) + BN1d + ReLU, Linear(hid -> K)) on the latent in `src`: the hidden layer
    // into the 32-wide buffer, then the FC2 pieces flagged `flag` (MF_VALUE or MF_REWARD), the first and last closing the
    // online softmax expectation
    bool cat_head(MezNet &net, const std::string &mlp, int src, int L, int hid, int K, int flag)
    {
        bool ok = layer(net, mlp + ".0", mlp + ".1", L, L, hid, 0, 32, L, src, MB_HID, MF_RELU);
        for (int r0 = 0; ok && r0 < K; r0 += L)
            ok = layer(net, mlp + ".3", "", hid, hid, K, r0, L, 32, MB_HID, MB_NONE,
                       flag | (r0 == 0 ? MF_CAT_BEGIN : 0) | (r0 + L >= K ? MF_CAT_END : 0));
        return ok;
    }

    // the dynamics MLP `D` over [z | one-hot of na] (muzero_model_mlp.py:428-440, efficientzero_model_mlp.py:440-468) and, for
    // MuZeroModelMLP (mz), its reward head.  Slots: the input latent z in slot 0; fc_dynamics_1 (+ z) -> slot 0 = the next
    // latent; fc_dynamics_2 -> slot 1, which the reward head reads.  Without res_connection_in_dynamics fc_dynamics -> slot 0 is
    // both the next latent and the reward head's input.  EfficientZeroModelMLP writes the reward head's input as the LSTM
    // input (MF_FEAT) of the value-prefix head (ez.cu) instead.
    bool dynamics(MezNet &net, const std::string &D, int L, int na, int K, int rh, bool res, bool mz, std::vector<float> &act)
    {
        if (res)     // next = fc_dynamics_1([z | a]) + z; LSTM / reward head input = fc_dynamics_2(next)
            return layer(net, D + "fc_dynamics_1.0", D + "fc_dynamics_1.1", L + na, L, L, 0, L, L, MB_SLOT0, MB_SLOT1, MF_RELU | MF_ACT, &act) &&
                   layer(net, D + "fc_dynamics_1.3", D + "fc_dynamics_1.4", L, L, L, 0, L, L, MB_SLOT1, MB_SLOT0, MF_RELU | MF_RES | MF_LATENT) &&
                   layer(net, D + "fc_dynamics_2.0", D + "fc_dynamics_2.1", L, L, L, 0, L, L, MB_SLOT0, MB_SLOT1, MF_RELU) &&
                   layer(net, D + "fc_dynamics_2.3", D + "fc_dynamics_2.4", L, L, L, 0, L, L, MB_SLOT1, mz ? MB_SLOT1 : MB_NONE,
                         MF_RELU | (mz ? 0 : MF_FEAT)) &&
                   (!mz || cat_head(net, D + "fc_reward_head", MB_SLOT1, L, rh, K, MF_REWARD));
        // next = LSTM / reward head input = fc_dynamics([z | a])
        return layer(net, D + "fc_dynamics.0", D + "fc_dynamics.1", L + na, L, L, 0, L, L, MB_SLOT0, MB_SLOT1, MF_RELU | MF_ACT, &act) &&
               layer(net, D + "fc_dynamics.3", D + "fc_dynamics.4", L, L, L, 0, L, L, MB_SLOT1, MB_SLOT0, MF_RELU | MF_LATENT | (mz ? 0 : MF_FEAT)) &&
               (!mz || cat_head(net, D + "fc_reward_head", MB_SLOT0, L, rh, K, MF_REWARD));
    }

    // prediction network `Q` with A policy outputs on the latent in `src` (common.py:1218-1292); the other slot is its work buffer
    bool predict(MezNet &net, const std::string &Q, int src, int L, int A, int K, int vh, int ph)
    {
        const int wk = src == MB_SLOT0 ? MB_SLOT1 : MB_SLOT0;
        bool ok = layer(net, Q + "fc_prediction_common.0", Q + "fc_prediction_common.1", L, L, L, 0, L, L, src, wk, MF_RELU) &&
                  layer(net, Q + "fc_prediction_common.3", Q + "fc_prediction_common.4", L, L, L, 0, L, L, wk, wk, MF_RELU) &&
                  cat_head(net, Q + "fc_value_head", wk, L, vh, K, MF_VALUE);
        ok = ok && layer(net, Q + "fc_policy_head.0", Q + "fc_policy_head.1", L, L, ph, 0, 32, L, wk, MB_HID, MF_RELU);
        for (int r0 = 0; ok && r0 < A; r0 += L) ok = layer(net, Q + "fc_policy_head.3", "", ph, ph, A, r0, L, 32, MB_HID, MB_NONE, MF_POLICY);
        return ok;
    }
};

}  // namespace

// EfficientZeroModelMLP, MuZeroModelMLP and StochasticMuZeroModelMLP share the representation and prediction programs and the
// dynamics MLP (MezPacker::dynamics).  StochasticMuZeroModelMLP (stochastic_muzero_model_mlp.py) has two recurrent programs:
// `after`, afterstate_dynamics_network over [latent | one-hot action] and afterstate_prediction_network with the C chance
// outcomes as its policy outputs (recurrent_inference(afterstate=False), stochastic_muzero_model.py:266-271), and `rec`,
// dynamics_network over [afterstate | one-hot chance outcome] and prediction_network (afterstate=True, :262-265).
int mez_finalize(lz_model *m)
{
    const MlpTcState &c = m->mez;
    const bool mz = !m->vp;
    const int L = c.latent, A = m->A, C = m->chance, K = m->K, kobs = (c.obs_dim + 31) / 32 * 32;
    MezPacker P;
    P.m = m;
    MezNet init, rec, after;
    memset(&init, 0, sizeof(init));
    memset(&rec, 0, sizeof(rec));
    memset(&after, 0, sizeof(after));
    const std::string R = "representation_network.", Q = "prediction_network.";
    std::vector<float> act, act_after;
    bool ok = P.layer(init, R + "fc_representation.0", R + "fc_representation.1", c.obs_dim, c.obs_dim, L, 0, L, kobs, MB_OBS, MB_SLOT0, MF_GELU) &&
              P.layer(init, R + "fc_representation.3", "", L, L, L, 0, L, L, MB_SLOT0, MB_SLOT0, MF_LN | MF_LATENT) &&
              P.predict(init, Q, MB_SLOT0, L, A, K, c.value_hidden, c.policy_hidden);
    ok = ok && P.dynamics(rec, "dynamics_network.", L, C ? C : A, K, c.reward_hidden, c.res, mz, act) &&
         P.predict(rec, Q, MB_SLOT0, L, A, K, c.value_hidden, c.policy_hidden);
    if (C)
        ok = ok && P.dynamics(after, "afterstate_dynamics_network.", L, A, K, c.reward_hidden, c.res, true, act_after) &&
             P.predict(after, "afterstate_prediction_network.", MB_SLOT0, L, C, K, c.value_hidden, c.policy_hidden);
    if (!ok) return LZ_EINVAL;
    auto lw = find_tensor(m, R + "norm.weight", L), lb = find_tensor(m, R + "norm.bias", L);
    if (!lw || !lb) return LZ_EINVAL;
    const size_t o_lw = P.tab.add(*lw), o_lb = P.tab.add(*lb), o_act = P.tab.add(act), o_act_after = P.tab.add(act_after);
    // one upload: the weight chunks, then the tables from the next 256-byte boundary
    const size_t wbytes = (P.w.size() + 255) & ~(size_t)255;
    P.w.resize(wbytes, 0);
    P.w.insert(P.w.end(), reinterpret_cast<const unsigned char *>(P.tab.host.data()),
               reinterpret_cast<const unsigned char *>(P.tab.host.data() + P.tab.host.size()));
    int rc = upload(&m->mez.d_mez, P.w.data(), P.w.size());
    if (rc != LZ_OK) return rc;
    const float *tab = reinterpret_cast<const float *>(m->mez.d_mez + wbytes);
    for (MezNet *n : {&init, &rec, &after}) {
        n->w = m->mez.d_mez; n->tab = tab; n->abias = tab + o_act; n->ln_w = tab + o_lw; n->ln_b = tab + o_lb;
        n->L = L; n->A = A; n->K = K; n->obs_dim = c.obs_dim; n->nact = A;
        n->support_min = m->support_min; n->support_step = m->support_step;
    }
    if (C) {
        rec.nact = C;
        after.A = C; after.abias = tab + o_act_after;
    }
    m->mez.init = init;
    m->mez.rec = rec;
    m->mez.after = after;
    if ((rc = mez_prepare_launch()) != LZ_OK) return rc;
    return m->vp ? ez_finalize(m, L, c.reward_hidden, false) : LZ_OK;
}

static MezIO mez_io(const lz_model *m, int B)
{
    MezIO e;
    memset(&e, 0, sizeof(e));
    e.B = B; e.npass = m->npass;
    return e;
}

int mez_recurrent(lz_model *m, const RecIO &io, cudaStream_t s)
{
    // EfficientZeroModelMLP's LSTM input goes on through the value-prefix head (ez.cu), MuZeroModelMLP's reward head is part of
    // the program
    const bool ez = m->vp;
    if (ez) {
        LZ_REQUIRE(io.B <= m->ez.B, LZ_ESTATE, "model_recurrent: EfficientZero scratch sized for %d roots, got %d (model_reserve)", m->ez.B, io.B);
        LZ_REQUIRE(io.h_base && io.c_base, LZ_EINVAL, "model_recurrent: EfficientZero needs the reward hidden state");
    }
    LZ_REQUIRE(!io.after_program || m->chance, LZ_EINVAL, "model_recurrent: the afterstate program is StochasticMuZeroModelMLP's");
    MezIO e = mez_io(m, io.B);
    e.latent_base = io.latent_base; e.ix = io.ix; e.slot_stride = io.slot_stride; e.action = io.action;
    e.row_mask = io.row_mask; e.row_mask_on = io.row_mask_on; e.policy_stride = io.policy_stride;
    e.latent_out = io.next_latent;
    if (ez) e.feat = m->ez.feat;
    else { e.reward = io.reward; e.reward_logits = io.reward_logits; }
    e.value = io.value; e.policy_logits = io.policy_logits; e.value_logits = io.value_logits;
    int rc = mez_launch(io.after_program ? m->mez.after : m->mez.rec, e, s);
    if (rc || !ez) return rc;
    return ez_tail(m, io, s);
}

int mez_initial(lz_model *m, int B, const float *d_obs, const TailIO &io_in, cudaStream_t s)
{
    MezIO e = mez_io(m, B);
    e.obs = d_obs; e.latent_out = io_in.latent; e.latent_out2 = io_in.latent2;
    e.value = io_in.value; e.policy_logits = io_in.policy_logits; e.value_logits = io_in.value_logits;
    e.policy_stride = io_in.policy_stride;
    return mez_launch(m->mez.init, e, s);
}

// lz_model_debug_net_stage of EfficientZeroModelMLP, MuZeroModelMLP and StochasticMuZeroModelMLP on the tensor cores: which 1
// is initial_inference on the observations d_in, 0 the recurrent program, 2 StochasticMuZeroModelMLP's afterstate program (its
// policy is chance_space_size wide)
int mez_debug_stage(lz_model *m, int which, int B, const float *d_in, const int32_t *d_action, int stage, void *d_out,
                           size_t out_bytes, int32_t *h_info, cudaStream_t st)
{
    LZ_REQUIRE(which != 2 || m->chance, LZ_EINVAL, "lz_model_debug_net_stage: which 2 is StochasticMuZeroModelMLP's afterstate program");
    MezNet net = which == 2 ? m->mez.after : which ? m->mez.init : m->mez.rec;   // a copy: the model's programs stay as they are
    const int L = net.L, K = net.K, A = net.A;
    const bool rew = which != 1 && !m->vp;           // MuZeroModelMLP's recurrent programs have the reward head
    int dense[kMezMaxLayers], D = 0;                        // the program indices of the L-wide layers outside the heads
    for (int l = 0; l < net.nlayers; ++l)
        if (net.layer[l].N == L && !(net.layer[l].flags & (MF_VALUE | MF_REWARD | MF_POLICY)) && net.layer[l].out != MB_HID) dense[D++] = l;
    LZ_REQUIRE(stage <= D, LZ_EINVAL, "lz_model_debug_net_stage: stage %d past the %d dense layers of the program", stage, D);
    const size_t nfl = stage < D ? (size_t)B * L : (size_t)B * (K + A + 1 + 2 * L + (rew ? K + 1 : 0));
    LZ_REQUIRE(out_bytes >= nfl * sizeof(float), LZ_EINVAL, "lz_model_debug_net_stage: stage %d needs %zu bytes, got %zu", stage,
               nfl * sizeof(float), out_bytes);
    MezIO io = mez_io(m, B);
    if (which == 1) io.obs = d_in;
    else { io.latent_base = d_in; io.action = d_action; }
    float *o = reinterpret_cast<float *>(d_out);
    if (stage < D) {
        // the program cut after dense layer `stage`, whose output is the only one written (the reward head before it, in
        // MuZeroModelMLP's recurrent program, runs with no output)
        const int cut = dense[stage];
        net.nlayers = cut + 1;
        net.nchunks = 0;
        for (int l = 0; l <= cut; ++l) {
            net.layer[l].flags &= ~(MF_LATENT | MF_FEAT);
            net.nchunks += net.layer[l].K / 32;
        }
        net.layer[cut].flags |= MF_LATENT;
        io.latent_out = o;
    } else {
        // the latent sections first: the kernel writes them as float2 pairs; then value logits, policy logits, value, and for
        // MuZeroModelMLP's recurrent program reward logits and reward (its LSTM-input section stays zero)
        LZ_CUDA_CHECK(cudaMemsetAsync(d_out, 0, nfl * sizeof(float), st));
        io.latent_out = o;
        if (!which && m->vp) io.feat = o + (size_t)B * L;
        io.value_logits = o + (size_t)2 * B * L; io.policy_logits = io.value_logits + (size_t)B * K; io.value = io.policy_logits + (size_t)B * A;
        if (rew) { io.reward_logits = io.value + B; io.reward = io.reward_logits + (size_t)B * K; }
    }
    const MezPlan p = mez_plan(net, B);
    const int32_t info[8] = {p.R, p.ctas, p.last, net.nlayers, m->npass, p.smem, p.stages, D};
    memcpy(h_info, info, sizeof(info));
    return mez_launch(net, io, st);
}

}  // namespace lz
