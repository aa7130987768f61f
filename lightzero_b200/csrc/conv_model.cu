// conv_model.cu -- the Conv family: MuZeroModel / EfficientZeroModel with the DownSample tower.  Forward paths
// (initial_inference / recurrent_inference): the DownSample stem, the launches of the tensor-core tower (conv_tc.cu) and of the
// latent-grid network (net_tc.cu), and the packing of their weight tables from the reference state_dict.
//
// Replaces the forward paths of lzero/model/muzero_model.py:210-272 (MuZeroModel), :309-374 (_dynamics
// one-hot encoding), :505-538 (DynamicsNetwork.forward), lzero/model/common.py:334-366 (DownSample),
// :764-787 (RepresentationNetwork) and :1189-1215 (PredictionNetwork), eval mode only.
#include <math.h>
#include <string.h>

#include <algorithm>

#include "model.cuh"
#include "tc_ptx.cuh"

namespace lz {

// ------------------------------------------------------------------------------------------------
// The stem of the DownSample tower (conv1 + norm1 + ReLU, common.py:334-366) for the input channel counts k_stem4_tcl does not
// take (e.g. 3- or 9-channel frames): direct 3x3 convolution of stride S = 2 from NCHW, written into the tensor-core layout of
// the first wgmma layer.  One thread per output pixel (128 consecutive linear pixels per CTA), 32 output channels per CTA.
// ------------------------------------------------------------------------------------------------
template <int S>
__global__ void __launch_bounds__(128)
k_conv3x3_generic(ConvG L, const float *__restrict__ in, int cic, int nrows_max, Tcl tcl, const uint8_t *__restrict__ in_u8)
{
    extern __shared__ __align__(16) float sm[];
    const int pitch = L.win + 2;
    float *in_t = sm;
    float *w_t = sm + (((size_t)cic * nrows_max * pitch + 3) & ~(size_t)3);
    const int b = blockIdx.z, co0 = blockIdx.y * 32, tid = threadIdx.x;
    const int npx = L.hout * L.wout;
    const int p0 = blockIdx.x * 128, p = p0 + tid;
    const bool valid = p < npx;
    const int y = valid ? p / L.wout : 0, x = valid ? p - y * L.wout : 0;
    const int y_first = p0 / L.wout, y_last = min(p0 + 127, npx - 1) / L.wout;
    const int r0 = y_first * S - 1, nrows = (y_last - y_first) * S + 3;
    float acc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = 0.0f;

    for (int c0 = 0; c0 < L.cin; c0 += cic) {
        const int per_c = nrows * pitch, nin = cic * per_c;
        for (int i = tid; i < nin; i += 128) {
            int cl = i / per_c, rem = i - cl * per_c, rr = rem / pitch, cc = rem - rr * pitch;
            int gy = r0 + rr, gx = cc - 1, c = c0 + cl;
            float v = 0.0f;
            if (c < L.cin && gy >= 0 && gy < L.hin && gx >= 0 && gx < L.win) {
                const size_t gi = (((size_t)b * L.cin + c) * L.hin + gy) * L.win + gx;
                // uint8 frames: the [0, 1] scaling of the reference's env wrapper (ScaledFloatFrameWrapper: (obs - 0) / 255 ->
                // float32, zoo/atari/envs/atari_wrappers.py:219-220) happens here; a correctly rounded fp32 division
                // reproduces that float64-divide-then-cast bit for bit for all 256 inputs (tests/test_host_logic_cpu.py)
                v = in_u8 ? __fdiv_rn((float)in_u8[gi], 255.0f) : in[gi];
            }
            in_t[((size_t)cl * nrows_max + rr) * pitch + cc] = v;
        }
        for (int i = tid; i < cic * 288; i += 128) {
            int cl = i / 288, rem = i - cl * 288, tap = rem >> 5, j = rem & 31, c = c0 + cl;
            w_t[i] = c < L.cin ? L.w[((size_t)c * 9 + tap) * L.cout + co0 + j] : 0.0f;
        }
        __syncthreads();
        if (valid) {
            for (int cl = 0; cl < cic; ++cl) {
#pragma unroll
                for (int ky = 0; ky < 3; ++ky) {
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx) {
                        const float v = in_t[((size_t)cl * nrows_max + (y - y_first) * S + ky) * pitch + x * S + kx];
                        const float4 *wv = reinterpret_cast<const float4 *>(w_t + (cl * 9 + ky * 3 + kx) * 32);
#pragma unroll
                        for (int q = 0; q < 8; ++q) {
                            const float4 w4 = wv[q];
                            acc[4 * q + 0] = fmaf(v, w4.x, acc[4 * q + 0]);
                            acc[4 * q + 1] = fmaf(v, w4.y, acc[4 * q + 1]);
                            acc[4 * q + 2] = fmaf(v, w4.z, acc[4 * q + 2]);
                            acc[4 * q + 3] = fmaf(v, w4.w, acc[4 * q + 3]);
                        }
                    }
                }
            }
        }
        __syncthreads();
    }
    if (valid) {
        // write the tensor-core layout of conv_tc.cuh (fp16 hi/lo, k-group planes over the padded grid)
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = fmaxf(fmaf(acc[j], __ldg(L.scale + co0 + j), __ldg(L.shift + co0 + j)), 0.0f);
        const int rho = (y + 1) * tcl.pitch + x;
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            unsigned char *op = tcl.base + (size_t)b * tcl.img_stride + ((size_t)(co0 / 8 + g) * tcl.plane_rows + rho + 1) * 16;
            store_split8(op, op + tcl.part_stride, v + 8 * g);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// The stem of the DownSample tower for 4 input channels (DownSample.conv1 + norm1 + ReLU, common.py:334-366; 3x3, stride 2,
// pad 1, 4 -> 32 channels) on the CUDA cores, written straight into the tensor-core layout (TCL) of the first wgmma layer.
// K = 36 is too thin for the tensor cores; the kernel is FFMA-bound by construction: the 1,152 weights and the folded BatchNorm
// tables travel BY VALUE in the kernel parameters, so every FFMA takes its weight operand from the constant bank (no weight
// loads at all) and the only shared-memory traffic is one activation load per 32 FFMAs.  CTA = rows_per_cta full output rows
// (thread = output pixel, 32 accumulators), input band staged with 16-byte loads (uint8 frames are scaled to [0, 1] here).
// ------------------------------------------------------------------------------------------------
struct StemP { float w[4 * 9 * 32]; float scale[32], shift[32]; };

template <bool U8>
__global__ void __launch_bounds__(256)
k_stem4_tcl(const __grid_constant__ StemP P, const float *__restrict__ in, const uint8_t *__restrict__ in_u8, int hin, int win,
            int hout, int wout, int rows_per_cta, Tcl tcl)
{
    extern __shared__ __align__(16) float sm[];      // [4][nrows][pitch], column gx at index 4 + gx (index 3: the left padding)
    const int tid = threadIdx.x, b = blockIdx.y, y0 = blockIdx.x * rows_per_cta;
    const int nrows = 2 * rows_per_cta + 1, pitch = win + 4, r0 = 2 * y0 - 1, nq = win >> 2;
    for (int i = tid; i < 4 * nrows * nq; i += 256) {
        const int q = i % nq, rr = (i / nq) % nrows, c = i / (nq * nrows), gy = r0 + rr;
        float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (gy >= 0 && gy < hin) {
            const size_t gi = (((size_t)b * 4 + c) * hin + gy) * win + 4 * q;
            if (U8) {
                // ScaledFloatFrameWrapper: obs / 255 in float64, cast to float32 == one correctly rounded fp32 division (see
                // k_conv3x3_generic)
                const uchar4 u = *reinterpret_cast<const uchar4 *>(in_u8 + gi);
                v = make_float4(__fdiv_rn((float)u.x, 255.0f), __fdiv_rn((float)u.y, 255.0f), __fdiv_rn((float)u.z, 255.0f),
                                __fdiv_rn((float)u.w, 255.0f));
            } else {
                v = *reinterpret_cast<const float4 *>(in + gi);
            }
        }
        *reinterpret_cast<float4 *>(sm + (size_t)(c * nrows + rr) * pitch + 4 + 4 * q) = v;
    }
    for (int i = tid; i < 4 * nrows; i += 256) sm[(size_t)i * pitch + 3] = 0.0f;
    __syncthreads();
    const int yl = tid / wout, x = tid - yl * wout, y = y0 + yl;
    if (yl >= rows_per_cta || y >= hout) return;
    float acc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = 0.0f;
    const float *row0 = sm + (size_t)(2 * yl) * pitch + 2 * x + 3;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const float v = row0[(size_t)(c * nrows + ky) * pitch + kx];
#pragma unroll
                for (int j = 0; j < 32; ++j) acc[j] = fmaf(v, P.w[(c * 9 + ky * 3 + kx) * 32 + j], acc[j]);
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = fmaxf(fmaf(acc[j], P.scale[j], P.shift[j]), 0.0f);
    const int rho = (y + 1) * tcl.pitch + x;
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        unsigned char *op = tcl.base + (size_t)b * tcl.img_stride + ((size_t)g * tcl.plane_rows + rho + 1) * 16;
        store_split8(op, op + tcl.part_stride, acc + 8 * g);
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
int conv_recurrent(lz_model *m, const RecIO &io, cudaStream_t s)
{
    TcIO t;
    memset(&t, 0, sizeof(t));
    t.B = io.B; t.npass = m->npass;
    t.latent_base = io.latent_base; t.ix = io.ix; t.slot_stride = io.slot_stride; t.action = io.action;
    t.latent_out = io.next_latent; t.reward = io.reward; t.value = io.value; t.policy_logits = io.policy_logits;
    t.reward_logits = io.reward_logits; t.value_logits = io.value_logits;
    t.skip_scratch = io.skip_scratch;
    if (!t.skip_scratch) {
        LZ_REQUIRE(io.B <= m->conv.tc_skip_B, LZ_ESTATE, "model_recurrent: scratch sized for %d roots, got %d (model_reserve)", m->conv.tc_skip_B, io.B);
        t.skip_scratch = m->conv.tc_skip;
    }
    if (m->vp) {
        // conv trunk + prediction heads on the tensor cores; the reward features go through the LSTM head (ez.cu)
        LZ_REQUIRE(io.B <= m->ez.B, LZ_ESTATE, "model_recurrent: EfficientZero scratch sized for %d roots, got %d (model_reserve)", m->ez.B, io.B);
        LZ_REQUIRE(io.h_base && io.c_base, LZ_EINVAL, "model_recurrent: EfficientZero needs the reward hidden state");
        t.reward = nullptr; t.reward_logits = nullptr; t.ez_feat = m->ez.feat;
        int rc = tc_launch(m->conv.tc_rec, t, s);
        if (rc) return rc;
        return ez_tail(m, io, s);
    }
    return tc_launch(m->conv.tc_rec, t, s);
}

// the stem for input channel counts other than 4 (k_stem4_tcl), into the first TCL tensor
static int launch_stem_generic(const ConvG &L, const float *in, const uint8_t *in_u8, int B, const Tcl &tcl, cudaStream_t s)
{
    const int cic = std::min(8, L.cin);
    const int rows_out_max = std::min(L.hout, 127 / L.wout + 2);
    const int nrows_max = (rows_out_max - 1) * 2 + 3;
    const int pitch = L.win + 2;
    const size_t smem = ((((size_t)cic * nrows_max * pitch + 3) & ~(size_t)3) + (size_t)cic * 288) * sizeof(float);
    dim3 grid(ceil_div(L.hout * L.wout, 128), L.cout / 32, B);
    LZ_REQUIRE(smem <= 200 * 1024, LZ_EINVAL, "DownSample stem needs %zu B shared memory", smem);
    k_conv3x3_generic<2><<<grid, 128, smem, s>>>(L, in, cic, nrows_max, tcl, in_u8);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

// skip scratch of the tensor-core latent-grid kernel (grown outside stream capture: API entry points and lz_search_create)
int conv_reserve_skip(lz_model *m, int B)
{
    if (B <= m->conv.tc_skip_B) return LZ_OK;
    ++m->generation;
    dev_free(m->conv.tc_skip);
    m->conv.tc_skip = nullptr; m->conv.tc_skip_B = 0;
    int rc = dev_alloc(&m->conv.tc_skip, (size_t)m->latent_floats * B);
    if (rc != LZ_OK) return rc;
    m->conv.tc_skip_B = B;
    return LZ_OK;
}

// the skip scratch, and the DownSample tower's workspace of initial inference (zeroed on s)
int conv_reserve(lz_model *m, int B, cudaStream_t s)
{
    {
        int rc = conv_reserve_skip(m, B);
        if (rc != LZ_OK) return rc;
    }
    if (B <= m->conv.ws_B) return LZ_OK;
    ++m->generation;
    dev_free(m->conv.pre_latent);
    m->conv.pre_latent = nullptr;
    {
        int rc = dev_alloc(&m->conv.pre_latent, (size_t)m->latent_floats * B);
        if (rc != LZ_OK) return rc;
    }
    m->conv.ws_B = B;
    // TCL activation workspace of the tensor-core tower (zeroed once: pad rows / columns are never written non-zero)
    {
        const int h1 = m->conv.stem.hout, h2 = (h1 - 1) / 2 + 1, h3 = (h2 - 1) / 2 + 1, c2 = kC / 2;
        const size_t bT = tcl_bytes(B, c2, h1, h1, 1), bT2 = tcl_bytes(B, c2, h1 / 2, h1 / 2, 4);
        const size_t bU = tcl_bytes(B, kC, h2, h2, 1), bV = tcl_bytes(B, kC, h3, h3, 1);
        const size_t total = bT + bT2 + 3 * bU + 2 * bV;
        dev_free(m->conv.tws);
        m->conv.tws = nullptr;
        int rc = dev_alloc(&m->conv.tws, total);
        if (rc != LZ_OK) return rc;
        LZ_CUDA_CHECK(cudaMemsetAsync(m->conv.tws, 0, total, s));
        unsigned char *q = m->conv.tws;
        m->conv.T0 = make_tcl(q, c2, h1, h1, 1); q += bT;
        m->conv.T1 = make_tcl(q, c2, h1 / 2, h1 / 2, 4); q += bT2;
        m->conv.U0 = make_tcl(q, kC, h2, h2, 1); q += bU;
        m->conv.U1 = make_tcl(q, kC, h2, h2, 1); q += bU;
        m->conv.U2 = make_tcl(q, kC, h2, h2, 1); q += bU;
        m->conv.V0 = make_tcl(q, kC, h3, h3, 1); q += bV;
        m->conv.V1 = make_tcl(q, kC, h3, h3, 1); q += bV;
    }
    return LZ_OK;
}

// ---- tensor-core (wgmma) tower ------------------------------------------------------------------
// picks the band height (and, for whole small images, the images per CTA) that fits shared memory and wastes the fewest MMA rows
static void pick_band(ConvTc &p)
{
    const int H = p.in.H, pitch = p.in.pitch, kg = p.in.C / 8;
    double best = -1.0;
    int best_h = 1, best_g = 1, best_st = 4;
    for (int G = 1; G <= 4; ++G)
        for (int bh = (G > 1 ? H : 1); bh <= H; ++bh)
            for (int st = 2; st <= 4; st += 2) {
                const int rin = (bh + 2) * pitch + 2, mcount = (G - 1) * rin + bh * pitch, NT = (mcount + 127) / 128;
                int PR = pitch + 1 + NT * 128 + pitch + 2;
                if (PR < G * rin) PR = G * rin;
                const size_t smem = (((size_t)PR * 16 * kg * 2 * p.in.nphase + 127) & ~(size_t)127) + st * (size_t)2 * kg * p.N * 16 + 1024;
                if (smem > 227 * 1024) continue;
                const int nb = (H + bh - 1) / bh;
                double score = (double)(G * H * (pitch - 1)) / ((double)nb * NT * 128);       // useful / issued MMA rows
                // two co-resident CTAs (N <= 64, see k_conv_tc) overlap one band's load / epilogue with the other's MMAs: initial_inference
                // at B = 1024 took 4.0 ms with this preference and 4.5 ms without it (H100 SXM, 700 W)
                if (p.N <= 64 && smem <= 113 * 1024) score *= 1.35;
                score *= (st == 4) ? 1.0 : 0.97;
                if (score > best + 1e-9) { best = score; best_h = bh; best_g = G; best_st = st; }
            }
    p.band_h = best_h;
    p.G = best_g;
    p.stages = best_st;
}

// stop_after < 8 ends the tower after that stage's launch (stage numbers of lz_model_debug_tower_stage); pre_latent is then
// not written
static int tower_tc_run(lz_model *m, int B, const float *d_obs, float *pre_latent, cudaStream_t s, const uint8_t *d_obs_u8 = nullptr,
                        int stop_after = 8)
{
    int rc;
    const int npass = m->npass;
    // stem: conv1 (stride 2) on the CUDA cores, written straight into TCL (uint8 frames are scaled to [0, 1] here)
    const ConvG &S0 = m->conv.stem;
    if (m->conv.stem_valid) {
        const int rows_per_cta = std::max(1, 256 / S0.wout);
        const size_t smem = (size_t)4 * (2 * rows_per_cta + 1) * (S0.win + 4) * sizeof(float);
        dim3 grid(ceil_div(S0.hout, rows_per_cta), B);
        const StemP &P = *reinterpret_cast<const StemP *>(m->conv.stem_params.data());
        if (d_obs_u8) k_stem4_tcl<true><<<grid, 256, smem, s>>>(P, nullptr, d_obs_u8, S0.hin, S0.win, S0.hout, S0.wout, rows_per_cta, m->conv.T0);
        else k_stem4_tcl<false><<<grid, 256, smem, s>>>(P, d_obs, nullptr, S0.hin, S0.win, S0.hout, S0.wout, rows_per_cta, m->conv.T0);
        LZ_KERNEL_CHECK();
    } else if ((rc = launch_stem_generic(S0, d_obs, d_obs_u8, B, m->conv.T0, s))) return rc;
    if (stop_after <= 0) return LZ_OK;
    auto run = [&](ConvTc p, const Tcl &in, const Tcl &o0, const Tcl *o1, const Tcl *res) {
        p.in = in; p.out[0] = o0;
        if (o1) p.out[1] = *o1;
        if (res) p.res = *res; else p.res.base = nullptr;
        p.B = B; p.npass = npass;
        return conv_tc_launch(p, s);
    };
    auto rb = [&](ResBlockTc p, const Tcl &in, const Tcl &out) {
        p.in = in; p.out = out;
        p.B = B; p.npass = npass;
        return resblock_tc_launch(p, s);
    };
    if ((rc = rb(m->conv.tower_rb[0], m->conv.T0, m->conv.T1))) return rc;                           // resblocks1.0 -> phase-split
    if (stop_after <= 1) return LZ_OK;
    if ((rc = run(m->conv.tower_tc[0], m->conv.T1, m->conv.U0, &m->conv.U1, nullptr))) return rc;         // downsample conv1 | conv3 (stride 2)
    if (stop_after <= 3) return LZ_OK;
    if ((rc = run(m->conv.tower_tc[1], m->conv.U0, m->conv.U2, nullptr, &m->conv.U1))) return rc;         // downsample conv2 + identity
    if (stop_after <= 4) return LZ_OK;
    if ((rc = rb(m->conv.tower_rb[1], m->conv.U2, m->conv.U0))) return rc;                           // resblocks2.0
    if (stop_after <= 5) return LZ_OK;
    if ((rc = pool_tcl_launch(m->conv.U0, m->conv.V0, B, s))) return rc;                        // pooling1
    if (stop_after <= 6) return LZ_OK;
    if ((rc = rb(m->conv.tower_rb[2], m->conv.V0, m->conv.V1))) return rc;                           // resblocks3.0
    if (stop_after <= 7) return LZ_OK;
    if (m->lat_h == 8) return tcl_to_nchw_launch(m->conv.V1, pre_latent, B, s);             // 64 px: no pooling2 -> [B][64][8][8]
    return pool_tcl_to_nchw_launch(m->conv.V1, pre_latent, B, m->lat_h, s);                  // pooling2 -> [B][64][6][6]
}

// the DownSample tower alone (obs -> pre-latent [B][64][P]) ...
int conv_initial_tower(lz_model *m, int B, const float *d_obs, float *pre_latent, cudaStream_t s, const uint8_t *d_obs_u8)
{
    LZ_REQUIRE(B <= m->conv.ws_B, LZ_ESTATE, "model_initial_tower: workspace sized for %d roots, got %d", m->conv.ws_B, B);
    return tower_tc_run(m, B, d_obs, pre_latent, s, d_obs_u8);
}

// ... and the latent-grid tail (representation ResBlocks -> latent -> prediction network)
int conv_initial_tail(lz_model *m, int B, const float *pre_latent, const TailIO &io_in, cudaStream_t s)
{
    TcIO t;
    memset(&t, 0, sizeof(t));
    t.B = B; t.npass = m->npass;
    t.latent_base = pre_latent; t.latent_out = io_in.latent; t.latent_out2 = io_in.latent2;
    t.value = io_in.value; t.policy_logits = io_in.policy_logits; t.value_logits = io_in.value_logits;
    LZ_REQUIRE(B <= m->conv.tc_skip_B, LZ_ESTATE, "model_initial_tail: scratch sized for %d roots, got %d (model_reserve)", m->conv.tc_skip_B, B);
    t.skip_scratch = m->conv.tc_skip;
    return tc_launch(m->conv.tc_tail, t, s);
}

int conv_initial(lz_model *m, int B, const float *d_obs, const TailIO &io_in, cudaStream_t s)
{
    LZ_REQUIRE(B <= m->conv.ws_B, LZ_ESTATE, "model_initial: workspace sized for %d roots, got %d (call model_reserve outside capture)", m->conv.ws_B, B);
    int rc = tower_tc_run(m, B, d_obs, m->conv.pre_latent, s);
    if (rc) return rc;
    return conv_initial_tail(m, B, m->conv.pre_latent, io_in, s);
}

// ---- weight ingestion -------------------------------------------------------------------------
struct ConvOff { size_t w, scale, shift; int cin, cout; };

// torch conv weight [cout][cin][3][3] -> [cin][9][cout]
static bool pack_conv3(lz_model *m, TablePacker &P, const std::string &wname, const std::string &bnprefix, int cin,
                       int cout, ConvOff &o)
{
    auto w = find_tensor(m, wname, (size_t)cout * cin * 9);
    if (!w) return false;
    std::vector<float> wp((size_t)cin * 9 * cout), scale(cout, 1.0f), shift(cout, 0.0f);
    for (int co = 0; co < cout; ++co)
        for (int ci = 0; ci < cin; ++ci)
            for (int t = 0; t < 9; ++t) wp[((size_t)ci * 9 + t) * cout + co] = (*w)[((size_t)co * cin + ci) * 9 + t];
    if (!bnprefix.empty() && !fold_bn(m, bnprefix, cout, scale, shift)) return false;
    o.w = P.add(wp); o.scale = P.add(scale); o.shift = P.add(shift);
    o.cin = cin; o.cout = cout;
    return true;
}

struct HeadOff { size_t s2, t2, b2; int hc, hid, K; };

// the fp32 tables of a head's FC part that k_net_tc reads (pack_tc packs the weights); fc empty: EfficientZero's reward head,
// whose FC part follows the LSTM (ez.cu), is recorded with hid = 0
static bool pack_head(lz_model *m, TablePacker &P, const std::string &fc, int hc, int hid, int K, HeadOff &o)
{
    o.s2 = o.t2 = o.b2 = 0;
    o.hc = hc; o.hid = 0; o.K = K;
    if (fc.empty()) return true;
    auto B0 = find_tensor(m, fc + ".0.bias", hid), B3 = find_tensor(m, fc + ".3.bias", K);
    std::vector<float> s2, t2;
    if (!B0 || !B3 || !fold_bn(m, fc + ".1", hid, s2, t2)) return false;
    for (int j = 0; j < hid; ++j) t2[j] += s2[j] * (*B0)[j];
    o.s2 = P.add(s2); o.t2 = P.add(t2); o.b2 = P.add(*B3);
    o.hid = hid;
    return true;
}

// ---- tensor-core tower tables (conv_tc.cu) ----
static int pack_tower_tc(lz_model *m)
{
    const std::string R = "representation_network.downsample_net.";
    const int c2 = kC / 2;
    const int h1 = m->conv.stem.hout, h2 = (h1 - 1) / 2 + 1, h3 = (h2 - 1) / 2 + 1;
    struct Item { std::string w, bn; int cin, cout; };
    // layer table: 0 rb1.c1, 1 rb1.c2, 2 ds.c1 | ds.c3 (merged N=128), 3 ds.c2, 4 rb2.c1, 5 rb2.c2, 6 rb3.c1, 7 rb3.c2
    // (layers 0-1, 4-5 and 6-7 run as fused ResBlocks, 2 and 3 as single convs)
    const Item items[9] = {
        {R + "resblocks1.0.conv1.0.weight", R + "resblocks1.0.conv1.1", c2, c2},
        {R + "resblocks1.0.conv2.0.weight", R + "resblocks1.0.conv2.1", c2, c2},
        {R + "downsample_block.conv1.0.weight", R + "downsample_block.conv1.1", c2, kC},
        {R + "downsample_block.conv3.0.weight", "", c2, kC},
        {R + "downsample_block.conv2.0.weight", R + "downsample_block.conv2.1", kC, kC},
        {R + "resblocks2.0.conv1.0.weight", R + "resblocks2.0.conv1.1", kC, kC},
        {R + "resblocks2.0.conv2.0.weight", R + "resblocks2.0.conv2.1", kC, kC},
        {R + "resblocks3.0.conv1.0.weight", R + "resblocks3.0.conv1.1", kC, kC},
        {R + "resblocks3.0.conv2.0.weight", R + "resblocks3.0.conv2.1", kC, kC},
    };
    // (layer index, item indices, N)
    struct Lay { int it0, it1, cin, N; };
    const Lay lays[8] = {{0, -1, c2, c2}, {1, -1, c2, c2}, {2, 3, c2, 2 * kC}, {4, -1, kC, kC},
                         {5, -1, kC, kC}, {6, -1, kC, kC}, {7, -1, kC, kC}, {8, -1, kC, kC}};
    size_t wbytes = 0;
    for (const Lay &l : lays) wbytes += conv_tc_packed_bytes(l.cin, l.N);
    size_t tab_off = (wbytes + 255) & ~(size_t)255;
    std::vector<unsigned char> host(tab_off + 8 * 2 * 128 * sizeof(float), 0);
    float *tab = reinterpret_cast<float *>(host.data() + tab_off);
    size_t woff[8], off = 0;
    for (int li = 0; li < 8; ++li) {
        const Lay &l = lays[li];
        woff[li] = off;
        float *scale = tab + li * 256, *shift = scale + 128;
        for (int part = 0; part < 2; ++part) {
            const int it = part == 0 ? l.it0 : l.it1;
            if (it < 0) continue;
            const Item &I = items[it];
            auto w = find_tensor(m, I.w, (size_t)I.cout * I.cin * 9);
            if (!w) return LZ_EINVAL;
            std::vector<float> sc(I.cout, 1.0f), sh(I.cout, 0.0f);
            if (!I.bn.empty() && !fold_bn(m, I.bn, I.cout, sc, sh)) return LZ_EINVAL;
            const int col0 = part * kC;
            const float ws = conv_tc_pack(w->data(), I.cin, I.cout, l.N, col0, host.data() + off);
            for (int k = 0; k < I.cout; ++k) { scale[col0 + k] = sc[k] / ws; shift[col0 + k] = sh[k]; }
        }
        off += conv_tc_packed_bytes(l.cin, l.N);
    }
    int rc = upload(&m->conv.d_tower, host.data(), host.size());
    if (rc != LZ_OK) return rc;
    const float *dtab = reinterpret_cast<const float *>(m->conv.d_tower + tab_off);
    auto base = [&](int li, int N, int H, int nphase_in, int C_in) {
        ConvTc p;
        memset(&p, 0, sizeof(p));
        p.w = m->conv.d_tower + woff[li];
        p.scale = dtab + li * 256; p.shift = p.scale + 128;
        p.N = N; p.relu[0] = 1; p.relu[1] = 0;
        p.in = make_tcl(nullptr, C_in, H, H, nphase_in);
        for (int t = 0; t < 9; ++t) {
            const int ky = t / 3, kx = t % 3;
            if (nphase_in == 1) { p.tap_phase[t] = 0; p.tap_shift[t] = (ky - 1) * p.in.pitch + (kx - 1); }
            else {   // stride 2 on the 4-phase input: row 2y+ky-1 -> phase (ky+1)&1, offset -(ky==0)
                p.tap_phase[t] = (((ky + 1) & 1) * 2) + ((kx + 1) & 1);
                p.tap_shift[t] = (ky == 0 ? -p.in.pitch : 0) + (kx == 0 ? -1 : 0);
            }
        }
        pick_band(p);
        return p;
    };
    m->conv.tower_tc[0] = base(2, 2 * kC, h2, 4, c2);
    m->conv.tower_tc[1] = base(3, kC, h2, 1, kC);
    // ResBlocks: layers (li, li + 1) are conv1 and conv2 of one block
    auto block = [&](ResBlockTc &p, int li, int C, int H) {
        memset(&p, 0, sizeof(p));
        for (int c = 0; c < 2; ++c) {
            p.w[c] = m->conv.d_tower + woff[li + c];
            p.scale[c] = dtab + (li + c) * 256; p.shift[c] = p.scale[c] + 128;
        }
        p.in = make_tcl(nullptr, C, H, H, 1);
        for (int t = 0; t < 9; ++t) p.tap_shift[t] = (t / 3 - 1) * p.in.pitch + (t % 3 - 1);
        return resblock_tc_plan(p);
    };
    if ((rc = block(m->conv.tower_rb[0], 0, c2, h1))) return rc;
    if ((rc = block(m->conv.tower_rb[1], 4, kC, h2))) return rc;
    if ((rc = block(m->conv.tower_rb[2], 6, kC, h3))) return rc;
    return conv_tc_prepare_launch();
}

// ---- tensor-core tables (net_tc.cu): fp16 hi/lo weights, folded BN, action-bias planes, layer programs ----
static int pack_tc(lz_model *m, const Head &reward, const Head &value, const Head &policy)
{
    const lz_model_config &c = m->conv.cfg;
    const int A = c.action_space_size, n = c.num_res_blocks;
    const int hw = m->lat_h, P = hw * hw, nfc1 = 16 * P / 32;      // latent grid, pixels, FC1 stages (16 P inputs at most)
    const int nconv = 1 + 6 * n;
    const size_t conv_bytes = (size_t)tc_conv_layout_bytes();
    const size_t off_convw = 0;
    const size_t off_headw = off_convw + conv_bytes * nconv;
    const size_t off_bn = off_headw + tc_head_layout_bytes();
    const size_t off_headbn = off_bn + (size_t)nconv * 128 * 4;
    const size_t off_abias = off_headbn + 96 * 4;
    // FC weight stream of the heads (16 KB stages for the shared-memory ring of k_net_tc, fp16 hi / lo, the weights are the
    // tensor cores' M operand): 16 P / 32 FC1 stages covering all three heads, then one stage per 128-output tile of each head's FC2
    const std::string fc_names[3] = {"dynamics_network.fc_reward_head", "prediction_network.fc_value", "prediction_network.fc_policy"};
    const Head *fc_heads[3] = {&reward, &value, &policy};
    size_t fc_off2[3];
    size_t off_fc = (off_abias + (size_t)A * kC * P * 4 + 127) & ~(size_t)127;
    const size_t off_fc0 = off_fc;
    off_fc += (size_t)nfc1 * 12288;
    for (int h = 0; h < 3; ++h) {
        fc_off2[h] = off_fc - off_fc0;
        if (fc_heads[h]->hid > 0) off_fc += (size_t)((fc_heads[h]->K + 127) / 128) * 16384;      // EfficientZero: the reward head's FC part lives in ez.cu
    }
    const size_t total = off_fc;
    std::vector<unsigned char> host(total, 0);
    float *bn = reinterpret_cast<float *>(host.data() + off_bn);
    float *head_bn = reinterpret_cast<float *>(host.data() + off_headbn);
    float *abias = reinterpret_cast<float *>(host.data() + off_abias);

    std::vector<std::pair<std::string, std::string>> convs;   // (weight name, bn prefix)
    const std::string D = "dynamics_network.", Q = "prediction_network.", R = "representation_network.";
    convs.push_back({D + "conv.weight", D + "norm_common"});
    for (const std::string &pre : {D, Q, R})
        for (int i = 0; i < n; ++i) {
            const std::string b = pre + "resblocks." + std::to_string(i);
            convs.push_back({b + ".conv1.0.weight", b + ".conv1.1"});
            convs.push_back({b + ".conv2.0.weight", b + ".conv2.1"});
        }
    for (int ci = 0; ci < nconv; ++ci) {
        const int cin_total = (ci == 0) ? kC + A : kC;
        auto w = find_tensor(m, convs[ci].first, (size_t)kC * cin_total * 9);
        std::vector<float> scale, shift;
        if (!w || !fold_bn(m, convs[ci].second, kC, scale, shift)) return LZ_EINVAL;
        const float ws = tc_pack_conv3(w->data(), cin_total, kC, host.data() + off_convw + conv_bytes * ci);
        for (int k = 0; k < kC; ++k) { bn[ci * 128 + k] = scale[k] / ws; bn[ci * 128 + 64 + k] = shift[k]; }
        if (ci == 0) {   // one-hot action planes (muzero_model.py:341-369): border-aware tap sums, times the BN scale
            for (int a = 0; a < A; ++a)
                for (int co = 0; co < kC; ++co)
                    for (int y = 0; y < hw; ++y)
                        for (int x = 0; x < hw; ++x) {
                            float acc = 0.0f;
                            for (int ky = 0; ky < 3; ++ky)
                                for (int kx = 0; kx < 3; ++kx) {
                                    const int yy = y + ky - 1, xx = x + kx - 1;
                                    if (yy < 0 || yy >= hw || xx < 0 || xx >= hw) continue;
                                    acc += (*w)[((size_t)co * cin_total + kC + a) * 9 + ky * 3 + kx];
                                }
                            abias[(((size_t)a * 16 + co / 4) * P + y * hw + x) * 4 + co % 4] = acc * scale[co];   // k_net_tc's internal [c / 4][P][c % 4] layout
                        }
        }
    }
    // 1x1 heads
    struct HD { std::string conv, norm; int hc, nco, co_off; size_t hi, lo; int bn_off; };
    const HD heads[3] = {
        {D + "conv1x1_reward", D + "norm_reward", c.reward_head_channels, 16, 0, off_headw, off_headw + 2048, 0},
        {Q + "conv1x1_value", Q + "norm_value", c.value_head_channels, 32, 0, off_headw + 4096, off_headw + 8192, 32},
        {Q + "conv1x1_policy", Q + "norm_policy", c.policy_head_channels, 32, 16, off_headw + 4096, off_headw + 8192, 64},
    };
    for (const HD &h : heads) {
        auto w1 = find_tensor(m, h.conv + ".weight", (size_t)h.hc * kC), b1 = find_tensor(m, h.conv + ".bias", h.hc);
        std::vector<float> s1, t1;
        if (!w1 || !b1 || !fold_bn(m, h.norm, h.hc, s1, t1)) return LZ_EINVAL;
        const float ws = tc_pack_conv1(w1->data(), h.hc, h.nco, h.co_off, host.data() + h.hi, host.data() + h.lo);
        for (int i = 0; i < h.hc; ++i) {
            head_bn[h.bn_off + i] = s1[i] / ws;
            head_bn[h.bn_off + 16 + i] = t1[i] + s1[i] * (*b1)[i];
        }
    }
    float fc1_inv[3] = {1.0f, 1.0f, 1.0f}, fc2_inv[3] = {1.0f, 1.0f, 1.0f};
    for (int h = 0; h < 3; ++h) {
        const Head &H = *fc_heads[h];
        if (H.hid <= 0) continue;
        const int nin = H.hc * P;
        LZ_REQUIRE(H.hid <= 32 && H.K <= 608 && nin <= 16 * P, LZ_EINVAL, "lz_model_finalize: tensor-core path needs head hidden <= 32, head channels <= 16 and support <= 608");
        auto W0 = find_tensor(m, fc_names[h] + ".0.weight", (size_t)H.hid * nin), W3 = find_tensor(m, fc_names[h] + ".3.weight", (size_t)H.K * H.hid);
        if (!W0 || !W3) return LZ_EINVAL;
        auto maxabs = [](const std::vector<float> &w) {
            float mx = 0.0f;
            for (float v : w) mx = std::max(mx, fabsf(v));
            return mx;
        };
        const float s1 = pow2_scale(maxabs(*W0)), s2 = pow2_scale(maxabs(*W3));
        fc1_inv[h] = 1.0f / s1; fc2_inv[h] = 1.0f / s2;
        auto put = [&](unsigned char *hi, unsigned char *lo, size_t off, float v) {
            split_hi_lo(v, *reinterpret_cast<__half *>(hi + off), *reinterpret_cast<__half *>(lo + off));
        };
        // FC1: stage i = inputs [32 i, 32 i + 32): [k-step 2][hi 3 KB | lo 3 KB], each [kg 2][96 rows][8]; row = 32 h + unit.  Only the 96 real
        // rows are stored and streamed (the M = 128 MMA reads 32 rows of whatever follows into accumulator lanes 96-127, which nobody reads)
        unsigned char *f1 = host.data() + off_fc0;
        for (int i = 0; i < nin; ++i)
            for (int j = 0; j < H.hid; ++j) {
                const int kstep = i >> 4, kg = (i >> 3) & 1, e = i & 7;
                unsigned char *base = f1 + (size_t)(kstep >> 1) * 12288 + (size_t)(kstep & 1) * 6144;
                put(base, base + 3072, ((size_t)kg * 96 + h * 32 + j) * 16 + e * 2, (*W0)[(size_t)j * nin + i] * s1);
            }
        // FC2: tile mt = outputs [128 mt, 128 mt + 128): [hi 8 KB | lo 8 KB], each [kg 4][128 rows][8]
        unsigned char *f2 = host.data() + off_fc0 + fc_off2[h];
        for (int k = 0; k < H.K; ++k)
            for (int j = 0; j < H.hid; ++j) {
                unsigned char *base = f2 + (size_t)(k >> 7) * 16384;
                put(base, base + 8192, ((size_t)(j >> 3) * 128 + (k & 127)) * 16 + (j & 7) * 2, (*W3)[(size_t)k * H.hid + j] * s2);
            }
    }
    int rc = upload(&m->conv.d_tc, host.data(), total);
    if (rc != LZ_OK) return rc;
    TcNet base;
    memset(&base, 0, sizeof(base));
    base.convw = m->conv.d_tc + off_convw; base.headw = m->conv.d_tc + off_headw;
    base.bn = reinterpret_cast<const float *>(m->conv.d_tc + off_bn);
    base.head_bn = reinterpret_cast<const float *>(m->conv.d_tc + off_headbn);
    base.abias = reinterpret_cast<const float *>(m->conv.d_tc + off_abias);
    base.reward = reward; base.value = value; base.policy = policy;
    base.fcw = m->conv.d_tc + off_fc0;
    for (int h = 0; h < 3; ++h) {
        base.fc[h].fc2_off = (uint32_t)fc_off2[h];
        base.fc[h].nin = fc_heads[h]->hid > 0 ? fc_heads[h]->hc * P : 0;
        base.fc[h].K = fc_heads[h]->hid > 0 ? fc_heads[h]->K : 0;
        base.fc[h].fc1_inv = fc1_inv[h]; base.fc[h].fc2_inv = fc2_inv[h];
    }
    base.hc[0] = c.reward_head_channels; base.hc[1] = c.value_head_channels; base.hc[2] = c.policy_head_channels;
    base.A = A; base.support_min = c.support_min; base.support_step = c.support_step;
    base.hw = hw;
    // conv indices: 0 dyn conv | 1..2n dyn blocks | 2n+1..4n pred blocks | 4n+1..6n rep blocks
    TcNet rec = base, tail = base;
    int L = 0;
    rec.layer_w[L] = 0; rec.layer_flags[L++] = LF_RES | LF_STORE_RES | LF_ACT_BIAS;
    for (int i = 0; i < n; ++i) {
        rec.layer_w[L] = 1 + 2 * i; rec.layer_flags[L++] = 0;
        rec.layer_w[L] = 2 + 2 * i; rec.layer_flags[L++] = LF_RES | LF_STORE_RES | (i == n - 1 ? (LF_WRITE_LATENT | LF_HOOK_REWARD) : 0);
    }
    for (int i = 0; i < n; ++i) {
        rec.layer_w[L] = 2 * n + 1 + 2 * i; rec.layer_flags[L++] = 0;
        rec.layer_w[L] = 2 * n + 2 + 2 * i; rec.layer_flags[L++] = LF_RES | LF_STORE_RES | (i == n - 1 ? LF_HOOK_VALPOL : 0);
    }
    rec.nlayers = L; rec.has_reward = 1;
    L = 0;
    for (int i = 0; i < n; ++i) {
        tail.layer_w[L] = 4 * n + 1 + 2 * i; tail.layer_flags[L++] = 0;
        tail.layer_w[L] = 4 * n + 2 + 2 * i; tail.layer_flags[L++] = LF_RES | LF_STORE_RES | (i == n - 1 ? LF_WRITE_LATENT : 0);
    }
    for (int i = 0; i < n; ++i) {
        tail.layer_w[L] = 2 * n + 1 + 2 * i; tail.layer_flags[L++] = 0;
        tail.layer_w[L] = 2 * n + 2 + 2 * i; tail.layer_flags[L++] = LF_RES | LF_STORE_RES | (i == n - 1 ? LF_HOOK_VALPOL : 0);
    }
    tail.nlayers = L; tail.has_reward = 0;
    m->conv.tc_rec = rec; m->conv.tc_tail = tail;
    return tc_prepare_launch();
}

int conv_finalize(lz_model *m)
{
    const lz_model_config &c = m->conv.cfg;
    const int A = c.action_space_size;
    TablePacker P;
    ConvOff stem;
    HeadOff hr, hv, hp;
    const std::string R = "representation_network.downsample_net.", D = "dynamics_network.", Q = "prediction_network.";
    bool ok = pack_conv3(m, P, R + "conv1.weight", R + "norm1", c.obs_c, kC / 2, stem) &&
              pack_head(m, P, m->vp ? std::string() : D + "fc_reward_head", c.reward_head_channels, c.reward_hidden, m->K, hr) &&
              pack_head(m, P, Q + "fc_value", c.value_head_channels, c.value_hidden, m->K, hv) &&
              pack_head(m, P, Q + "fc_policy", c.policy_head_channels, c.policy_hidden, A, hp);
    if (!ok) return LZ_EINVAL;
    if (m->vp) {      // the value-prefix head on the reward_head_channels x P LSTM input (efficientzero_model.py:511-525, 556-569)
        const int rc0 = ez_finalize(m, c.reward_head_channels * m->lat_h * m->lat_w, c.reward_hidden, true);
        if (rc0 != LZ_OK) return rc0;
    }
    int rc = upload(&m->conv.d_weights, P.host.data(), P.host.size() * sizeof(float));
    if (rc != LZ_OK) return rc;
    const float *base = m->conv.d_weights;
    auto mkh = [&](const HeadOff &o) {
        Head H;
        H.s2 = o.hid ? base + o.s2 : nullptr; H.t2 = o.hid ? base + o.t2 : nullptr; H.b2 = o.hid ? base + o.b2 : nullptr;
        H.hc = o.hc; H.hid = o.hid; H.K = o.K;
        return H;
    };

    // DownSample geometry: conv s2 p1: h -> (h-1)/2+1
    const int h0 = c.obs_h, h1 = (h0 - 1) / 2 + 1, h2 = (h1 - 1) / 2 + 1, h3 = (h2 - 1) / 2 + 1;
    ConvG &S0 = m->conv.stem;
    S0.w = base + stem.w; S0.scale = base + stem.scale; S0.shift = base + stem.shift;
    S0.cin = stem.cin; S0.cout = stem.cout;
    S0.hin = S0.win = h0; S0.hout = S0.wout = h1;
    // host copy of the stem's weights / folded BatchNorm for k_stem4_tcl (kernel-parameter operands)
    m->conv.stem_valid = 0;
    if (stem.cin == 4 && stem.cout == 32 && h0 % 4 == 0 && (h0 / 2) <= 256) {
        m->conv.stem_params.assign(sizeof(StemP) / sizeof(float), 0.0f);
        StemP &SP = *reinterpret_cast<StemP *>(m->conv.stem_params.data());
        memcpy(SP.w, P.host.data() + stem.w, sizeof(SP.w));
        memcpy(SP.scale, P.host.data() + stem.scale, sizeof(SP.scale));
        memcpy(SP.shift, P.host.data() + stem.shift, sizeof(SP.shift));
        m->conv.stem_valid = 1;
    }
    const int h4 = (h3 - 1) / 2 + 1, grid = h0 == 64 ? h3 : h4;      // 64 px: no pooling2
    LZ_REQUIRE(grid == m->lat_h && (grid == 6 || grid == 8), LZ_EINVAL, "lz_model_finalize: latent grid %d is neither 6 nor 8", grid);
    // opt-in shared memory size, set once outside any stream capture
    LZ_CUDA_CHECK(cudaFuncSetAttribute(k_conv3x3_generic<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    rc = pack_tc(m, mkh(hr), mkh(hv), mkh(hp));
    if (rc != LZ_OK) return rc;
    return pack_tower_tc(m);
}

// lz_model_debug_net_stage of the latent-grid network: which 1 is the tail program (representation ResBlocks + prediction) on
// the DownSample output d_in
int conv_debug_stage(lz_model *m, int which, int B, const float *d_latent, const int32_t *d_action, int stage, void *d_out,
                     size_t out_bytes, int32_t *h_info, cudaStream_t st)
{
    TcNet net = which ? m->conv.tc_tail : m->conv.tc_rec;          // a copy: the model's programs stay as they are
    const int nl = net.nlayers, K = m->K, A = m->A;
    const bool ez = m->vp && which == 0;
    const int nfeat = ez ? m->ez.net.nin : 0;
    LZ_REQUIRE(stage <= nl, LZ_EINVAL, "lz_model_debug_net_stage: stage %d past the %d layers of the program", stage, nl);
    {
        int rc = model_reserve(m, B, st);
        if (rc != LZ_OK) return rc;
    }
    const size_t nfl = stage < nl ? (size_t)B * m->latent_floats : (size_t)B * (2 * K + 2 * A + 4 + nfeat);
    LZ_REQUIRE(out_bytes >= nfl * sizeof(float), LZ_EINVAL, "lz_model_debug_net_stage: stage %d needs %zu bytes, got %zu", stage,
               nfl * sizeof(float), out_bytes);
    float *o = reinterpret_cast<float *>(d_out);
    TcIO t;
    memset(&t, 0, sizeof(t));
    t.B = B; t.npass = m->npass;
    t.latent_base = d_latent; t.action = which ? nullptr : d_action;
    t.skip_scratch = m->conv.tc_skip;
    t.ez_feat = ez ? m->ez.feat : nullptr;
    int rc;
    if (stage < nl) {
        // the program cut after layer `stage`, whose output is the only latent written
        net.nlayers = stage + 1;
        for (int L = 0; L <= stage; ++L) net.layer_flags[L] &= ~LF_WRITE_LATENT;
        net.layer_flags[stage] |= LF_WRITE_LATENT;
        t.latent_out = o;
        tc_describe(net, t, h_info);
        return tc_launch(net, t, st);
    }
    // the whole program: [reward logits B x K | value logits B x K | policy logits B x A | reward B | value B] with the raw logits
    // requested, then [policy logits B x A | reward B | value B] without them (the joint categorical read-out), then ez_feat
    LZ_CUDA_CHECK(cudaMemsetAsync(d_out, 0, nfl * sizeof(float), st));
    float *rl = o, *vl = rl + (size_t)B * K, *pl = vl + (size_t)B * K, *r = pl + (size_t)B * A, *v = r + B;
    float *pl2 = v + B, *r2 = pl2 + (size_t)B * A, *v2 = r2 + B, *feat = v2 + B;
    if (ez) t.ez_feat = feat;
    const bool rew = net.has_reward && !ez;
    t.policy_logits = pl; t.value_logits = vl; t.value = v;
    t.reward_logits = rew ? rl : nullptr; t.reward = rew ? r : nullptr;
    tc_describe(net, t, h_info);
    if ((rc = tc_launch(net, t, st))) return rc;
    t.policy_logits = pl2; t.value_logits = nullptr; t.value = v2;
    t.reward_logits = nullptr; t.reward = rew ? r2 : nullptr;
    return tc_launch(net, t, st);
}

}  // namespace lz

using namespace lz;

extern "C" {

/* debug: replace the layer program of the tensor-core recurrent kernel (which == 0) or tail kernel (which == 1) */
int lz_model_debug_tc_program(lz_model *m, int which, int nlayers, const int *layer_w, const int *layer_flags, int has_reward)
{
    LZ_REQUIRE(m && m->finalized && m->family == ModelFamily::Conv && nlayers >= 1 && nlayers <= kTcMaxLayers, LZ_EINVAL, "lz_model_debug_tc_program: bad argument");
    ++m->generation;
    TcNet &n = which ? m->conv.tc_tail : m->conv.tc_rec;
    n.nlayers = nlayers;
    for (int i = 0; i < nlayers; ++i) { n.layer_w[i] = layer_w[i]; n.layer_flags[i] = layer_flags[i]; }
    n.has_reward = has_reward;
    return LZ_OK;
}

int lz_model_debug_tower_stage(lz_model *m, int B, const float *d_obs, const uint8_t *d_obs_u8, int stage, void *d_out,
                               size_t out_bytes, int32_t *h_info, lz_stream s)
{
    LZ_REQUIRE(m && B > 0 && (d_obs == nullptr) != (d_obs_u8 == nullptr) && d_out && h_info && stage >= 0 && stage <= 8, LZ_EINVAL,
               "lz_model_debug_tower_stage: bad argument");
    LZ_REQUIRE(m->finalized && m->family == ModelFamily::Conv, LZ_ESTATE, "lz_model_debug_tower_stage: not a finalized conv model with a tensor-core tower");
    if (B > m->conv.ws_B) {
        int rc = model_reserve(m, B, (cudaStream_t)s);
        if (rc != LZ_OK) return rc;
    }
    LZ_REQUIRE(B <= m->conv.ws_B, LZ_ESTATE, "lz_model_debug_tower_stage: workspace sized for %d roots, got %d", m->conv.ws_B, B);
    // stage -> the tensor it leaves and the launch that wrote it (tower_tc_run)
    const Tcl *outs[8] = {&m->conv.T0, &m->conv.T1, &m->conv.U0, &m->conv.U1, &m->conv.U2, &m->conv.U0, &m->conv.V0, &m->conv.V1};
    int32_t info[10] = {0};
    size_t bytes;
    if (stage < 8) {
        const Tcl &t = *outs[stage];
        info[0] = t.C; info[1] = t.H; info[2] = t.W; info[3] = t.nphase; info[4] = t.plane_rows;
        bytes = (size_t)B * t.img_stride;
    } else {
        info[0] = kC; info[1] = m->lat_h; info[2] = m->lat_h;                // fp32 NCHW: nphase = plane_rows = 0
        bytes = (size_t)B * m->latent_floats * sizeof(float);
    }
    LZ_REQUIRE(out_bytes >= bytes, LZ_EINVAL, "lz_model_debug_tower_stage: stage %d needs %zu bytes, got %zu", stage, bytes, out_bytes);
    const ConvG &S0 = m->conv.stem;
    auto pool_ctas = [&](const Tcl &in, int hout) {
        return (int)std::min<size_t>(((size_t)B * (in.C / 8) * hout * hout + 255) / 256, kNumSMs * 32);
    };
    auto plan = [&](const auto &p) {     // ResBlockTc or ConvTc
        info[5] = p.G; info[6] = p.band_h; info[7] = p.stages;
        info[8] = (B + p.G - 1) / p.G * ((p.in.H + p.band_h - 1) / p.band_h);
    };
    switch (stage) {
        case 0:
            info[5] = 1;
            if (m->conv.stem_valid) {
                const int rows_per_cta = std::max(1, 256 / S0.wout);
                info[6] = rows_per_cta;
                info[8] = ceil_div(S0.hout, rows_per_cta) * B;
            } else {
                info[8] = ceil_div(S0.hout * S0.wout, 128) * (S0.cout / 32) * B;
            }
            break;
        case 1: plan(m->conv.tower_rb[0]); break;
        case 2: case 3: plan(m->conv.tower_tc[0]); break;
        case 4: plan(m->conv.tower_tc[1]); break;
        case 5: plan(m->conv.tower_rb[1]); break;
        case 6: info[5] = 1; info[8] = pool_ctas(m->conv.U0, m->conv.V0.H); break;
        case 7: plan(m->conv.tower_rb[2]); break;
        default: info[5] = 1; info[8] = m->lat_h == 8 ? tcl_to_nchw_ctas(m->conv.V1, B) : pool_ctas(m->conv.V1, m->lat_h); break;
    }
    info[9] = m->npass;
    const cudaStream_t st = (cudaStream_t)s;
    int rc = tower_tc_run(m, B, d_obs, stage == 8 ? reinterpret_cast<float *>(d_out) : nullptr, st, d_obs_u8, stage);
    if (rc != LZ_OK) return rc;
    if (stage < 8) LZ_CUDA_CHECK(cudaMemcpyAsync(d_out, outs[stage]->base, bytes, cudaMemcpyDeviceToDevice, st));
    memcpy(h_info, info, sizeof(info));
    return LZ_OK;
}

}  // extern "C"
