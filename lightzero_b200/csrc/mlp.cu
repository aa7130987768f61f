// mlp.cu -- MuZeroModelMLP forward paths (vector observations; BASELINE config 1, CartPole plumbing) as fused
// fp32 CUDA kernels.  Replaces lzero/model/muzero_model_mlp.py:146-205 (initial/recurrent_inference),
// :241-295 (_dynamics one-hot concat), :417-442 (DynamicsNetwork.forward), lzero/model/common.py:845-850
// (RepresentationNetworkMLP.forward), :1280-1292 (PredictionNetworkMLP.forward), eval mode.
//
// The whole network for up to 4 roots runs in one CTA of 128 threads: thread j owns output neuron j of the
// current dense layer, the weight matrix is stored input-major so a layer is `in` coalesced 512-byte row
// loads (8 in flight), activations ping-pong through shared memory.  Work per root is ~150 kMAC: this
// path exists for interface completeness (the search engine accepts either model), not for throughput.
#include <math.h>
#include <string.h>

#include <algorithm>

#include "model.cuh"

namespace lz {

constexpr int kMlpThreads = 128, kMlpRoots = 4, kMlpWidth = 160, kMlpK = 608;

__device__ __forceinline__ float gelu_tanh(float x)
{
    const float k0 = 0.7978845608028654f, k1 = 0.044715f;      // sqrt(2/pi), torch.nn.GELU(approximate='tanh')
    return 0.5f * x * (1.0f + tanhf(k0 * (x + k1 * x * x * x)));
}

// y[r][j] = act(scale[j] * sum_i x[r][i] * wt[i][j] + shift[j]); one-hot action rows are appended inputs
__device__ __forceinline__ void dense(const Dense &L, const float *x, float *y, int ldx, int ldy, const int *act_row /*[RB] or null*/)
{
    for (int j = threadIdx.x; j < L.out; j += kMlpThreads) {
        float acc[kMlpRoots];
#pragma unroll
        for (int r = 0; r < kMlpRoots; ++r) acc[r] = 0.0f;
        const int nin = act_row ? L.in - L.nact : L.in;
        for (int i = 0; i < nin; i += 8) {
            float w[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) w[u] = (i + u < nin) ? __ldg(L.wt + (size_t)(i + u) * L.out + j) : 0.0f;
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int ii = min(i + u, nin - 1);
#pragma unroll
                for (int r = 0; r < kMlpRoots; ++r) acc[r] = fmaf(x[r * ldx + ii], w[u], acc[r]);
            }
        }
        if (act_row) {
#pragma unroll
            for (int r = 0; r < kMlpRoots; ++r) acc[r] += __ldg(L.wt + (size_t)(nin + act_row[r]) * L.out + j);
        }
        const float s = __ldg(L.scale + j), t = __ldg(L.shift + j);
#pragma unroll
        for (int r = 0; r < kMlpRoots; ++r) {
            float v = fmaf(acc[r], s, t);
            if (L.act == 1) v = fmaxf(v, 0.0f);
            else if (L.act == 2) v = gelu_tanh(v);
            y[r * ldy + j] = v;
        }
    }
    __syncthreads();
}

// Test hook of lz_model_debug_net_stage: the kTap instantiations of the kernels below stop after the layer numbered `cut` and
// write its fp32 output rows [B][width] to `out`, and nothing else.  Inference and the searches launch the kTap = false
// instantiations, in which every tap is a compile-time no-op.
struct MlpTap {
    float *out;
    int cut;
};

// true when the program stops here: `stage` is the cut, whose rows y [RB][ldy] (width valid columns) are written
template <bool kTap>
__device__ __forceinline__ bool tap(const MlpTap &t, int stage, const float *y, int ldy, int width, int root0, int B)
{
    if constexpr (!kTap) {
        return false;
    } else {
        if (stage != t.cut) return false;
        for (int i = threadIdx.x; i < kMlpRoots * width; i += kMlpThreads) {
            const int r = i / width, c = i - r * width, b = root0 + r;
            if (b < B) t.out[(size_t)b * width + c] = y[r * ldy + c];
        }
        return true;
    }
}

// prediction network + outputs for the latents in `lat` (shared, [RB][kMlpWidth]); its layers are tap stages s0 .. s0 + 5
template <bool kTap>
__device__ __forceinline__ void mlp_predict(const MlpNet &net, const float *lat, float *b0, float *b1, float *logits,
                                            int root0, int B, float *o_value, float *o_policy, float *o_value_logits,
                                            const MlpTap &tp, int s0)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    dense(net.pc0, lat, b0, kMlpWidth, kMlpWidth, nullptr);
    if (tap<kTap>(tp, s0, b0, kMlpWidth, net.pc0.out, root0, B)) return;
    dense(net.pc1, b0, b1, kMlpWidth, kMlpWidth, nullptr);
    if (tap<kTap>(tp, s0 + 1, b1, kMlpWidth, net.pc1.out, root0, B)) return;
    dense(net.v0, b1, b0, kMlpWidth, kMlpWidth, nullptr);
    if (tap<kTap>(tp, s0 + 2, b0, kMlpWidth, net.v0.out, root0, B)) return;
    dense(net.v1, b0, logits, kMlpWidth, kMlpK, nullptr);
    if (tap<kTap>(tp, s0 + 3, logits, kMlpK, net.v1.out, root0, B)) return;
    if (root0 + warp < B) {
        const float v = categorical_to_scalar(logits + warp * kMlpK, net.v1.out, net.support_min, net.support_step, lane);
        if (lane == 0 && o_value) o_value[root0 + warp] = v;
        if (o_value_logits)
            for (int k = lane; k < net.v1.out; k += 32) o_value_logits[(size_t)(root0 + warp) * net.v1.out + k] = logits[warp * kMlpK + k];
    }
    __syncthreads();
    dense(net.p0, b1, b0, kMlpWidth, kMlpWidth, nullptr);
    if (tap<kTap>(tp, s0 + 4, b0, kMlpWidth, net.p0.out, root0, B)) return;
    dense(net.p1, b0, logits, kMlpWidth, kMlpK, nullptr);
    if (tap<kTap>(tp, s0 + 5, logits, kMlpK, net.p1.out, root0, B)) return;
    if (root0 + warp < B && o_policy)
        for (int a = lane; a < net.A; a += 32) o_policy[(size_t)(root0 + warp) * net.A + a] = logits[warp * kMlpK + a];
    __syncthreads();
}

// tap stages: with res_connection_in_dynamics fc_dynamics_1.0 (with the one-hot rows) 0, fc_dynamics_1.3 1, + latent 2,
// fc_dynamics_2.0 3, fc_dynamics_2.3 4, reward head 5 6, prediction 7 .. 12; without it fc_dynamics.0 0, fc_dynamics.3 1,
// reward head 2 3, prediction 4 .. 9
template <bool kTap>
__global__ void __launch_bounds__(kMlpThreads) k_mlp_recurrent(MlpNet net, RecIO io, MlpTap tp)
{
    __shared__ float xa[kMlpRoots * kMlpWidth], xb[kMlpRoots * kMlpWidth], xc[kMlpRoots * kMlpWidth], logits[kMlpRoots * kMlpK];
    __shared__ int act_row[kMlpRoots];
    const int root0 = blockIdx.x * kMlpRoots, Ld = net.latent;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < kMlpRoots * Ld; i += kMlpThreads) {
        const int r = i / Ld, c = i - r * Ld, b = root0 + r;
        float v = 0.0f;
        if (b < io.B) {
            const size_t slot = io.ix ? (size_t)io.ix[b] : 0;
            v = io.latent_base[slot * io.slot_stride + (size_t)b * Ld + c];
        }
        xa[r * kMlpWidth + c] = v;
    }
    if (threadIdx.x < kMlpRoots) {
        const int b = root0 + threadIdx.x;
        act_row[threadIdx.x] = b < io.B ? min(max(io.action[b], 0), net.A - 1) : 0;
    }
    __syncthreads();
    const float *nxt, *enc;
    if (net.res) {                                   // muzero_model_mlp.py:428-434
        dense(net.d1a, xa, xb, kMlpWidth, kMlpWidth, act_row);
        if (tap<kTap>(tp, 0, xb, kMlpWidth, Ld, root0, io.B)) return;
        dense(net.d1b, xb, xc, kMlpWidth, kMlpWidth, nullptr);
        if (tap<kTap>(tp, 1, xc, kMlpWidth, Ld, root0, io.B)) return;
        for (int i = threadIdx.x; i < kMlpRoots * Ld; i += kMlpThreads) {
            const int r = i / Ld, c = i - r * Ld;
            xc[r * kMlpWidth + c] += xa[r * kMlpWidth + c];
        }
        __syncthreads();
        if (tap<kTap>(tp, 2, xc, kMlpWidth, Ld, root0, io.B)) return;
        dense(net.d2a, xc, xb, kMlpWidth, kMlpWidth, nullptr);
        if (tap<kTap>(tp, 3, xb, kMlpWidth, Ld, root0, io.B)) return;
        dense(net.d2b, xb, xa, kMlpWidth, kMlpWidth, nullptr);
        if (tap<kTap>(tp, 4, xa, kMlpWidth, Ld, root0, io.B)) return;
        nxt = xc; enc = xa;
    } else {                                         // :436-438
        dense(net.d1a, xa, xb, kMlpWidth, kMlpWidth, act_row);
        if (tap<kTap>(tp, 0, xb, kMlpWidth, Ld, root0, io.B)) return;
        dense(net.d1b, xb, xc, kMlpWidth, kMlpWidth, nullptr);
        if (tap<kTap>(tp, 1, xc, kMlpWidth, Ld, root0, io.B)) return;
        nxt = xc; enc = xc;
    }
    const int sr = net.res ? 5 : 2;                  // tap stage of the reward head's first layer
    if (io.next_latent)
        for (int i = threadIdx.x; i < kMlpRoots * Ld; i += kMlpThreads) {
            const int r = i / Ld, c = i - r * Ld, b = root0 + r;
            if (b < io.B) io.next_latent[(size_t)b * Ld + c] = nxt[r * kMlpWidth + c];
        }
    // reward head (:440)
    dense(net.r0, enc, xb, kMlpWidth, kMlpWidth, nullptr);
    if (tap<kTap>(tp, sr, xb, kMlpWidth, net.r0.out, root0, io.B)) return;
    dense(net.r1, xb, logits, kMlpWidth, kMlpK, nullptr);
    if (tap<kTap>(tp, sr + 1, logits, kMlpK, net.r1.out, root0, io.B)) return;
    if (root0 + warp < io.B) {
        const float rv = categorical_to_scalar(logits + warp * kMlpK, net.r1.out, net.support_min, net.support_step, lane);
        if (lane == 0 && io.reward) io.reward[root0 + warp] = rv;
        if (io.reward_logits)
            for (int k = lane; k < net.r1.out; k += 32) io.reward_logits[(size_t)(root0 + warp) * net.r1.out + k] = logits[warp * kMlpK + k];
    }
    __syncthreads();
    // prediction on the next latent: nxt lives in xc; xa / xb are scratch (enc no longer needed)
    mlp_predict<kTap>(net, nxt, xa, xb, logits, root0, io.B, io.value, io.policy_logits, io.value_logits, tp, sr + 2);
}

// tap stages: fc_representation.0 (+ BN + GELU) 0, fc_representation.3 1, LayerNorm 2, prediction 3 .. 8
template <bool kTap>
__global__ void __launch_bounds__(kMlpThreads) k_mlp_initial(MlpNet net, const float *obs, TailIO io, MlpTap tp)
{
    __shared__ float xa[kMlpRoots * kMlpWidth], xb[kMlpRoots * kMlpWidth], xc[kMlpRoots * kMlpWidth], logits[kMlpRoots * kMlpK];
    const int root0 = blockIdx.x * kMlpRoots, Ld = net.latent;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < kMlpRoots * net.obs_dim; i += kMlpThreads) {
        const int r = i / net.obs_dim, c = i - r * net.obs_dim, b = root0 + r;
        xa[r * kMlpWidth + c] = b < io.B ? obs[(size_t)b * net.obs_dim + c] : 0.0f;
    }
    __syncthreads();
    dense(net.e0, xa, xb, kMlpWidth, kMlpWidth, nullptr);          // Linear + BN + GELU(tanh)
    if (tap<kTap>(tp, 0, xb, kMlpWidth, Ld, root0, io.B)) return;
    dense(net.e1, xb, xc, kMlpWidth, kMlpWidth, nullptr);          // Linear
    if (tap<kTap>(tp, 1, xc, kMlpWidth, Ld, root0, io.B)) return;
    {   // nn.LayerNorm(latent), eps 1e-5, biased variance: one warp per root
        float s = 0.0f;
        for (int c = lane; c < Ld; c += 32) s += xc[warp * kMlpWidth + c];
        const float mean = warp_sum(s) / (float)Ld;
        float q = 0.0f;
        for (int c = lane; c < Ld; c += 32) { const float d = xc[warp * kMlpWidth + c] - mean; q += d * d; }
        const float rstd = rsqrtf(warp_sum(q) / (float)Ld + 1e-5f);
        for (int c = lane; c < Ld; c += 32)
            xc[warp * kMlpWidth + c] = (xc[warp * kMlpWidth + c] - mean) * rstd * __ldg(net.ln_w + c) + __ldg(net.ln_b + c);
    }
    __syncthreads();
    if (tap<kTap>(tp, 2, xc, kMlpWidth, Ld, root0, io.B)) return;
    for (int i = threadIdx.x; i < kMlpRoots * Ld; i += kMlpThreads) {
        const int r = i / Ld, c = i - r * Ld, b = root0 + r;
        if (b < io.B) {
            if (io.latent) io.latent[(size_t)b * Ld + c] = xc[r * kMlpWidth + c];
            if (io.latent2) io.latent2[(size_t)b * Ld + c] = xc[r * kMlpWidth + c];
        }
    }
    mlp_predict<kTap>(net, xc, xa, xb, logits, root0, io.B, io.value, io.policy_logits, io.value_logits, tp, 3);
}

int mlp_recurrent(lz_model *m, const RecIO &io, cudaStream_t s)
{
    k_mlp_recurrent<false><<<ceil_div(io.B, kMlpRoots), kMlpThreads, 0, s>>>(m->mlp.net, io, MlpTap{});
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

int mlp_initial(lz_model *m, int B, const float *d_obs, const TailIO &io_in, cudaStream_t s)
{
    TailIO io = io_in;
    io.B = B;
    k_mlp_initial<false><<<ceil_div(B, kMlpRoots), kMlpThreads, 0, s>>>(m->mlp.net, d_obs, io, MlpTap{});
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

// lz_model_debug_net_stage of the fp32 MLP kernels: the kTap instantiations cut after dense layer `stage`; stage == D (the
// number of tap stages) launches the production kernel with every output in d_out
int mlp_debug_stage(lz_model *m, int which, int B, const float *d_in, const int32_t *d_action, int stage, void *d_out,
                    size_t out_bytes, int32_t *h_info, cudaStream_t s)
{
    const MlpNet &n = m->mlp.net;
    const int L = n.latent, K = m->K, A = n.A;
    int w[16], D = 0;                                // output width of each tap stage, in program order
    if (which) {
        w[D++] = L; w[D++] = L; w[D++] = L;
    } else {
        w[D++] = L; w[D++] = L;
        if (n.res) { w[D++] = L; w[D++] = L; w[D++] = L; }
        w[D++] = n.r0.out; w[D++] = K;
    }
    w[D++] = L; w[D++] = L; w[D++] = n.v0.out; w[D++] = K; w[D++] = n.p0.out; w[D++] = A;
    LZ_REQUIRE(stage <= D, LZ_EINVAL, "lz_model_debug_net_stage: stage %d past the %d dense layers of the program", stage, D);
    const size_t nfl = stage < D ? (size_t)B * w[stage] : (size_t)B * (L + 2 * K + A + 2);
    LZ_REQUIRE(out_bytes >= nfl * sizeof(float), LZ_EINVAL, "lz_model_debug_net_stage: stage %d needs %zu bytes, got %zu", stage,
               nfl * sizeof(float), out_bytes);
    const int ctas = ceil_div(B, kMlpRoots);
    const int32_t info[8] = {kMlpRoots, ctas, B - (ctas - 1) * kMlpRoots, D, stage < D ? w[stage] : 0, 0, 0, 0};
    memcpy(h_info, info, sizeof(info));
    float *o = reinterpret_cast<float *>(d_out);
    const MlpTap tp{o, stage};
    if (which) {
        TailIO io;
        memset(&io, 0, sizeof(io));
        io.B = B;
        if (stage < D) {
            k_mlp_initial<true><<<ctas, kMlpThreads, 0, s>>>(n, d_in, io, tp);
        } else {                                     // [latent B x L | value logits B x K | policy logits B x A | value B]
            io.latent = o; io.value_logits = o + (size_t)B * L; io.policy_logits = io.value_logits + (size_t)B * K;
            io.value = io.policy_logits + (size_t)B * A;
            k_mlp_initial<false><<<ctas, kMlpThreads, 0, s>>>(n, d_in, io, MlpTap{});
        }
    } else {
        RecIO io;
        memset(&io, 0, sizeof(io));
        io.B = B; io.latent_base = d_in; io.action = d_action;
        if (stage < D) {
            k_mlp_recurrent<true><<<ctas, kMlpThreads, 0, s>>>(n, io, tp);
        } else {                                     // the same, then [reward logits B x K | reward B]
            io.next_latent = o; io.value_logits = o + (size_t)B * L; io.policy_logits = io.value_logits + (size_t)B * K;
            io.value = io.policy_logits + (size_t)B * A; io.reward_logits = io.value + B; io.reward = io.reward_logits + (size_t)B * K;
            k_mlp_recurrent<false><<<ctas, kMlpThreads, 0, s>>>(n, io, MlpTap{});
        }
    }
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

// ---- weights ----------------------------------------------------------------------------------
struct DenseOff { size_t wt, scale, shift; int in, out, act, nact; };

// Linear `lin` (weight [out][in], bias [out]) optionally followed by eval BatchNorm1d `bn`
static bool pack_dense(lz_model *m, TablePacker &P, const std::string &lin, const std::string &bn, int in, int out, int act,
                       int nact, DenseOff &o)
{
    auto W = find_tensor(m, lin + ".weight", (size_t)out * in), b = find_tensor(m, lin + ".bias", out);
    if (!W || !b) return false;
    std::vector<float> scale(out, 1.0f), shift(*b);
    if (!bn.empty() && !fold_bn_linear(m, bn, *b, scale, shift)) return false;
    std::vector<float> wt((size_t)in * out);
    for (int j = 0; j < out; ++j)
        for (int i = 0; i < in; ++i) wt[(size_t)i * out + j] = (*W)[(size_t)j * in + i];
    o.wt = P.add(wt); o.scale = P.add(scale); o.shift = P.add(shift);
    o.in = in; o.out = out; o.act = act; o.nact = nact;
    return true;
}

int mlp_finalize(lz_model *m)
{
    const lz_mlp_config &c = m->mlp.cfg;
    const int L = c.latent_dim, A = c.action_space_size, K = m->K;
    TablePacker P;
    DenseOff e0, e1, d1a, d1b, d2a, d2b, r0, r1, pc0, pc1, v0, v1, p0, p1;
    memset(&d2a, 0, sizeof(d2a)); memset(&d2b, 0, sizeof(d2b));
    const std::string R = "representation_network.", D = "dynamics_network.", Q = "prediction_network.";
    bool ok = pack_dense(m, P, R + "fc_representation.0", R + "fc_representation.1", c.obs_dim, L, 2, 0, e0) &&
              pack_dense(m, P, R + "fc_representation.3", "", L, L, 0, 0, e1);
    if (ok && c.res_connection_in_dynamics)
        ok = pack_dense(m, P, D + "fc_dynamics_1.0", D + "fc_dynamics_1.1", L + A, L, 1, A, d1a) &&
             pack_dense(m, P, D + "fc_dynamics_1.3", D + "fc_dynamics_1.4", L, L, 1, 0, d1b) &&
             pack_dense(m, P, D + "fc_dynamics_2.0", D + "fc_dynamics_2.1", L, L, 1, 0, d2a) &&
             pack_dense(m, P, D + "fc_dynamics_2.3", D + "fc_dynamics_2.4", L, L, 1, 0, d2b);
    else if (ok)
        ok = pack_dense(m, P, D + "fc_dynamics.0", D + "fc_dynamics.1", L + A, L, 1, A, d1a) &&
             pack_dense(m, P, D + "fc_dynamics.3", D + "fc_dynamics.4", L, L, 1, 0, d1b);
    ok = ok && pack_dense(m, P, D + "fc_reward_head.0", D + "fc_reward_head.1", L, c.reward_hidden, 1, 0, r0) &&
         pack_dense(m, P, D + "fc_reward_head.3", "", c.reward_hidden, K, 0, 0, r1) &&
         pack_dense(m, P, Q + "fc_prediction_common.0", Q + "fc_prediction_common.1", L, L, 1, 0, pc0) &&
         pack_dense(m, P, Q + "fc_prediction_common.3", Q + "fc_prediction_common.4", L, L, 1, 0, pc1) &&
         pack_dense(m, P, Q + "fc_value_head.0", Q + "fc_value_head.1", L, c.value_hidden, 1, 0, v0) &&
         pack_dense(m, P, Q + "fc_value_head.3", "", c.value_hidden, K, 0, 0, v1) &&
         pack_dense(m, P, Q + "fc_policy_head.0", Q + "fc_policy_head.1", L, c.policy_hidden, 1, 0, p0) &&
         pack_dense(m, P, Q + "fc_policy_head.3", "", c.policy_hidden, A, 0, 0, p1);
    if (!ok) return LZ_EINVAL;
    auto lw = find_tensor(m, R + "norm.weight", L), lb = find_tensor(m, R + "norm.bias", L);
    if (!lw || !lb) return LZ_EINVAL;
    const size_t o_lw = P.add(*lw), o_lb = P.add(*lb);
    int rc = upload(&m->mlp.d_weights, P.host.data(), P.host.size() * sizeof(float));
    if (rc != LZ_OK) return rc;
    const float *base = m->mlp.d_weights;
    auto mk = [&](const DenseOff &o) { Dense d; d.wt = base + o.wt; d.scale = base + o.scale; d.shift = base + o.shift; d.in = o.in; d.out = o.out; d.act = o.act; d.nact = o.nact; return d; };
    MlpNet &n = m->mlp.net;
    memset(&n, 0, sizeof(n));
    n.e0 = mk(e0); n.e1 = mk(e1); n.d1a = mk(d1a); n.d1b = mk(d1b);
    if (c.res_connection_in_dynamics) { n.d2a = mk(d2a); n.d2b = mk(d2b); }
    n.r0 = mk(r0); n.r1 = mk(r1); n.pc0 = mk(pc0); n.pc1 = mk(pc1); n.v0 = mk(v0); n.v1 = mk(v1); n.p0 = mk(p0); n.p1 = mk(p1);
    n.ln_w = base + o_lw; n.ln_b = base + o_lb;
    n.latent = L; n.obs_dim = c.obs_dim; n.A = A; n.res = c.res_connection_in_dynamics;
    n.support_min = c.support_min; n.support_step = c.support_step;
    return LZ_OK;
}

}  // namespace lz

using namespace lz;

// The fp32 kernels above take the configs they were sized for; every other config inside k_mez_tc's envelope (mlp_tc.cu) runs
// there, as the MlpTc family.  The choice follows from the config alone, and a config both take stays on these kernels, so its
// outputs do not change.
static bool mlp_fits(const lz_mlp_config &c)
{
    return c.latent_dim >= 8 && c.latent_dim <= 128 && c.obs_dim >= 1 && c.obs_dim <= kMlpWidth && c.action_space_size >= 1 &&
           c.latent_dim + c.action_space_size <= kMlpWidth && c.reward_hidden <= kMlpWidth && c.value_hidden <= kMlpWidth &&
           c.policy_hidden <= kMlpWidth;
}

static bool mez_fits(const lz_mlp_config &c)
{
    auto hid = [](int h) { return h >= 1 && h <= kMezMaxHid; };
    return c.latent_dim >= 32 && c.latent_dim <= kMezMaxL && c.latent_dim % 32 == 0 && c.obs_dim >= 1 && c.obs_dim <= kMezMaxObs &&
           c.action_space_size >= 1 && c.action_space_size <= kMezMaxOut && hid(c.reward_hidden) && hid(c.value_hidden) &&
           hid(c.policy_hidden);
}

extern "C" int lz_model_create_mlp(const lz_mlp_config *cfg, lz_model **out)
{
    LZ_REQUIRE(cfg && out, LZ_EINVAL, "lz_model_create_mlp: null argument");
    const lz_mlp_config &c = *cfg;
    const bool fp32 = mlp_fits(c);
    LZ_REQUIRE(fp32 || mez_fits(c), LZ_EINVAL,
               "lz_model_create_mlp: latent_dim %d, obs_dim %d, action_space_size %d, head hidden sizes %d / %d / %d fit neither the "
               "fp32 MLP kernels (latent_dim in [8,128], obs_dim in [1,%d], latent_dim + action_space_size <= %d, head hidden sizes <= %d) "
               "nor the tensor-core MLP kernel (latent_dim a multiple of 32 in [32,%d], obs_dim in [1,%d], action_space_size in [1,%d], "
               "head hidden sizes in [1,%d])",
               c.latent_dim, c.obs_dim, c.action_space_size, c.reward_hidden, c.value_hidden, c.policy_hidden, kMlpWidth, kMlpWidth,
               kMlpWidth, kMezMaxL, kMezMaxObs, kMezMaxOut, kMezMaxHid);
    int K = 0;
    int rc = check_create("lz_model_create_mlp", c.support_min, c.support_max, c.support_step, kMlpK, &K);
    if (rc != LZ_OK) return rc;
    lz_model *m = new lz_model();
    m->family = fp32 ? ModelFamily::MlpFp32 : ModelFamily::MlpTc;
    m->A = c.action_space_size; m->K = K; m->support_min = c.support_min; m->support_step = c.support_step;
    m->lat_c = m->latent_floats = c.latent_dim; m->lat_h = m->lat_w = 1;
    m->obs_elems = c.obs_dim;
    if (fp32) m->mlp.cfg = c;
    else m->mez = MlpTcState{c.obs_dim, c.latent_dim, c.reward_hidden, c.value_hidden, c.policy_hidden, c.res_connection_in_dynamics};
    *out = m;
    return LZ_OK;
}
