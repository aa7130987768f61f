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

// prediction network + outputs for the latents in `lat` (shared, [RB][kMlpWidth])
__device__ __forceinline__ void mlp_predict(const MlpNet &net, const float *lat, float *b0, float *b1, float *logits,
                                            int root0, int B, float *o_value, float *o_policy, float *o_value_logits)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    dense(net.pc0, lat, b0, kMlpWidth, kMlpWidth, nullptr);
    dense(net.pc1, b0, b1, kMlpWidth, kMlpWidth, nullptr);
    dense(net.v0, b1, b0, kMlpWidth, kMlpWidth, nullptr);
    dense(net.v1, b0, logits, kMlpWidth, kMlpK, nullptr);
    if (root0 + warp < B) {
        const float v = categorical_to_scalar(logits + warp * kMlpK, net.v1.out, net.support_min, net.support_step, lane);
        if (lane == 0 && o_value) o_value[root0 + warp] = v;
        if (o_value_logits)
            for (int k = lane; k < net.v1.out; k += 32) o_value_logits[(size_t)(root0 + warp) * net.v1.out + k] = logits[warp * kMlpK + k];
    }
    __syncthreads();
    dense(net.p0, b1, b0, kMlpWidth, kMlpWidth, nullptr);
    dense(net.p1, b0, logits, kMlpWidth, kMlpK, nullptr);
    if (root0 + warp < B && o_policy)
        for (int a = lane; a < net.A; a += 32) o_policy[(size_t)(root0 + warp) * net.A + a] = logits[warp * kMlpK + a];
    __syncthreads();
}

__global__ void __launch_bounds__(kMlpThreads) k_mlp_recurrent(MlpNet net, RecIO io)
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
        dense(net.d1b, xb, xc, kMlpWidth, kMlpWidth, nullptr);
        for (int i = threadIdx.x; i < kMlpRoots * Ld; i += kMlpThreads) {
            const int r = i / Ld, c = i - r * Ld;
            xc[r * kMlpWidth + c] += xa[r * kMlpWidth + c];
        }
        __syncthreads();
        dense(net.d2a, xc, xb, kMlpWidth, kMlpWidth, nullptr);
        dense(net.d2b, xb, xa, kMlpWidth, kMlpWidth, nullptr);
        nxt = xc; enc = xa;
    } else {                                         // :436-438
        dense(net.d1a, xa, xb, kMlpWidth, kMlpWidth, act_row);
        dense(net.d1b, xb, xc, kMlpWidth, kMlpWidth, nullptr);
        nxt = xc; enc = xc;
    }
    if (io.next_latent)
        for (int i = threadIdx.x; i < kMlpRoots * Ld; i += kMlpThreads) {
            const int r = i / Ld, c = i - r * Ld, b = root0 + r;
            if (b < io.B) io.next_latent[(size_t)b * Ld + c] = nxt[r * kMlpWidth + c];
        }
    // reward head (:440)
    dense(net.r0, enc, xb, kMlpWidth, kMlpWidth, nullptr);
    dense(net.r1, xb, logits, kMlpWidth, kMlpK, nullptr);
    if (root0 + warp < io.B) {
        const float rv = categorical_to_scalar(logits + warp * kMlpK, net.r1.out, net.support_min, net.support_step, lane);
        if (lane == 0 && io.reward) io.reward[root0 + warp] = rv;
        if (io.reward_logits)
            for (int k = lane; k < net.r1.out; k += 32) io.reward_logits[(size_t)(root0 + warp) * net.r1.out + k] = logits[warp * kMlpK + k];
    }
    __syncthreads();
    // prediction on the next latent: nxt lives in xc; xa / xb are scratch (enc no longer needed)
    mlp_predict(net, nxt, xa, xb, logits, root0, io.B, io.value, io.policy_logits, io.value_logits);
}

__global__ void __launch_bounds__(kMlpThreads) k_mlp_initial(MlpNet net, const float *obs, TailIO io)
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
    dense(net.e1, xb, xc, kMlpWidth, kMlpWidth, nullptr);          // Linear
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
    for (int i = threadIdx.x; i < kMlpRoots * Ld; i += kMlpThreads) {
        const int r = i / Ld, c = i - r * Ld, b = root0 + r;
        if (b < io.B) {
            if (io.latent) io.latent[(size_t)b * Ld + c] = xc[r * kMlpWidth + c];
            if (io.latent2) io.latent2[(size_t)b * Ld + c] = xc[r * kMlpWidth + c];
        }
    }
    mlp_predict(net, xc, xa, xb, logits, root0, io.B, io.value, io.policy_logits, io.value_logits);
}

int mlp_recurrent(lz_model *m, const RecIO &io, cudaStream_t s)
{
    k_mlp_recurrent<<<ceil_div(io.B, kMlpRoots), kMlpThreads, 0, s>>>(m->mlp, io);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

int mlp_initial(lz_model *m, int B, const float *d_obs, const TailIO &io_in, cudaStream_t s)
{
    TailIO io = io_in;
    io.B = B;
    k_mlp_initial<<<ceil_div(B, kMlpRoots), kMlpThreads, 0, s>>>(m->mlp, d_obs, io);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

// ---- weights ----------------------------------------------------------------------------------
static const std::vector<float> *mfind(lz_model *m, const std::string &name, size_t expect)
{
    auto it = m->tensors.find(name);
    if (it == m->tensors.end()) { set_error("lz_model_finalize: missing tensor '%s'", name.c_str()); return nullptr; }
    if (expect && it->second.size() != expect) {
        set_error("lz_model_finalize: tensor '%s' has %zu elements, expected %zu", name.c_str(), it->second.size(), expect);
        return nullptr;
    }
    return &it->second;
}

struct DenseOff { size_t wt, scale, shift; int in, out, act, nact; };

// Linear `lin` (weight [out][in], bias [out]) optionally followed by eval BatchNorm1d `bn`
static bool pack_dense(lz_model *m, std::vector<float> &host, const std::string &lin, const std::string &bn, int in, int out,
                       int act, int nact, DenseOff &o)
{
    auto W = mfind(m, lin + ".weight", (size_t)out * in), b = mfind(m, lin + ".bias", out);
    if (!W || !b) return false;
    std::vector<float> scale(out, 1.0f), shift(*b);
    if (!bn.empty()) {
        auto g = mfind(m, bn + ".weight", out), be = mfind(m, bn + ".bias", out);
        auto mu = mfind(m, bn + ".running_mean", out), var = mfind(m, bn + ".running_var", out);
        if (!g || !be || !mu || !var) return false;
        for (int j = 0; j < out; ++j) {
            const float s = (*g)[j] / sqrtf((*var)[j] + 1e-5f);
            scale[j] = s;
            shift[j] = (*be)[j] - (*mu)[j] * s + s * (*b)[j];
        }
    }
    auto add = [&](const std::vector<float> &v) {
        while (host.size() % 4) host.push_back(0.0f);
        size_t off = host.size();
        host.insert(host.end(), v.begin(), v.end());
        return off;
    };
    std::vector<float> wt((size_t)in * out);
    for (int j = 0; j < out; ++j)
        for (int i = 0; i < in; ++i) wt[(size_t)i * out + j] = (*W)[(size_t)j * in + i];
    o.wt = add(wt); o.scale = add(scale); o.shift = add(shift);
    o.in = in; o.out = out; o.act = act; o.nact = nact;
    return true;
}

int mlp_finalize(lz_model *m)
{
    const lz_mlp_config &c = m->mcfg;
    const int L = c.latent_dim, A = c.action_space_size, K = m->K;
    std::vector<float> host;
    DenseOff e0, e1, d1a, d1b, d2a, d2b, r0, r1, pc0, pc1, v0, v1, p0, p1;
    memset(&d2a, 0, sizeof(d2a)); memset(&d2b, 0, sizeof(d2b));
    const std::string R = "representation_network.", D = "dynamics_network.", Q = "prediction_network.";
    bool ok = pack_dense(m, host, R + "fc_representation.0", R + "fc_representation.1", c.obs_dim, L, 2, 0, e0) &&
              pack_dense(m, host, R + "fc_representation.3", "", L, L, 0, 0, e1);
    if (ok && c.res_connection_in_dynamics)
        ok = pack_dense(m, host, D + "fc_dynamics_1.0", D + "fc_dynamics_1.1", L + A, L, 1, A, d1a) &&
             pack_dense(m, host, D + "fc_dynamics_1.3", D + "fc_dynamics_1.4", L, L, 1, 0, d1b) &&
             pack_dense(m, host, D + "fc_dynamics_2.0", D + "fc_dynamics_2.1", L, L, 1, 0, d2a) &&
             pack_dense(m, host, D + "fc_dynamics_2.3", D + "fc_dynamics_2.4", L, L, 1, 0, d2b);
    else if (ok)
        ok = pack_dense(m, host, D + "fc_dynamics.0", D + "fc_dynamics.1", L + A, L, 1, A, d1a) &&
             pack_dense(m, host, D + "fc_dynamics.3", D + "fc_dynamics.4", L, L, 1, 0, d1b);
    ok = ok && pack_dense(m, host, D + "fc_reward_head.0", D + "fc_reward_head.1", L, c.reward_hidden, 1, 0, r0) &&
         pack_dense(m, host, D + "fc_reward_head.3", "", c.reward_hidden, K, 0, 0, r1) &&
         pack_dense(m, host, Q + "fc_prediction_common.0", Q + "fc_prediction_common.1", L, L, 1, 0, pc0) &&
         pack_dense(m, host, Q + "fc_prediction_common.3", Q + "fc_prediction_common.4", L, L, 1, 0, pc1) &&
         pack_dense(m, host, Q + "fc_value_head.0", Q + "fc_value_head.1", L, c.value_hidden, 1, 0, v0) &&
         pack_dense(m, host, Q + "fc_value_head.3", "", c.value_hidden, K, 0, 0, v1) &&
         pack_dense(m, host, Q + "fc_policy_head.0", Q + "fc_policy_head.1", L, c.policy_hidden, 1, 0, p0) &&
         pack_dense(m, host, Q + "fc_policy_head.3", "", c.policy_hidden, A, 0, 0, p1);
    if (!ok) return LZ_EINVAL;
    auto lw = mfind(m, R + "norm.weight", L), lb = mfind(m, R + "norm.bias", L);
    if (!lw || !lb) return LZ_EINVAL;
    while (host.size() % 4) host.push_back(0.0f);
    const size_t o_lw = host.size();
    host.insert(host.end(), lw->begin(), lw->end());
    const size_t o_lb = host.size();
    host.insert(host.end(), lb->begin(), lb->end());
    if (m->d_weights) cudaFree(m->d_weights);
    m->d_weights = nullptr;
    int rc = dev_alloc(&m->d_weights, host.size());
    if (rc != LZ_OK) return rc;
    LZ_CUDA_CHECK(cudaMemcpy(m->d_weights, host.data(), host.size() * sizeof(float), cudaMemcpyHostToDevice));
    const float *base = m->d_weights;
    auto mk = [&](const DenseOff &o) { Dense d; d.wt = base + o.wt; d.scale = base + o.scale; d.shift = base + o.shift; d.in = o.in; d.out = o.out; d.act = o.act; d.nact = o.nact; return d; };
    MlpNet &n = m->mlp;
    memset(&n, 0, sizeof(n));
    n.e0 = mk(e0); n.e1 = mk(e1); n.d1a = mk(d1a); n.d1b = mk(d1b);
    if (c.res_connection_in_dynamics) { n.d2a = mk(d2a); n.d2b = mk(d2b); }
    n.r0 = mk(r0); n.r1 = mk(r1); n.pc0 = mk(pc0); n.pc1 = mk(pc1); n.v0 = mk(v0); n.v1 = mk(v1); n.p0 = mk(p0); n.p1 = mk(p1);
    n.ln_w = base + o_lw; n.ln_b = base + o_lb;
    n.latent = L; n.obs_dim = c.obs_dim; n.A = A; n.res = c.res_connection_in_dynamics;
    n.support_min = c.support_min; n.support_step = c.support_step;
    m->finalized = true;
    m->tensors.clear();
    return LZ_OK;
}

}  // namespace lz

using namespace lz;

extern "C" int lz_model_create_mlp(const lz_mlp_config *cfg, lz_model **out)
{
    LZ_REQUIRE(cfg && out, LZ_EINVAL, "lz_model_create_mlp: null argument");
    LZ_REQUIRE(cfg->latent_dim >= 8 && cfg->latent_dim <= 128 && cfg->obs_dim >= 1 && cfg->obs_dim <= kMlpWidth, LZ_EINVAL,
               "lz_model_create_mlp: latent_dim must be in [8,128], obs_dim in [1,%d]", kMlpWidth);
    LZ_REQUIRE(cfg->action_space_size >= 1 && cfg->latent_dim + cfg->action_space_size <= kMlpWidth, LZ_EINVAL,
               "lz_model_create_mlp: latent_dim + action_space_size must be <= %d", kMlpWidth);
    LZ_REQUIRE(cfg->reward_hidden <= kMlpWidth && cfg->value_hidden <= kMlpWidth && cfg->policy_hidden <= kMlpWidth, LZ_EINVAL,
               "lz_model_create_mlp: head hidden sizes must be <= %d", kMlpWidth);
    const int K = (int)ceil((cfg->support_max - cfg->support_min) / cfg->support_step);
    LZ_REQUIRE(K >= 2 && K <= kMlpK, LZ_EINVAL, "lz_model_create_mlp: support size %d not in [2, %d]", K, kMlpK);
    int ndev = 0;
    LZ_CUDA_CHECK(cudaGetDeviceCount(&ndev));
    LZ_REQUIRE(ndev > 0, LZ_ECUDA, "lz_model_create_mlp: no CUDA device (this library has no CPU fallback)");
    lz_model *m = new lz_model();
    memset(&m->cfg, 0, sizeof(m->cfg));
    m->cfg.action_space_size = cfg->action_space_size;
    m->cfg.support_min = cfg->support_min; m->cfg.support_max = cfg->support_max; m->cfg.support_step = cfg->support_step;
    m->mcfg = *cfg;
    m->kind = 1;
    m->latent_floats = cfg->latent_dim;
    m->finalized = false;
    m->d_weights = nullptr; m->d_tc = nullptr; m->d_tower = nullptr; m->tws = nullptr; m->tws_bytes = 0;
    m->hw = 1; m->P = 1; m->K = K;
    m->pre_latent = nullptr; m->ws_B = 1 << 30;
    *out = m;
    return LZ_OK;
}
