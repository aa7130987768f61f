// model.cu -- the lz_model_* C entry points: each switches on the model's family and calls the module that owns it (conv_model.cu,
// board_tc.cu, mlp.cu, mlp_tc.cu; ez.cu for EfficientZero's value-prefix head), and the state_dict reader / packing kit that
// every family's finalize uses.  lz_inverse_scalar_transform replaces lzero/policy/scaling_transform.py:82-92
// (InverseScalarTransform).
#include <math.h>
#include <string.h>

#include <algorithm>

#include "model.cuh"

namespace lz {

constexpr int kKpad = 608;                   // largest support size of the tensor-core heads (601 padded)

__global__ void k_inverse_scalar(const float *logits, float *out, int B, int K, float smin, float sstep)
{
    const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= B) return;
    float v = categorical_to_scalar(logits + (size_t)b * K, K, smin, sstep, lane);
    if (lane == 0) out[b] = v;
}

// ---- the state_dict reader and packing kit (model.cuh) -----------------------------------------------------------------------
const std::vector<float> *find_tensor(const lz_model *m, const std::string &name, size_t expect)
{
    auto it = m->tensors.find(name);
    if (it == m->tensors.end()) { set_error("lz_model_finalize: missing tensor '%s'", name.c_str()); return nullptr; }
    if (expect && it->second.size() != expect) {
        set_error("lz_model_finalize: tensor '%s' has %zu elements, expected %zu", name.c_str(), it->second.size(), expect);
        return nullptr;
    }
    return &it->second;
}

bool fold_bn(const lz_model *m, const std::string &prefix, int n, std::vector<float> &scale, std::vector<float> &shift)
{
    auto g = find_tensor(m, prefix + ".weight", n), bta = find_tensor(m, prefix + ".bias", n);
    auto mu = find_tensor(m, prefix + ".running_mean", n), var = find_tensor(m, prefix + ".running_var", n);
    if (!g || !bta || !mu || !var) return false;
    scale.resize(n); shift.resize(n);
    for (int i = 0; i < n; ++i) {
        float invstd = 1.0f / sqrtf((*var)[i] + 1e-5f);
        scale[i] = (*g)[i] * invstd;
        shift[i] = (*bta)[i] - (*mu)[i] * scale[i];
    }
    return true;
}

bool fold_bn_linear(const lz_model *m, const std::string &prefix, const std::vector<float> &b, std::vector<float> &scale,
                    std::vector<float> &shift)
{
    const size_t n = b.size();
    auto g = find_tensor(m, prefix + ".weight", n), be = find_tensor(m, prefix + ".bias", n);
    auto mu = find_tensor(m, prefix + ".running_mean", n), var = find_tensor(m, prefix + ".running_var", n);
    if (!g || !be || !mu || !var) return false;
    scale.resize(n); shift.resize(n);
    for (size_t j = 0; j < n; ++j) {
        const float s = (*g)[j] / sqrtf((*var)[j] + 1e-5f);
        scale[j] = s;
        shift[j] = (*be)[j] - (*mu)[j] * s + s * b[j];
    }
    return true;
}

size_t TablePacker::add(const std::vector<float> &v)
{
    while (host.size() % 4) host.push_back(0.0f);
    size_t off = host.size();
    host.insert(host.end(), v.begin(), v.end());
    return off;
}

float pow2_scale(float maxabs)
{
    int e = 0;
    if (maxabs > 0.0f) frexpf(maxabs, &e);     // maxabs = f * 2^e, f in [0.5, 1)
    return ldexpf(1.0f, 13 - e);
}

int check_create(const char *fn, float support_min, float support_max, float support_step, int kmax, int *K)
{
    *K = (int)ceil((support_max - support_min) / support_step);      // len(torch.arange(min, max, step))
    LZ_REQUIRE(*K >= 2 && *K <= kmax, LZ_EINVAL, "%s: support size %d not in [2, %d]", fn, *K, kmax);
    int ndev = 0;
    LZ_CUDA_CHECK(cudaGetDeviceCount(&ndev));
    LZ_REQUIRE(ndev > 0, LZ_ECUDA, "%s: no CUDA device (this library has no CPU fallback)", fn);
    return LZ_OK;
}

// ---- the internal launch API (model.cuh) -------------------------------------------------------------------------------------
int model_recurrent(lz_model *m, const RecIO &io, cudaStream_t s)
{
    LZ_REQUIRE((!io.after_program && !io.row_mask) || m->family == ModelFamily::MlpTc, LZ_EINVAL,
               "model_recurrent: afterstate programs and row masks are StochasticMuZeroModelMLP's");
    switch (m->family) {
        case ModelFamily::Conv: return conv_recurrent(m, io, s);
        case ModelFamily::Board: return board_recurrent(m, io, s);
        case ModelFamily::MlpFp32: return mlp_recurrent(m, io, s);
        case ModelFamily::MlpTc: return mez_recurrent(m, io, s);
    }
    return LZ_EINVAL;
}

int model_initial(lz_model *m, int B, const float *d_obs, const TailIO &io, cudaStream_t s)
{
    LZ_REQUIRE(!io.policy_stride || io.policy_stride == m->A || m->family == ModelFamily::MlpTc, LZ_EINVAL,
               "model_initial: policy logits at a row stride of %d other than the %d actions are the MlpTc programs'", io.policy_stride, m->A);
    switch (m->family) {
        case ModelFamily::Conv: return conv_initial(m, B, d_obs, io, s);
        case ModelFamily::Board: return board_initial(m, B, d_obs, io, s);
        case ModelFamily::MlpFp32: return mlp_initial(m, B, d_obs, io, s);
        case ModelFamily::MlpTc: return mez_initial(m, B, d_obs, io, s);
    }
    return LZ_EINVAL;
}

// the Board and MLP networks have no workspace; the value-prefix head has its LSTM scratch
int model_reserve(lz_model *m, int B, cudaStream_t s)
{
    int rc = m->family == ModelFamily::Conv ? conv_reserve(m, B, s) : LZ_OK;
    if (rc == LZ_OK && m->vp) rc = ez_reserve(m, B);
    return rc;
}

}  // namespace lz

using namespace lz;

extern "C" {

int lz_model_create(const lz_model_config *cfg, lz_model **out)
{
    LZ_REQUIRE(cfg && out, LZ_EINVAL, "lz_model_create: null argument");
    const bool board = cfg->downsample == 0;
    if (board) {
        LZ_REQUIRE(cfg->num_channels == 16 || cfg->num_channels == 32 || cfg->num_channels == 64, LZ_EINVAL,
                   "lz_model_create: the board network (downsample=False) takes num_channels 16, 32 or 64 (got %d)", cfg->num_channels);
        LZ_REQUIRE(cfg->obs_h >= 1 && cfg->obs_h <= kBoardMaxHW && cfg->obs_w >= 1 && cfg->obs_w <= kBoardMaxHW, LZ_EINVAL,
                   "lz_model_create: observation %dx%d not supported by the board network (downsample=False): boards up to %dx%d",
                   cfg->obs_h, cfg->obs_w, kBoardMaxHW, kBoardMaxHW);
        LZ_REQUIRE(cfg->obs_c >= 1 && cfg->obs_c <= 16, LZ_EINVAL, "lz_model_create: the board network takes 1 to 16 observation planes (got %d)", cfg->obs_c);
        LZ_REQUIRE(cfg->action_space_size >= 1 && cfg->action_space_size <= 64, LZ_EINVAL,
                   "lz_model_create: the board network takes 1 to 64 actions (got %d)", cfg->action_space_size);
        LZ_REQUIRE(!cfg->efficientzero, LZ_EINVAL, "lz_model_create: the board network (downsample=False) is MuZero only");
    } else {
        LZ_REQUIRE(cfg->num_channels == kC, LZ_EINVAL, "lz_model_create: num_channels must be %d (got %d)", kC, cfg->num_channels);
        LZ_REQUIRE(cfg->obs_h == cfg->obs_w && (cfg->obs_h == 64 || cfg->obs_h == 84 || cfg->obs_h == 96), LZ_EINVAL,
                   "lz_model_create: observation %dx%d not supported (64x64 -> 8x8 latent, 84x84 and 96x96 -> 6x6 latent)", cfg->obs_h, cfg->obs_w);
    }
    LZ_REQUIRE(cfg->num_res_blocks >= 1 && cfg->num_res_blocks <= kMaxResBlocks, LZ_EINVAL, "lz_model_create: num_res_blocks must be in [1,%d]", kMaxResBlocks);
    LZ_REQUIRE(cfg->reward_head_channels >= 1 && cfg->reward_head_channels <= 16 && cfg->value_head_channels >= 1 &&
                   cfg->value_head_channels <= 16 && cfg->policy_head_channels >= 1 && cfg->policy_head_channels <= 16,
               LZ_EINVAL, "lz_model_create: head channels must be in [1, 16] (got %d, %d, %d)", cfg->reward_head_channels,
               cfg->value_head_channels, cfg->policy_head_channels);
    LZ_REQUIRE(cfg->reward_hidden >= 1 && cfg->reward_hidden <= 32 && cfg->value_hidden >= 1 && cfg->value_hidden <= 32 &&
                   cfg->policy_hidden >= 1 && cfg->policy_hidden <= 32,
               LZ_EINVAL, "lz_model_create: head hidden sizes must be in [1, 32] (got %d, %d, %d)", cfg->reward_hidden,
               cfg->value_hidden, cfg->policy_hidden);
    LZ_REQUIRE(cfg->action_space_size >= 1 && cfg->action_space_size <= 1024, LZ_EINVAL, "lz_model_create: action_space_size out of range");
    int K = 0;
    int rc = check_create("lz_model_create", cfg->support_min, cfg->support_max, cfg->support_step, kKpad, &K);
    if (rc != LZ_OK) return rc;
    LZ_REQUIRE(!cfg->efficientzero || (cfg->lstm_hidden_size > 0 && cfg->lstm_hidden_size <= 512 && cfg->lstm_hidden_size % 16 == 0),
               LZ_EINVAL, "lz_model_create: lstm_hidden_size must be a multiple of 16 in [16, 512] (got %d)", cfg->lstm_hidden_size);
    lz_model *m = new lz_model();
    m->family = board ? ModelFamily::Board : ModelFamily::Conv;
    m->vp = cfg->efficientzero != 0;
    m->lstm_hidden = m->vp ? cfg->lstm_hidden_size : 0;
    m->A = cfg->action_space_size; m->K = K; m->support_min = cfg->support_min; m->support_step = cfg->support_step;
    // DownSample (common.py:334-366): 64 px -> 8x8 (no pooling2), 84 / 96 px -> 6x6; the board network keeps the board's H x W
    const int hw = cfg->obs_h == 64 ? 8 : kHW;
    m->lat_c = board ? cfg->num_channels : kC;
    m->lat_h = board ? cfg->obs_h : hw;
    m->lat_w = board ? cfg->obs_w : hw;
    m->latent_floats = m->lat_c * m->lat_h * m->lat_w;
    m->obs_elems = (size_t)cfg->obs_c * cfg->obs_h * cfg->obs_w;
    if (board) m->board.cfg = *cfg;
    else m->conv.cfg = *cfg;
    *out = m;
    return LZ_OK;
}

int lz_model_create_mlp_ez(const lz_mlp_ez_config *cfg, lz_model **out)
{
    LZ_REQUIRE(cfg && out, LZ_EINVAL, "lz_model_create_mlp_ez: null argument");
    const lz_mlp_ez_config &c = *cfg;
    LZ_REQUIRE(c.latent_dim >= 32 && c.latent_dim <= kMezMaxL && c.latent_dim % 32 == 0, LZ_EINVAL,
               "lz_model_create_mlp_ez: latent_dim must be a multiple of 32 in [32, %d] (got %d)", kMezMaxL, c.latent_dim);
    LZ_REQUIRE(c.lstm_hidden_size >= 16 && c.lstm_hidden_size <= 512 && c.lstm_hidden_size % 16 == 0, LZ_EINVAL,
               "lz_model_create_mlp_ez: lstm_hidden_size must be a multiple of 16 in [16, 512] (got %d)", c.lstm_hidden_size);
    LZ_REQUIRE(c.obs_dim >= 1 && c.obs_dim <= kMezMaxObs, LZ_EINVAL, "lz_model_create_mlp_ez: obs_dim must be in [1, %d] (got %d)",
               kMezMaxObs, c.obs_dim);
    LZ_REQUIRE(c.action_space_size >= 1 && c.action_space_size <= kMezMaxOut, LZ_EINVAL,
               "lz_model_create_mlp_ez: action_space_size must be in [1, %d] (got %d)", kMezMaxOut, c.action_space_size);
    LZ_REQUIRE(c.reward_hidden >= 1 && c.reward_hidden <= kMezMaxHid && c.value_hidden >= 1 && c.value_hidden <= kMezMaxHid &&
                   c.policy_hidden >= 1 && c.policy_hidden <= kMezMaxHid, LZ_EINVAL,
               "lz_model_create_mlp_ez: head hidden sizes must be in [1, %d] (got %d, %d, %d)", kMezMaxHid, c.reward_hidden,
               c.value_hidden, c.policy_hidden);
    int K = 0;
    int rc = check_create("lz_model_create_mlp_ez", c.support_min, c.support_max, c.support_step, kMezMaxOut, &K);
    if (rc != LZ_OK) return rc;
    lz_model *m = new lz_model();
    m->family = ModelFamily::MlpTc;
    m->vp = true;
    m->lstm_hidden = c.lstm_hidden_size;
    m->A = c.action_space_size; m->K = K; m->support_min = c.support_min; m->support_step = c.support_step;
    m->lat_c = m->latent_floats = c.latent_dim; m->lat_h = m->lat_w = 1;
    m->obs_elems = c.obs_dim;
    m->mez = MlpTcState{c.obs_dim, c.latent_dim, c.reward_hidden, c.value_hidden, c.policy_hidden, c.res_connection_in_dynamics};
    *out = m;
    return LZ_OK;
}

int lz_model_create_mlp_stochastic(const lz_mlp_stochastic_config *cfg, lz_model **out)
{
    LZ_REQUIRE(cfg && out, LZ_EINVAL, "lz_model_create_mlp_stochastic: null argument");
    const lz_mlp_stochastic_config &c = *cfg;
    LZ_REQUIRE(c.latent_dim >= 32 && c.latent_dim <= kMezMaxL && c.latent_dim % 32 == 0, LZ_EINVAL,
               "lz_model_create_mlp_stochastic: latent_dim must be a multiple of 32 in [32, %d] (got %d)", kMezMaxL, c.latent_dim);
    LZ_REQUIRE(c.obs_dim >= 1 && c.obs_dim <= kMezMaxObs, LZ_EINVAL,
               "lz_model_create_mlp_stochastic: obs_dim must be in [1, %d] (got %d)", kMezMaxObs, c.obs_dim);
    LZ_REQUIRE(c.action_space_size >= 1 && c.action_space_size <= kMezMaxOut, LZ_EINVAL,
               "lz_model_create_mlp_stochastic: action_space_size must be in [1, %d] (got %d)", kMezMaxOut, c.action_space_size);
    LZ_REQUIRE(c.chance_space_size >= 1 && c.chance_space_size <= kMezMaxOut, LZ_EINVAL,
               "lz_model_create_mlp_stochastic: chance_space_size must be in [1, %d] (got %d)", kMezMaxOut, c.chance_space_size);
    LZ_REQUIRE(c.reward_hidden >= 1 && c.reward_hidden <= kMezMaxHid && c.value_hidden >= 1 && c.value_hidden <= kMezMaxHid &&
                   c.policy_hidden >= 1 && c.policy_hidden <= kMezMaxHid, LZ_EINVAL,
               "lz_model_create_mlp_stochastic: head hidden sizes must be in [1, %d] (got %d, %d, %d)", kMezMaxHid, c.reward_hidden,
               c.value_hidden, c.policy_hidden);
    int K = 0;
    int rc = check_create("lz_model_create_mlp_stochastic", c.support_min, c.support_max, c.support_step, kMezMaxOut, &K);
    if (rc != LZ_OK) return rc;
    lz_model *m = new lz_model();
    m->family = ModelFamily::MlpTc;
    m->A = c.action_space_size; m->K = K; m->support_min = c.support_min; m->support_step = c.support_step;
    m->lat_c = m->latent_floats = c.latent_dim; m->lat_h = m->lat_w = 1;
    m->obs_elems = c.obs_dim;
    m->mez = MlpTcState{c.obs_dim, c.latent_dim, c.reward_hidden, c.value_hidden, c.policy_hidden, c.res_connection_in_dynamics,
                        c.chance_space_size};
    *out = m;
    return LZ_OK;
}

int lz_model_destroy(lz_model *m)
{
    if (!m) return LZ_OK;
    const ConvState &c = m->conv;
    cudaFree(c.d_weights); cudaFree(c.d_tc); cudaFree(c.d_tower); cudaFree(c.tws); cudaFree(c.tc_skip); cudaFree(c.pre_latent);
    cudaFree(m->board.d_board);
    cudaFree(m->mlp.d_weights);
    cudaFree(m->mez.d_mez);
    cudaFree(m->ez.d_tables); cudaFree(m->ez.d_wtc); cudaFree(m->ez.feat); cudaFree(m->ez.htmp);
    delete m;
    return LZ_OK;
}

int lz_model_set_tensor(lz_model *m, const char *name, const float *h_data, int64_t numel)
{
    LZ_REQUIRE(m && name && h_data && numel >= 0, LZ_EINVAL, "lz_model_set_tensor: bad argument");
    std::string n(name);
    if (n.find("num_batches_tracked") != std::string::npos) return 1;
    const bool stochastic = m->family == ModelFamily::MlpTc && m->mez.chance;     // StochasticMuZeroModelMLP's afterstate networks
    if (n.rfind("representation_network.", 0) != 0 && n.rfind("dynamics_network.", 0) != 0 &&
        n.rfind("prediction_network.", 0) != 0 &&
        !(stochastic && (n.rfind("afterstate_dynamics_network.", 0) == 0 || n.rfind("afterstate_prediction_network.", 0) == 0)))
        return 1;   // e.g. the optional SSL projection heads (muzero_model.py:198-208) and Stochastic MuZero's chance_encoder,
                    // unused at inference
    m->tensors[n].assign(h_data, h_data + numel);
    m->finalized = false;
    return LZ_OK;
}

int lz_model_finalize(lz_model *m)
{
    LZ_REQUIRE(m, LZ_EINVAL, "lz_model_finalize: null model");
    ++m->generation;          // every device table is re-allocated below: graphs captured against the old ones are stale
    int rc = LZ_EINVAL;
    switch (m->family) {
        case ModelFamily::Conv: rc = conv_finalize(m); break;
        case ModelFamily::Board: rc = board_finalize(m); break;
        case ModelFamily::MlpFp32: rc = mlp_finalize(m); break;
        case ModelFamily::MlpTc: rc = mez_finalize(m); break;
    }
    if (rc != LZ_OK) return rc;
    m->finalized = true;
    m->tensors.clear();
    return LZ_OK;
}

int lz_model_set_math(lz_model *m, int mode)
{
    LZ_REQUIRE(m && (mode == 1 || mode == 2), LZ_EINVAL,
               "lz_model_set_math: mode must be 1 (tc3: tensor-core fp16 hi/lo, fp32-accurate) or 2 (tc1: tensor-core single fp16 pass)");
    LZ_REQUIRE(m->family != ModelFamily::MlpFp32, LZ_EINVAL, "lz_model_set_math: the MLP model has no math mode");
    const int npass = mode == 1 ? 3 : 1;
    if (m->npass != npass) ++m->generation;      // captured search graphs bake the pass count in
    m->npass = npass;
    return LZ_OK;
}

/* debug: copies the 64 clock64 stamps of the last instrumented tensor-core launch (env LZ_TC_DEBUG=1) to the host */
int lz_debug_tc_stamps(unsigned long long *h_out)
{
    LZ_REQUIRE(h_out && tc_debug_buffer(), LZ_ESTATE, "lz_debug_tc_stamps: no instrumented launch yet");
    LZ_CUDA_CHECK(cudaMemcpy(h_out, tc_debug_buffer(), 64 * 8, cudaMemcpyDeviceToHost));
    return LZ_OK;
}

int lz_model_latent_hw(const lz_model *m) { return m ? (m->lat_h == m->lat_w ? m->lat_h : 0) : 0; }
int lz_model_latent_shape(const lz_model *m, int32_t *h_c, int32_t *h_h, int32_t *h_w)
{
    LZ_REQUIRE(m, LZ_EINVAL, "lz_model_latent_shape: null model");
    if (h_c) *h_c = m->lat_c;
    if (h_h) *h_h = m->lat_h;
    if (h_w) *h_w = m->lat_w;
    return LZ_OK;
}
int lz_model_support_size(const lz_model *m) { return m ? m->K : 0; }

int lz_model_initial_inference(lz_model *m, int B, const float *d_obs, float *d_latent, float *d_policy_logits,
                               float *d_value_logits, float *d_value, lz_stream s)
{
    LZ_REQUIRE(m && d_obs && B > 0, LZ_EINVAL, "lz_model_initial_inference: bad argument");
    LZ_REQUIRE(m->finalized, LZ_ESTATE, "lz_model_initial_inference: model not finalized");
    int rc = model_reserve(m, B, (cudaStream_t)s);
    if (rc != LZ_OK) return rc;
    TailIO io;
    memset(&io, 0, sizeof(io));
    io.latent = d_latent; io.policy_logits = d_policy_logits; io.value_logits = d_value_logits; io.value = d_value;
    return model_initial(m, B, d_obs, io, (cudaStream_t)s);
}

int lz_model_debug_net_stage(lz_model *m, int which, int B, const float *d_latent, const int32_t *d_action, int stage, void *d_out,
                             size_t out_bytes, int32_t *h_info, lz_stream s_)
{
    LZ_REQUIRE(m && which >= 0 && which <= 2 && B > 0 && d_latent && (which == 1 || d_action) && d_out && h_info && stage >= 0,
               LZ_EINVAL, "lz_model_debug_net_stage: bad argument");
    LZ_REQUIRE(m->finalized, LZ_ESTATE, "lz_model_debug_net_stage: model not finalized");
    LZ_REQUIRE(which != 2 || (m->family == ModelFamily::MlpTc && m->mez.chance), LZ_EINVAL,
               "lz_model_debug_net_stage: which 2 (the afterstate program) is StochasticMuZeroModelMLP's");
    const cudaStream_t s = (cudaStream_t)s_;
    switch (m->family) {
        case ModelFamily::Conv: return conv_debug_stage(m, which, B, d_latent, d_action, stage, d_out, out_bytes, h_info, s);
        case ModelFamily::Board: return board_debug_stage(m, which, B, d_latent, d_action, stage, d_out, out_bytes, h_info, s);
        case ModelFamily::MlpFp32: return mlp_debug_stage(m, which, B, d_latent, d_action, stage, d_out, out_bytes, h_info, s);
        case ModelFamily::MlpTc: return mez_debug_stage(m, which, B, d_latent, d_action, stage, d_out, out_bytes, h_info, s);
    }
    return LZ_EINVAL;
}

int lz_model_recurrent_inference(lz_model *m, int B, const float *d_latent, const int32_t *d_action,
                                 float *d_next_latent, float *d_reward_logits, float *d_value_logits,
                                 float *d_policy_logits, float *d_reward, float *d_value, lz_stream s)
{
    LZ_REQUIRE(m && d_latent && d_action && B > 0, LZ_EINVAL, "lz_model_recurrent_inference: bad argument");
    LZ_REQUIRE(m->finalized, LZ_ESTATE, "lz_model_recurrent_inference: model not finalized");
    if (m->family == ModelFamily::Conv) {
        int rc = conv_reserve_skip(m, B);
        if (rc != LZ_OK) return rc;
    }
    RecIO io;
    memset(&io, 0, sizeof(io));
    io.B = B; io.latent_base = d_latent; io.ix = nullptr; io.slot_stride = 0; io.action = d_action;
    io.next_latent = d_next_latent; io.reward = d_reward; io.value = d_value; io.policy_logits = d_policy_logits;
    io.reward_logits = d_reward_logits; io.value_logits = d_value_logits;
    return model_recurrent(m, io, (cudaStream_t)s);
}

int lz_model_recurrent_inference_stochastic(lz_model *m, int afterstate, int B, const float *d_state, const int32_t *d_option,
                                            const int32_t *d_row_mask, int row_mask_on, float *d_next_state,
                                            float *d_reward_logits, float *d_value_logits, float *d_policy_logits,
                                            float *d_reward, float *d_value, lz_stream s)
{
    LZ_REQUIRE(m && d_state && d_option && B > 0, LZ_EINVAL, "lz_model_recurrent_inference_stochastic: bad argument");
    LZ_REQUIRE(m->finalized && m->family == ModelFamily::MlpTc && m->mez.chance, LZ_ESTATE,
               "lz_model_recurrent_inference_stochastic: not a finalized StochasticMuZeroModelMLP");
    RecIO io;
    memset(&io, 0, sizeof(io));
    io.B = B; io.latent_base = d_state; io.action = d_option;
    io.next_latent = d_next_state; io.reward = d_reward; io.value = d_value; io.policy_logits = d_policy_logits;
    io.reward_logits = d_reward_logits; io.value_logits = d_value_logits;
    io.after_program = !afterstate;      // afterstate = 0: the state is a latent, the afterstate program makes an afterstate of it
    io.row_mask = d_row_mask; io.row_mask_on = row_mask_on & 1;
    return model_recurrent(m, io, (cudaStream_t)s);
}

int lz_model_recurrent_inference_ez(lz_model *m, int B, const float *d_latent, const float *d_hidden0, const float *d_hidden1,
                                    const int32_t *d_action, float *d_next_latent, float *d_next_hidden0, float *d_next_hidden1,
                                    float *d_value_prefix_logits, float *d_value_logits, float *d_policy_logits,
                                    float *d_value_prefix, float *d_value, lz_stream s)
{
    LZ_REQUIRE(m && d_latent && d_hidden0 && d_hidden1 && d_action && d_next_latent && B > 0, LZ_EINVAL, "lz_model_recurrent_inference_ez: bad argument");
    LZ_REQUIRE(m->finalized && m->vp, LZ_ESTATE, "lz_model_recurrent_inference_ez: not a finalized EfficientZero model");
    int rc = model_reserve(m, B, (cudaStream_t)s);
    if (rc != LZ_OK) return rc;
    RecIO io;
    memset(&io, 0, sizeof(io));
    io.B = B; io.latent_base = d_latent; io.action = d_action;
    io.next_latent = d_next_latent; io.reward = d_value_prefix; io.value = d_value; io.policy_logits = d_policy_logits;
    io.reward_logits = d_value_prefix_logits; io.value_logits = d_value_logits;
    io.h_base = d_hidden0; io.c_base = d_hidden1; io.h_out = d_next_hidden0; io.c_out = d_next_hidden1;
    return model_recurrent(m, io, (cudaStream_t)s);
}

int lz_model_lstm_hidden_size(const lz_model *m) { return m ? m->lstm_hidden : 0; }

int lz_inverse_scalar_transform(lz_model *m, int B, const float *d_logits, float *d_out, lz_stream s)
{
    LZ_REQUIRE(m && d_logits && d_out && B > 0, LZ_EINVAL, "lz_inverse_scalar_transform: bad argument");
    k_inverse_scalar<<<ceil_div(B, 4), 128, 0, (cudaStream_t)s>>>(d_logits, d_out, B, m->K, m->support_min, m->support_step);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

}  // extern "C"
