// model.cuh -- the model families' state, the common lz_model fields, the internal launch API and the state_dict reader /
// weight-packing kit that every family's finalize uses (model.cu).
#pragma once
#include <cuda_fp16.h>
#include <math.h>

#include <map>
#include <string>
#include <vector>

#include "lz_common.cuh"
#include "net6.cuh"
#include "net_tc.cuh"
#include "conv_tc.cuh"
#include "ez.cuh"
#include "board_tc.cuh"
#include "mlp_tc.cuh"

namespace lz {

constexpr int kMaxResBlocks = 4;

struct ConvG {                        // DownSample stem (conv1 + norm1 + ReLU, 3x3 stride 2) of any input channel count
    const float *w;                   // [cin][9][cout]
    const float *scale, *shift;       // [cout]
    int cin, cout, hin, win, hout, wout;
};

struct Dense {                        // y = act(scale * (W x) + shift); wt is input-major [in][out]
    const float *wt, *scale, *shift;
    int in, out, act, nact;           // act: 0 none, 1 ReLU, 2 GELU(tanh); nact: trailing one-hot action inputs
};

struct MlpNet {                       // MuZeroModelMLP (muzero_model_mlp.py)
    Dense e0, e1;                     // representation: Linear+BN+GELU, Linear (+ LayerNorm)
    Dense d1a, d1b, d2a, d2b;         // dynamics: fc_dynamics_1 (or fc_dynamics), fc_dynamics_2
    Dense r0, r1, pc0, pc1, v0, v1, p0, p1;
    const float *ln_w, *ln_b;
    int latent, obs_dim, A, res;
    float support_min, support_step;
};

struct RecIO {
    int B;
    const float *latent_base;         // latent source: base + ix[b]*slot_stride + b*C*P  (ix == nullptr: slot 0)
    const int *ix;
    size_t slot_stride;
    const int *action;                // [B]
    float *next_latent;               // [B][C][P] destination (pool slot or API buffer) or nullptr
    float *reward, *value;            // [B] scalars or nullptr
    float *policy_logits;             // [B][A] or nullptr
    float *reward_logits, *value_logits;   // [B][K] or nullptr
    float *skip_scratch;              // [B][64 P] scratch of the tensor-core path (nullptr: the model's own, ConvState::tc_skip)
    // EfficientZero (reward == value prefix): LSTM state in / out, see ez.cuh
    const float *h_base, *c_base;     // base + ix[b]*hslot_stride + b*H
    size_t hslot_stride;
    float *h_out, *c_out;
    const int *is_reset;
    // Stochastic MuZero models (lz_model::chance != 0): after_program != 0 runs the afterstate program (afterstate dynamics +
    // afterstate prediction, C chance logits into policy_logits) instead of the dynamics program; row_mask / row_mask_on as MezIO's
    int after_program;
    const int *row_mask;
    int row_mask_on;
    int policy_stride;                // row stride of policy_logits (0: the program's policy outputs)
};

struct TailIO {
    int B;
    const float *pre_latent;          // [B][C][P] output of the DownSample tower
    float *latent;                    // [B][C][P] (NCHW) or nullptr
    float *latent2;                   // second copy (latent pool slot 0) or nullptr
    float *value;                     // [B] scalar or nullptr
    float *policy_logits;             // [B][A] (row stride policy_stride) or nullptr
    float *value_logits;              // [B][K] or nullptr
    int policy_stride;                // row stride of policy_logits (0: A); only the Stochastic MuZero models take a stride other than A
};

// The model families: each has its own state below and its own module; model.cu switches on the family at every lz_model_*
// entry point and calls the owning module's function.
enum class ModelFamily {
    Conv,                             // MuZeroModel / EfficientZeroModel with the DownSample tower (conv_model.cu)
    Board,                            // MuZeroModel with downsample=False, the board games (board_tc.cu)
    MlpFp32,                          // MuZeroModelMLP on the fp32 kernels (mlp.cu)
    MlpTc,                            // EfficientZeroModelMLP, and the MuZeroModelMLP configs mlp.cu does not take (mlp_tc.cu)
};

struct ConvState {
    lz_model_config cfg;
    float *d_weights;                 // fp32 tables of the stem and of the heads' FC parts
    ConvG stem;                       // DownSample conv1 + norm1 (fp32 tables in d_weights)
    std::vector<float> stem_params;   // host copy of the Cin = 4 stem's weights + folded BN (kernel-parameter operands of k_stem4_tcl)
    int stem_valid;
    unsigned char *d_tc;              // packed fp16 hi/lo weights + tables of the latent-grid network (net_tc.cu)
    TcNet tc_rec, tc_tail;
    float *tc_skip;                   // [tc_skip_B][64 P] ResBlock skip scratch of k_net_tc for launches outside a search
    int tc_skip_B;
    // tensor-core DownSample tower: packed weights / folded BN per layer, TCL activation workspace
    unsigned char *d_tower;           // weights + scale/shift tables
    ConvTc tower_tc[2];               // downsample block: conv1 | conv3 (stride 2), conv2 (+ identity)
    ResBlockTc tower_rb[3];           // resblocks1, resblocks2, resblocks3
    unsigned char *tws;               // TCL workspace (one allocation)
    Tcl T0, T1, U0, U1, U2, V0, V1;
    // workspace for initial inference (grown on demand, outside graph capture)
    float *pre_latent;                // [ws_B][latent_floats] DownSample output, input of the latent-grid tail
    int ws_B;
};

struct BoardState {
    lz_model_config cfg;
    unsigned char *d_board;           // packed conv weights, BN / action-plane tables and fp32 head tables
    BoardNet rec, init;               // recurrent_inference / initial_inference programs
    BoardNet after;                   // StochasticMuZeroModel's afterstate program (rec is its dynamics program on afterstates)
};

struct MlpFp32State {
    lz_mlp_config cfg;
    float *d_weights;
    MlpNet net;
};

struct MlpTcState {
    int obs_dim, latent, reward_hidden, value_hidden, policy_hidden, res;   // res: res_connection_in_dynamics
    unsigned char *d_mez;             // packed fp16 hi / lo weights and fp32 tables of the dense layers
    MezNet rec, init;                 // recurrent_inference (dense part) / initial_inference programs
    MezNet after;                     // StochasticMuZeroModelMLP's afterstate program (rec is its dynamics program on afterstates)
};

// EfficientZero's value-prefix head (ez.cu) on the LSTM input features that the Conv or the MlpTc network writes into `feat`
struct EzHead {
    EzNet net;
    float *d_tables;                  // fp32 tables of the LSTM and of fc_reward_head
    unsigned char *d_wtc;             // LSTM weights in the tensor-core layout
    float *feat, *htmp;               // [B][nin], [B][H] scratch between the network kernel and the LSTM kernels
    int B;
};

}  // namespace lz

struct lz_model {
    lz::ModelFamily family;
    bool vp;                          // EfficientZero: the reward is a value prefix from the LSTM head in `ez`
    int lstm_hidden;                  // its LSTM width (0 without the head)
    int A, K;                         // actions, support size
    int chance;                       // Stochastic MuZero models (StochasticMuZeroModelMLP, StochasticMuZeroModel): chance_space_size;
                                      // 0 for every other model
    float support_min, support_step;
    int lat_c, lat_h, lat_w;          // latent shape of one root ([latent_dim][1][1] for the MLP families)
    int latent_floats;                // lat_c * lat_h * lat_w
    size_t obs_elems;                 // observation elements of one root
    int npass = 3;                    // MMA passes per product of the tensor-core kernels: 3 = tc3 (fp16 hi/lo, fp32-accurate), 1 = tc1
    unsigned long long generation;    // bumped when device tables / workspaces that captured search graphs point into are re-allocated
                                      // or the pass count changes (finalize, set_math, model_reserve): lz_search re-captures
    bool finalized;
    std::map<std::string, std::vector<float>> tensors;   // raw reference state_dict (host)
    lz::ConvState conv;
    lz::BoardState board;
    lz::MlpFp32State mlp;
    lz::MlpTcState mez;
    lz::EzHead ez;
};

namespace lz {
// ---- the state_dict reader and weight-packing kit (model.cu) ----
// the tensor `name` of the state_dict given to lz_model_set_tensor, with `expect` elements (0: any); nullptr and the error set
// when it is missing or has another size
const std::vector<float> *find_tensor(const lz_model *m, const std::string &name, size_t expect);

// Eval-mode BatchNorm (eps = 1e-5) as y = x * scale + shift.  The two folds round differently and each family's tables were
// fixed with its own: fold_bn computes g * (1 / sqrt(v + eps)) and leaves any preceding bias to the caller (the conv families);
// fold_bn_linear computes g / sqrt(v + eps) and folds the Linear bias b into the shift as be - mu s + s b (the MLP families).
bool fold_bn(const lz_model *m, const std::string &prefix, int n, std::vector<float> &scale, std::vector<float> &shift);
bool fold_bn_linear(const lz_model *m, const std::string &prefix, const std::vector<float> &b, std::vector<float> &scale,
                    std::vector<float> &shift);

// fp32 tables appended at 16-byte aligned float offsets
struct TablePacker {
    std::vector<float> host;
    size_t add(const std::vector<float> &v);
};

// the power-of-two scale that puts a weight matrix's largest |w| (`maxabs`) in [4096, 8192): the lo parts of the fp16 hi / lo
// split stay in fp16's normal range.  The scale is exact; callers fold its inverse into the layer's fp32 scale.
float pow2_scale(float maxabs);

inline void split_hi_lo(float v, __half &hi, __half &lo)
{
    hi = __float2half_rn(v);
    lo = __float2half_rn(v - __half2float(hi));
}

// replaces the device table *dst with a copy of `bytes` host bytes, complete on return (setup_upload).  Freeing a table that
// already exists (a weight reload) waits for all work on the device, so no search in flight still reads it.
template <typename T>
int upload(T **dst, const void *src, size_t bytes)
{
    dev_free(*dst);
    *dst = nullptr;
    int rc = dev_alloc(reinterpret_cast<unsigned char **>(dst), bytes);
    if (rc != LZ_OK) return rc;
    return setup_upload(*dst, src, bytes);
}

// the create functions' common checks: the support size K = len(torch.arange(min, max, step)) in [2, kmax], and a CUDA device
int check_create(const char *fn, float support_min, float support_max, float support_step, int kmax, int *K);

// ---- the families behind the entry points ----
int model_recurrent(lz_model *m, const RecIO &io, cudaStream_t s);
int model_initial(lz_model *m, int B, const float *d_obs, const TailIO &io, cudaStream_t s);
// sizes the scratch of launches outside a search, outside capture; a growth frees the old scratch (waits for the whole device)
// and zeroes what must start zeroed on `s`
int model_reserve(lz_model *m, int B, cudaStream_t s);
// lz_model_debug_net_stage of each family: `which` 0 is the recurrent program on the latents d_in and actions d_action, 1 the
// initial_inference program on the observations d_in

// Conv (conv_model.cu)
int conv_finalize(lz_model *m);
int conv_reserve(lz_model *m, int B, cudaStream_t s);
int conv_reserve_skip(lz_model *m, int B);   // the skip scratch alone (lz_model_recurrent_inference)
int conv_recurrent(lz_model *m, const RecIO &io, cudaStream_t s);
int conv_initial(lz_model *m, int B, const float *d_obs, const TailIO &io, cudaStream_t s);
int conv_initial_tower(lz_model *m, int B, const float *d_obs, float *pre_latent, cudaStream_t s, const uint8_t *d_obs_u8 = nullptr);   // exactly one of d_obs / d_obs_u8
int conv_initial_tail(lz_model *m, int B, const float *pre_latent, const TailIO &io, cudaStream_t s);
int conv_debug_stage(lz_model *m, int which, int B, const float *d_in, const int32_t *d_action, int stage, void *d_out, size_t out_bytes,
                     int32_t *h_info, cudaStream_t s);
// Board (board_tc.cu)
int board_finalize(lz_model *m);
int board_recurrent(lz_model *m, const RecIO &io, cudaStream_t s);
int board_initial(lz_model *m, int B, const float *d_obs, const TailIO &io, cudaStream_t s);
int board_debug_stage(lz_model *m, int which, int B, const float *d_in, const int32_t *d_action, int stage, void *d_out, size_t out_bytes,
                      int32_t *h_info, cudaStream_t s);
// MlpFp32 (mlp.cu)
int mlp_finalize(lz_model *m);
int mlp_recurrent(lz_model *m, const RecIO &io, cudaStream_t s);
int mlp_initial(lz_model *m, int B, const float *d_obs, const TailIO &io, cudaStream_t s);
int mlp_debug_stage(lz_model *m, int which, int B, const float *d_in, const int32_t *d_action, int stage, void *d_out, size_t out_bytes,
                    int32_t *h_info, cudaStream_t s);
// MlpTc (mlp_tc.cu)
int mez_finalize(lz_model *m);
int mez_recurrent(lz_model *m, const RecIO &io, cudaStream_t s);
int mez_initial(lz_model *m, int B, const float *d_obs, const TailIO &io, cudaStream_t s);
int mez_debug_stage(lz_model *m, int which, int B, const float *d_in, const int32_t *d_action, int stage, void *d_out, size_t out_bytes,
                    int32_t *h_info, cudaStream_t s);
// the value-prefix head (ez.cu)
int ez_finalize(lz_model *m, int nin, int hid, bool vp_norm);
int ez_reserve(lz_model *m, int B);
int ez_tail(lz_model *m, const RecIO &io, cudaStream_t s);
}  // namespace lz
