// model.cuh -- device-side weight tables of the MuZero conv model and the internal launch API.
#pragma once
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
    float *skip_scratch;              // [B][64 P] scratch of the tensor-core path (nullptr: the model's own, lz_model::tc_skip)
    // EfficientZero (reward == value prefix): LSTM state in / out, see ez.cuh
    const float *h_base, *c_base;     // base + ix[b]*hslot_stride + b*H
    size_t hslot_stride;
    float *h_out, *c_out;
    const int *is_reset;
};

struct TailIO {
    int B;
    const float *pre_latent;          // [B][C][P] output of the DownSample tower
    float *latent;                    // [B][C][P] (NCHW) or nullptr
    float *latent2;                   // second copy (latent pool slot 0) or nullptr
    float *value;                     // [B] scalar or nullptr
    float *policy_logits;             // [B][A] or nullptr
    float *value_logits;              // [B][K] or nullptr
};

}  // namespace lz

struct lz_model {
    int kind;                         // 0 = conv MuZeroModel / EfficientZeroModel (cfg.efficientzero), 1 = MuZeroModelMLP (mlp.cu),
                                      // 2 = board MuZeroModel (downsample=False, board_tc.cu), 3 = EfficientZeroModelMLP (mlp_tc.cu),
                                      // 4 = MuZeroModelMLP on the tensor cores (mlp_tc.cu): the configs mlp.cu does not take
                                      // (lz_model_create_mlp picks 1 or 4)
    unsigned char *d_board;           // kind 2: packed conv weights, BN / action-plane tables and fp32 head tables
    lz::BoardNet board_rec, board_init;   // kind 2: recurrent_inference / initial_inference programs
    lz_mlp_ez_config ecfg;            // kinds 3 and 4 (kind 4: the lz_mlp_config fields, lstm_hidden_size 0)
    unsigned char *d_mez;             // kinds 3, 4: packed fp16 hi / lo weights and fp32 tables of the dense layers
    lz::MezNet mez_rec, mez_init;     // kinds 3, 4: recurrent_inference (dense part) / initial_inference programs
    int lat_c, lat_h, lat_w;          // latent shape of one root
    lz::EzNet ez;                     // EfficientZero value-prefix head tables (device pointers into d_weights)
    float *ez_feat, *ez_htmp;         // [ws_B][hc*36], [ws_B][H] scratch between the conv kernel and the LSTM kernels
    int ez_B;
    unsigned char *d_ez_wtc;          // LSTM weights in the tensor-core layout (ez.cu)
    int latent_floats;                // floats per root latent (64*36, 64*64 or latent_dim)
    lz_mlp_config mcfg;               // kinds 1 and 4
    lz::MlpNet mlp;
    lz_model_config cfg;
    std::map<std::string, std::vector<float>> tensors;   // raw reference state_dict (host)
    bool finalized;
    float *d_weights;                 // one packed device allocation
    size_t n_weight_floats;
    lz::ConvG stem;                   // DownSample conv1 + norm1 (fp32 tables in d_weights)
    std::vector<float> stem_params;   // host copy of the Cin = 4 stem's weights + folded BN (kernel-parameter operands of k_stem4_tcl, model.cu)
    int stem_valid;
    int hw, P, K;
    int npass;                        // MMA passes per product of the tensor-core kernels: 3 = tc3 (fp16 hi/lo, fp32-accurate), 1 = tc1
    unsigned char *d_tc;              // packed fp16 hi/lo weights + tables of the tensor-core path
    lz::TcNet tc_rec, tc_tail;
    float *tc_skip;                   // [tc_skip_B][64 P] ResBlock skip scratch of k_net_tc for launches outside a search (model_reserve)
    int tc_skip_B;
    // tensor-core DownSample tower: packed weights / folded BN per layer, TCL activation workspace
    unsigned char *d_tower;           // weights + scale/shift tables
    lz::ConvTc tower_tc[2];           // downsample block: conv1 | conv3 (stride 2), conv2 (+ identity)
    lz::ResBlockTc tower_rb[3];       // resblocks1, resblocks2, resblocks3
    unsigned char *tws;               // TCL workspace (one allocation)
    size_t tws_bytes;
    lz::Tcl T0, T1, U0, U1, U2, V0, V1;
    // workspace for initial inference (grown on demand, outside graph capture)
    float *pre_latent;                // [ws_B][latent_floats] DownSample output, input of the latent-grid tail
    int ws_B;
    unsigned long long generation;    // bumped when device tables / workspaces that captured search graphs point into are re-allocated
                                      // or the pass count changes (finalize, set_math, model_reserve): lz_search re-captures
};

namespace lz {
int model_recurrent(lz_model *m, const RecIO &io, cudaStream_t s);
int model_initial(lz_model *m, int B, const float *d_obs, const TailIO &io, cudaStream_t s);
int model_initial_tower(lz_model *m, int B, const float *d_obs, float *pre_latent, cudaStream_t s, const uint8_t *d_obs_u8 = nullptr);   // exactly one of d_obs / d_obs_u8
int model_initial_tail(lz_model *m, int B, const float *pre_latent, const TailIO &io, cudaStream_t s);
int model_reserve(lz_model *m, int B);   // sizes the initial-inference workspace (synchronous)
int mlp_recurrent(lz_model *m, const RecIO &io, cudaStream_t s);
int mlp_initial(lz_model *m, int B, const float *d_obs, const TailIO &io, cudaStream_t s);
int mlp_finalize(lz_model *m);
int mlp_debug_stage(lz_model *m, int which, int B, const float *d_in, const int32_t *d_action, int stage, void *d_out,
                    size_t out_bytes, int32_t *h_info, cudaStream_t s);
bool model_is_ez(const lz_model *m);     // EfficientZero (value-prefix LSTM head): conv EfficientZeroModel or EfficientZeroModelMLP
}  // namespace lz
