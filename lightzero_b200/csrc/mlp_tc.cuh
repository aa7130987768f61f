// mlp_tc.cuh -- interface of the tensor-core (wgmma) network of EfficientZeroModelMLP and MuZeroModelMLP (mlp_tc.cu): vector
// observations, a latent of L = 32 .. 256 (a multiple of 32) features, the representation / dynamics / prediction MLPs as one
// layer program per launch.  EfficientZeroModelMLP's LSTM value-prefix head that follows the dynamics network is ez.cu's;
// MuZeroModelMLP's categorical reward head is part of the recurrent program.
#pragma once
#include "lz_common.cuh"

namespace lz {

constexpr int kMezMaxLayers = 66;     // 6 dense layers + 3 head hidden layers + the reward, value and policy FC2 cut into
                                      // pieces of <= L outputs (K, A <= 608: 19 pieces each at L = 32)
constexpr int kMezRows = 64;          // roots per CTA: one m64 wgmma tile
constexpr int kMezMaxL = 256, kMezMaxObs = 4096, kMezMaxOut = 608, kMezMaxHid = 32;

// layer flags of a program
enum : int {
    MF_RELU = 1, MF_GELU = 2,
    MF_ACT = 4,                       // + the one-hot action's weight column (times the BN scale), gathered from abias
    MF_RES = 8,                       // + the fp32 input latent (fc_dynamics_1's residual, after its ReLU)
    MF_LN = 16,                       // LayerNorm over the L outputs (representation network)
    MF_LATENT = 32,                   // write the output as the latent
    MF_FEAT = 64,                     // write the output as the LSTM input (fp32 [B][L])
    MF_VALUE = 128, MF_POLICY = 256,  // an FC2 piece of the value / policy head: logits columns col0 .. col0 + N
    MF_CAT_BEGIN = 512, MF_CAT_END = 1024,  // first / last piece of a categorical head's softmax expectation (with MF_VALUE
                                            // or MF_REWARD: the head whose scalar MF_CAT_END writes)
    MF_REWARD = 2048                  // an FC2 piece of MuZeroModelMLP's reward head (fc_reward_head.3)
};
// operand buffers: the two L-wide activation slots, the 32-wide head hidden buffer, the observation (streamed from global)
enum : int { MB_NONE = -1, MB_SLOT0 = 0, MB_SLOT1 = 1, MB_HID = 2, MB_OBS = 3 };

struct MezLayer {
    uint32_t woff;                    // byte offset of the layer's weight chunks
    int K, N;                         // padded: K a multiple of 32, N a multiple of 32 (<= L)
    int in, out, flags;
    int bn;                           // float offset of [scale N | shift N] in tab (power-of-two weight scale folded into scale)
    int col0;                         // FC2 pieces: first logits column
};

struct MezNet {
    const unsigned char *w;           // per layer, per 32-wide K chunk: [4 k-groups][N hi rows | N lo rows][8 halves] fp16
    const float *tab;                 // folded BN / bias tables
    const float *abias;               // [A][L]
    const float *ln_w, *ln_b;         // [L]
    int L, A, K, obs_dim, nlayers, nchunks;
    int nact;                         // width of the one-hot input of MF_ACT (A, or the chance outcomes of a StochasticMuZeroModelMLP
                                      // dynamics program, whose policy head has A outputs and whose afterstate program has K = C)
    MezLayer layer[kMezMaxLayers];
    float support_min, support_step;
};

struct MezIO {
    int B, npass;
    const float *obs;                 // [B][obs_dim] (initial_inference)
    const float *latent_base;         // input latents: base + ix[b] * slot_stride + b * L
    const int *ix;
    size_t slot_stride;
    const int *action;                // [B]
    float *latent_out, *latent_out2;  // [B][L] or nullptr
    float *feat;                      // [B][L] LSTM input (EfficientZeroModelMLP) or nullptr
    float *reward;                    // [B] or nullptr (MuZeroModelMLP's reward head)
    float *reward_logits;             // [B][K] or nullptr
    float *value;                     // [B] or nullptr
    float *policy_logits;             // [B][A] (row stride policy_stride) or nullptr
    float *value_logits;              // [B][K] or nullptr
    // optional row mask: with row_mask, row b is computed only when (row_mask[b] & 1) == row_mask_on; any other row is not
    // read and none of its outputs is written (the fused Stochastic MuZero search runs its two recurrent programs over the
    // same leaf batch, split by the parity of the leaf depth)
    const int *row_mask;
    int row_mask_on;
    int policy_stride;                // row stride of policy_logits (0: A)
};

// plan of a launch: roots per CTA, CTAs, roots of the last CTA, shared memory bytes, weight ring stages
struct MezPlan { int R, ctas, last, smem, stages; };

MezPlan mez_plan(const MezNet &net, int B);
int mez_launch(const MezNet &net, const MezIO &io, cudaStream_t s);
int mez_prepare_launch();

}  // namespace lz
