// board_tc.cuh -- interface of the board-grid tensor-core network (board_tc.cu): MuZeroModel with downsample=False, the network of
// the board-game configs (tictactoe, connect4, gomoku), and StochasticMuZeroModel with downsample=False (2048): every layer at
// the board's own H x W, C in {16, 32, 64} channels.
#pragma once
#include "lz_common.cuh"

namespace lz {

constexpr int kBoardMaxLayers = 1 + 4 * 4;     // representation / dynamics conv + two ResBlock stacks of up to 4 blocks
constexpr int kBoardMaxHW = 8;

// layer flags of a board program
enum : int { BF_OBS = 1, BF_RES = 2, BF_STORE_RES = 4, BF_ACT_BIAS = 8, BF_WRITE_LATENT = 16, BF_HOOK_REWARD = 32, BF_HOOK_VALPOL = 64 };

struct BoardHead {                 // conv1x1 -> BN -> ReLU -> Linear(hc*P -> hid) -> BN1d -> ReLU -> Linear(hid -> K), fp32
    const float *w1, *s1, *t1;     // [hc][C], [hc], [hc] (conv bias folded into t1)
    const float *fc1, *s2, *t2;    // [hid][hc*P], [hid], [hid] (Linear bias folded into t2)
    const float *fc2, *b2;         // [K][hid], [K]
    int hc, hid, K;
};

struct BoardNet {
    const unsigned char *convw;    // per conv: [9 taps][cin / 8 k-groups][C hi rows | C lo rows][8] fp16, K-major core matrices
    const float *bn;               // per conv: [scale C | shift C] (the weights' power-of-two scale folded into scale)
    const float *abias;            // [nopt][C][P]: the option encoding planes' share of the dynamics conv, times its BN scale
    BoardHead head[3];             // reward, value, policy (the policy head is K = chance_space_size wide in the afterstate program)
    int C, H, W;
    int nopt;                      // options of the program's dynamics conv (actions, or chance outcomes): rows of abias
    int nlayers;
    uint32_t layer_woff[kBoardMaxLayers];   // byte offset of the layer's conv weights in convw
    int layer_bn[kBoardMaxLayers];          // float offset of its [scale | shift] in bn
    int layer_flags[kBoardMaxLayers];
    float support_min, support_step;
};

struct BoardIO {
    int B, npass;
    const float *obs;              // [B][obs_c][H][W] (BF_OBS programs)
    int obs_c;
    const float *latent_base;      // input latents: base + ix[b] * slot_stride + b * C * P (NCHW)
    const int *ix;                 // or nullptr
    size_t slot_stride;
    const int *action;             // [B] options (actions or chance outcomes)
    float *latent_out, *latent_out2;   // [B][C][P] or nullptr
    float *reward, *value;         // [B] or nullptr
    float *policy_logits;          // [B][policy_stride] or nullptr
    float *reward_logits, *value_logits;   // [B][K] or nullptr
    int policy_stride;             // row stride of policy_logits (0: the policy head's width)
    // optional row mask: with row_mask, root b is computed only when (row_mask[b] & 1) == row_mask_on; any other root is an
    // absent root (its latent and option are not read, none of its outputs is written)
    const int *row_mask;
    int row_mask_on;
};

// plan of a launch: roots per CTA, 64-row tiles per CTA, CTAs, roots of the last CTA, shared memory bytes
struct BoardPlan { int R, NT, ctas, last, smem; };

BoardPlan board_plan(const BoardNet &net, int B);
int board_launch(const BoardNet &net, const BoardIO &io, cudaStream_t s);
int board_prepare_launch();      // opt-in shared memory sizes, set outside any stream capture
// packs one 3x3 conv (torch [C][cin_total][3][3], input channels [0, cin_used) of cin_pad) into the layout of BoardNet::convw;
// returns the power-of-two scale applied to the weights
float board_pack_conv3(const float *w, int C, int cin_total, int cin_used, int cin_pad, unsigned char *dst);

}  // namespace lz
