// net_tc.cuh -- interface of the tensor-core (wgmma) network path (net_tc.cu).
#pragma once
#include "lz_common.cuh"
#include "net6.cuh"
#include "tree.cuh"

namespace lz {

constexpr int kMaxResBlocksTc = 4;
constexpr int kTcMaxLayers = 1 + 4 * kMaxResBlocksTc;

struct TcFc {                      // fully connected part of one head on the tensor cores (net_tc.cu, heads section)
    uint32_t fc2_off;              // byte offset into TcNet::fcw of this head's FC2 tiles ([ceil(K/128)][hi 8 KB | lo 8 KB], [kg 4][128 outputs][8])
    int nin, K;                    // FC1 inputs (hc*P), FC2 outputs (0: the head has no FC part here)
    float fc1_inv, fc2_inv;        // 1 / the power-of-two scale applied to the fp16 weights
};

struct TcNet {
    const unsigned char *convw;    // [nconv][9 taps][8 k-groups][64 hi rows | 64 lo rows][8] fp16, K-major core-matrix layout
    const float *bn;               // [nconv][scale 64 | shift 64] (weight power-of-two scale folded in)
    const unsigned char *headw;    // [reward hi 2K | lo 2K][value+policy hi 4K | lo 4K]
    const float *head_bn;          // [reward s16 t16 | value s16 t16 | policy s16 t16]
    const float *abias;            // [A][16][P][4] ([c / 4][pixel][c % 4]) action-plane contribution of the dynamics conv, x BN scale
    const unsigned char *fcw;      // FC weight stream: 16 P / 32 FC1 stages of 12 KB ([2 k-steps][hi 3 KB | lo 3 KB], [kg 2][96 rows = 32 head + unit][8]) then the FC2 tiles
    TcFc fc[3];                    // reward, value, policy
    int hw;                        // latent grid hw x hw: 6 (84 / 96-pixel observations) or 8 (64): selects the k_net_tc instantiation
    Head reward, value, policy;    // folded BN / bias tables of the FC parts (fp32, in lz_model::d_weights)
    int hc[3];
    int nlayers;
    int layer_w[kTcMaxLayers];     // conv index into convw / bn
    int layer_flags[kTcMaxLayers];
    int has_reward;
    int A;
    float support_min, support_step;
};

struct TcIO {
    int B;
    int roots_per_cta;             // filled by tc_launch
    int npass;                     // 3 = fp32-accurate (hi*hi + hi*lo + lo*hi), 1 = fast (hi*hi)
    const float *latent_base;      // input latents: base + ix[b]*slot_stride + b*64*P (NCHW [64][P])
    const int *ix;                 // or nullptr
    size_t slot_stride;
    const int *action;             // [B] (recurrent) or nullptr
    float *latent_out, *latent_out2;   // [B][64][P] or nullptr
    float *reward, *value;         // [B] scalars
    float *policy_logits;          // [B][A]
    float *reward_logits, *value_logits;   // [B][K] or nullptr
    // persistent search (the whole num_simulations loop in one launch; tree + network per CTA of up to 8 (6x6) / 4 (8x8) roots)
    int persistent, nsims, sim0, deterministic;
    int *ix_rw, *action_rw;        // [B] tree -> network hand-off (same arrays as ix / action)
    float *latent_pool_rw;         // == latent_base; slot s+1 receives the latents of simulation s
    float *skip_scratch;           // [B][16][P][4] fp32: ResBlock skip tensors parked between layers (thread-private rows, L2-resident)
    int pool_cl;                   // latent pool slots >= 1 and latent_out use the kernel-internal [c / 4][P][c % 4] layout (persistent search); else NCHW
    float *ez_feat;                // EfficientZero: the reward head stops after conv1x1+BN+ReLU and writes [B][hc*P] here
    unsigned long long *dbg;       // optional [64] clock64 stamps of CTA 0 (bring-up instrumentation)
};

enum : int { LF_RES = 1, LF_STORE_RES = 2, LF_WRITE_LATENT = 4, LF_ACT_BIAS = 8, LF_HOOK_REWARD = 16, LF_HOOK_VALPOL = 32 };

float tc_pack_conv3(const float *w_torch, int cin_total, int cin_used, unsigned char *dst);
float tc_pack_conv1(const float *w, int hc, int nco, int co_offset, unsigned char *dst_hi, unsigned char *dst_lo);
int tc_head_layout_bytes();
int tc_conv_layout_bytes();
int tc_prepare_launch();
int tc_launch(const TcNet &net, const TcIO &io, cudaStream_t s, const TreeParams *tp = nullptr);
void tc_describe(const TcNet &net, const TcIO &io, int32_t *info);   // info[8]: the plan of tc_launch(net, io) (net_tc.cu)
void tc_describe_search(const TcNet &net, const TcIO &io, int N, int32_t *info);   // info[6]: the plan of a persistent search launch
unsigned long long *tc_debug_buffer();   // device buffer [64] used when env LZ_TC_DEBUG=1

}  // namespace lz
