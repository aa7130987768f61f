// ez.cuh -- EfficientZero value-prefix head (lzero/model/efficientzero_model.py:552-569): one LSTM step over the flattened
// reward features as a batched GEMM across all roots, then BatchNorm1d -> ReLU -> MLP -> categorical expectation.
#pragma once
#include "net6.cuh"

namespace lz {

struct EzNet {
    const float *wcat;        // [nin + H][4H]: rows = inputs (reward features, then h_in), columns n = unit * 4 + gate (i, f, g, o)
    const float *bias;        // [4H] same column order: bias_ih + bias_hh
    const unsigned char *wtc; // tensor-core path: [n-tile 32][k-chunk 17][hi 8 KB | lo 8 KB], each [k-group 8][n 64][8 halves] fp16, scaled by wtc_scale
    float wtc_inv_scale;      // 1 / (power-of-two scale applied to wtc)
    const float *vp_s, *vp_t; // norm_value_prefix folded: y = relu(h' * s + t)
    const float *fc1;         // [H][hid] input-major
    const float *s2, *t2;     // [hid] (Linear bias folded)
    const float *fc2;         // [hid][K]
    const float *b2;          // [K]
    int nin, H, hid, K;
    float support_min, support_step;
};

struct EzIO {
    int B;
    const float *feat;        // [B][nin] from the conv kernel
    const float *h_base, *c_base;   // hidden-state source: base + ix[b] * slot_stride + b * H   (ix == nullptr: slot 0)
    const int *ix;
    size_t slot_stride;       // B * H
    float *h_out, *c_out;     // [B][H] next state (zeroed where is_reset[b], mcts_ctree.py:859-860)
    const int *is_reset;      // [B] or nullptr
    float *h_tmp;             // [B][H] un-reset h' (input of the value-prefix head)
    float *value_prefix;      // [B] scalar or nullptr
    float *vp_logits;         // [B][K] or nullptr
};

int ez_launch(const EzNet &net, const EzIO &io, cudaStream_t s);   // LSTM GEMM on the tensor cores (wgmma 3xFP16) where ez_tc_shape, else fp32 FFMA
int ez_prepare_launch();
bool ez_tc_shape(int nin, int H);   // k_ez_lstm_tc runs K = nin + H in whole chunks of 64 and N = 4H in tiles of 64
// host: pack W ([4H][nin] and [4H][H], torch gate order) into the tensor-core layout; returns the scale applied
size_t ez_wtc_bytes(int nin, int H);
float ez_pack_wtc(const float *w_ih, const float *w_hh, int nin, int H, unsigned char *dst);

}  // namespace lz
