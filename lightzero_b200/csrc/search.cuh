// search.cuh -- the fused search object (lz_search) shared by search.cu and the ReZero reanalyze sweep (rezero.cu).
#pragma once
#include "model.cuh"
#include "tree.cuh"

struct SearchGraph {              // one instantiated search graph and what it baked in
    cudaGraphExec_t exec;
    unsigned long long gen_model, gen_tree;   // model / tree generation at capture
    int num_kernels;              // kernel nodes
};

struct lz_search {
    lz_tree *tree;
    lz_model *model;
    int S, B, A;
    float *pool;                 // [(S+1)][B][C*P] latent pool, slot-major, NCHW per root
    size_t slot_stride;          // B*C*P floats
    int32_t *d_ix, *d_action;    // [B]
    float *d_reward, *d_value;   // [B]
    float *d_policy;             // [B][A]
    float *d_root_logits;        // [B][A]
    float *d_root_value;         // [B]
    float *d_skip;               // [B][C*P] ResBlock skip scratch of the tensor-core network kernel (per search: searches may overlap on streams)
    // EfficientZero: LSTM state pools [(S+1)][B][H] (tuple element 0 / 1 of reward_hidden_state, mcts_ctree.py:775-776)
    // and the per-leaf is_reset flags handed from the traverse to the LSTM kernel and the back-up (:856-861)
    float *hpool, *cpool;
    size_t hslot_stride;
    int32_t *d_is_reset;
    // Stochastic MuZero: the depth of each leaf the last descent reached; its parity selects the recurrent program of the row
    int32_t *d_len;
    // ReZero search_with_reuse: library-owned copies of the caller's per-root true action / reuse value (graph-stable addresses)
    int32_t *d_true_action;
    float *d_reuse_value;
    SearchGraph graphs[4];       // plain search with deterministic 0 / 1, search with reuse, Gumbel search
    cudaStream_t capture_stream; // library-owned: the caller's stream may be the legacy default stream,
                                 // which cannot be captured; the instantiated graph launches on the caller's
    int num_kernels;             // kernel nodes of the graph launched last
    // host-buffer collect: staging + copy stream so the H2D of chunk i+1 overlaps the tower of chunk i
    cudaStream_t copy_stream, copy_stream2;   // chunks alternate between two copy streams (two DMA engines)
    cudaEvent_t ev_chunk[8], ev_start;
    float *d_obs_stage, *d_noise_stage, *d_pre_stage;
    uint8_t *d_mask_stage;
    int32_t *d_tp_stage;
    size_t obs_elems;            // floats per observation
    // ReZero reanalyze sweep (rezero.cu): initial_inference of all N*L rows, latents [rows][latent_floats] and logits [rows][A]
    float *rz_latent, *rz_logits;
    size_t rz_rows;
};

namespace lz {
// Launches the captured search graph of q on s: the plain search (MuZero: with this deterministic flag; EfficientZero: the tree's
// tie rule) or, with reuse, search_with_reuse on q->d_true_action / q->d_reuse_value.  The graph is captured on the first call
// and again only after the model, the tree parameters or the tie rule changed (generation counters).
int search_run_graph(lz_search *q, int deterministic, bool reuse, cudaStream_t s);
// Allocates q->d_true_action / q->d_reuse_value on first use.
int search_reuse_buffers(lz_search *q);
}  // namespace lz
