// gumbel.cuh -- Gumbel MuZero mode of the device trees (gumbel.cu): the state it adds beside TreeParams.
#pragma once
#include "tree.cuh"

namespace lz {

// Passed by value NEXT TO TreeParams (which stays unchanged, so the MuZero / EfficientZero kernels are untouched).
struct GumbelParams {
    int m, S;                 // max_num_considered_actions, num_simulations
    const float *gumbel;      // [A] 10 * Gumbel(0, 1) draws of std::mt19937(0): a root with n legal actions uses [0, n)
    const int *considered;    // [S] row min(m, S) of the considered-visit table (sequential halving)
    float *raw_value;         // [B][N] value-network estimate of every expanded node (CNode::raw_value)
};

// Host-side tables of the reference (ctree_gumbel_muzero/lib/cnode.cpp:1041-1076, 1133-1151), computed with <random> and
// the same float / double overloads as the reference binary.
void gumbel_host_tables(int m, int S, int A, int *seq, float *gumbel);

// One k_gumbel_step launch: back-up of latent_index (> 0), then the next Gumbel descent (a.traverse).
int gumbel_launch_step(lz_tree *t, const TreeStep &a, cudaStream_t s);
void gumbel_free(lz_tree *t);

}  // namespace lz

struct lz_gumbel {
    lz::GumbelParams g;
    void *alloc;
    bool prepared;            // lz_tree_prepare_gumbel since the last reset / prepare
    bool pending;             // a descent waits for its back-up
    int traversals;           // descents since the last prepare (the table has S columns)
};
