// rezero.cu -- the policy-target reanalyze sweep of ReZero (ReZeroMZGameBuffer._compute_target_policy_reanalyzed,
// lzero/mcts/buffer/game_buffer_rezero_mz.py:194-404; ReZeroEZGameBuffer, game_buffer_rezero_ez.py:126-330) on the device.
//
// The reference runs initial_inference over the N*L sampled positions, splits them into L position groups, last position
// first (compute_all_filters, game_buffer_rezero_mz.py:19-26), searches the last group with a plain search and walks backward
// with L - 1 search_with_reuse calls, each reusing the root values of the group searched before it; then it turns the visit
// counts into [N, L, A] targets in Python.  Here the whole sweep is enqueued on the caller's stream with no host synchronisation:
//   initial_inference in mini_infer_size slices -> L x [k_rezero_handoff, captured search graph, k_rezero_targets].
// k_rezero_handoff gathers the next group's latents, true actions and (zero) LSTM state into the search's fixed buffers, copies
// the finished group's root values into the reuse-value buffer and resets + prepares the trees from the group's mask, logits,
// noise and to_play; so the captured graphs of lz_search_run / lz_search_run_with_reuse are replayed, never re-captured, along the sweep.
// Compiled with -fmad=false like tree.cu: the reset / prepare arithmetic is the tree's.
#include <limits.h>
#include <string.h>

#include <algorithm>

#include "lz_common.cuh"
#include "search.cuh"

namespace lz {

constexpr int kRezeroBlock = 64;   // one warp per root, as the tree kernels

// The caller's flat arrays, row i = segment * L + position (the reference's policy_obs_list order)
struct RezeroRows {
    int L;
    int latent_floats;
    const float *latent;        // [N*L][latent_floats]
    const float *logits;        // [N*L][A]
    const uint8_t *mask;        // [N*L][A]
    const int32_t *to_play;     // [N*L] or nullptr (-1)
    const int32_t *true_action; // [N*L]
    const float *noise;         // [N*L][A] legal order, or nullptr (prepare_no_noise)
    float noise_w;
};

// Between two searches of the sweep (and before the first): tree b becomes the root of segment b at position pos.
//   reuse_value[b] = root value of the search just finished (position pos + 1), read before the reset clears it;
//   pool0 (latent pool slot 0), true_action, h0 / c0 (EfficientZero LSTM state at the roots: zeros after initial_inference);
//   CRoots(legal from the mask) + prepare(noise, reward 0, logits, to_play) of the tree;
//   warp 0: players_max of the group (what the prepare of every root accumulates), a fresh tie-draw epoch, zeroed per-simulation
//   inference counts.
__global__ void __launch_bounds__(kRezeroBlock)
k_rezero_handoff(TreeParams p, RezeroRows r, int pos, int copy_values, float *pool0, int32_t *true_action, float *reuse_value,
                 float *h0, float *c0, int H)
{
    const int b = blockIdx.x * (kRezeroBlock / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= p.B) return;
    const int A = p.A;
    const size_t row = (size_t)b * r.L + pos;
    if (lane == 0) {
        if (copy_values) reuse_value[b] = tree_root_value(p, b);
        if (true_action) true_action[b] = r.true_action[row];
    }
    const int lf = r.latent_floats;
    for (int k = lane; k < lf; k += 32) pool0[(size_t)b * lf + k] = r.latent[row * lf + k];
    if (h0) {
        for (int k = lane; k < H; k += 32) {
            h0[(size_t)b * H + k] = 0.0f;
            c0[(size_t)b * H + k] = 0.0f;
        }
    }
    __syncwarp();
    tree_reset_root(p, b, lane, r.mask + row * A, nullptr, 0);
    __syncwarp();
    tree_prepare_root(p, b, lane, r.logits + row * A, r.noise ? r.noise + row * A : nullptr, r.noise_w, 0.0f,
                      r.to_play ? r.to_play[row] : -1);
    if (b == 0) {
        int m = INT_MIN;
        for (int k = lane; k < p.B; k += 32) m = max(m, r.to_play ? r.to_play[(size_t)k * r.L + pos] : -1);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0) {
            *p.players_max = m;
            *p.rng_epoch += 1ull;
        }
        for (int k = lane; k < p.N; k += 32) p.infer_count[k] = 0;
    }
}

// After the search of position pos: the rows segment * L + pos of the outputs.
//   child_visits[k] = visit_k / sum(visits) for the k-th legal action (float64 true division, as Python divides two ints: both
//   operands are exact, so the quotient is the correctly rounded one), zeros past the legal list;
//   targets = the same by legal position (fixed_action_space) or scattered to the action ids (scatter), zeros where policy_mask == 0;
//   root_values = get_values(); infer_out (reuse searches) = the per-simulation inference counts.
__global__ void __launch_bounds__(kRezeroBlock)
k_rezero_targets(TreeParams p, int L, int pos, const uint8_t *policy_mask, int scatter, double *targets, float *root_values,
                 double *child_visits, int32_t *infer_out, int S)
{
    const int b = blockIdx.x * (kRezeroBlock / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= p.B) return;
    const int A = p.A;
    const size_t row = (size_t)b * L + pos;
    const uint32_t *nb = p.edges + (size_t)b * p.N * kEdgeFields * A;      // root block
    const int *lg = p.legal + (size_t)b * A;
    const int n = p.nlegal[b];
    int sum = 0;
    for (int k = lane; k < n; k += 32) sum += (int)nb[F_VISIT * A + lg[k]];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const double total = (double)sum;
    double *tr = targets + row * A, *cv = child_visits + row * A;
    for (int a = lane; a < A; a += 32) {
        tr[a] = 0.0;
        cv[a] = 0.0;
    }
    __syncwarp();
    if (policy_mask[row] != 0) {
        for (int k = lane; k < n; k += 32) {
            const double v = __ddiv_rn((double)(int)nb[F_VISIT * A + lg[k]], total);
            cv[k] = v;
            tr[scatter ? lg[k] : k] = v;
        }
    }
    if (lane == 0) root_values[row] = tree_root_value(p, b);
    if (b == 0 && infer_out)
        for (int k = lane; k < S; k += 32) infer_out[k] = p.infer_count[k];
}

struct SweepArgs {
    int L, reuse, mini, deterministic, scatter;
    const float *obs, *latent, *logits;
    const uint8_t *mask, *policy_mask;
    const int32_t *to_play, *true_action;
    const float *noise;
    float noise_w;
    double *targets, *child_visits;
    float *root_values;
    int32_t *infer_count;
};

static int grow(float **buf, size_t floats)
{
    dev_free(*buf);
    *buf = nullptr;
    return dev_alloc(buf, floats);
}

static int sweep(lz_search *q, const SweepArgs &a, cudaStream_t s)
{
    lz_tree *t = q->tree;
    lz_model *m = q->model;
    const int N = q->B, A = q->A, L = a.L;
    LZ_REQUIRE(L >= 1, LZ_EINVAL, "lz_rezero_reanalyze: length L = %d must be >= 1", L);
    LZ_REQUIRE(a.mask && a.true_action && a.policy_mask && a.targets && a.root_values && a.child_visits, LZ_EINVAL,
               "lz_rezero_reanalyze: null argument");
    LZ_REQUIRE(a.obs ? !a.latent && !a.logits : a.latent && a.logits, LZ_EINVAL,
               "lz_rezero_reanalyze: pass the observations d_obs, or the latents d_latent and policy logits d_logits of a prior initial_inference");
    LZ_REQUIRE(!a.obs || a.mini > 0, LZ_EINVAL, "lz_rezero_reanalyze: mini_infer_size %d must be > 0", a.mini);
    LZ_REQUIRE(!(a.reuse && L > 1) || a.infer_count, LZ_EINVAL, "lz_rezero_reanalyze: d_infer_count is needed when L > 1 with reuse");
    LZ_REQUIRE(!t->gumbel, LZ_ESTATE, "lz_rezero_reanalyze: Gumbel tree (the sweep runs MuZero and EfficientZero trees)");
    LZ_REQUIRE(!t->p.nc, LZ_ESTATE, "lz_rezero_reanalyze: stochastic tree (the sweep runs MuZero and EfficientZero trees)");
    // search_with_reuse breaks ties with rand() only (cnode.cpp:610-640, ctree_efficientzero cnode.cpp:691): the first maximum, the
    // draw with rand() == 0.  Changing the rule re-captures the graphs once; a sweep keeps it.
    int rc = lz_tree_set_tiebreak(t, 1);
    if (rc == LZ_OK && a.reuse && L > 1) rc = search_reuse_buffers(q);
    if (rc) return rc;
    const size_t rows = (size_t)N * L;
    const float *latent = a.latent, *logits = a.logits;
    if (a.obs) {       // initial_inference over every row, in mini_infer_size slices (game_buffer_rezero_mz.py:243-262)
        if (rows > q->rz_rows) {
            q->rz_rows = 0;
            if ((rc = grow(&q->rz_latent, rows * m->latent_floats)) || (rc = grow(&q->rz_logits, rows * A))) return rc;
            q->rz_rows = rows;
        }
        const int slice = (int)std::min<size_t>((size_t)a.mini, rows);
        if ((rc = model_reserve(m, slice, s))) return rc;
        for (size_t beg = 0; beg < rows; beg += (size_t)slice) {
            const int cnt = (int)std::min<size_t>((size_t)slice, rows - beg);
            TailIO io;
            memset(&io, 0, sizeof(io));
            io.latent = q->rz_latent + beg * m->latent_floats;
            io.policy_logits = q->rz_logits + beg * A;
            if ((rc = model_initial(m, cnt, a.obs + beg * m->obs_elems, io, s))) return rc;
        }
        latent = q->rz_latent;
        logits = q->rz_logits;
    }
    RezeroRows r;
    r.L = L; r.latent_floats = m->latent_floats; r.latent = latent; r.logits = logits; r.mask = a.mask; r.to_play = a.to_play;
    r.true_action = a.true_action; r.noise = a.noise; r.noise_w = a.noise_w;
    const dim3 grid(ceil_div(N, kRezeroBlock / 32));
    const int H = q->hpool ? m->lstm_hidden : 0;
    for (int it = 0; it < L; ++it) {
        const int pos = L - 1 - it;
        const bool reuse = a.reuse && it > 0;
        k_rezero_handoff<<<grid, kRezeroBlock, 0, s>>>(t->p, r, pos, reuse ? 1 : 0, q->pool, reuse ? q->d_true_action : nullptr,
                                                        q->d_reuse_value, q->hpool, q->cpool, H);
        LZ_KERNEL_CHECK();
        t->prepared = true;
        if ((rc = search_run_graph(q, q->hpool ? 1 : a.deterministic, reuse, s))) return rc;
        k_rezero_targets<<<grid, kRezeroBlock, 0, s>>>(t->p, L, pos, a.policy_mask, a.scatter, a.targets, a.root_values,
                                                        a.child_visits, reuse ? a.infer_count + (size_t)(it - 1) * q->S : nullptr, q->S);
        LZ_KERNEL_CHECK();
    }
    return LZ_OK;
}

}  // namespace lz

using namespace lz;

extern "C" {

int lz_rezero_reanalyze(lz_search *q, int L, int reuse_search, int mini_infer_size, const float *d_obs, const float *d_latent,
                        const float *d_logits, const uint8_t *d_mask, const int32_t *d_to_play, const int32_t *d_true_action,
                        const uint8_t *d_policy_mask, const float *d_noise, float noise_weight, int deterministic, int scatter_legal,
                        double *d_targets, float *d_root_values, double *d_child_visits, int32_t *d_infer_count, lz_stream s)
{
    LZ_REQUIRE(q, LZ_EINVAL, "lz_rezero_reanalyze: null search");
    SweepArgs a = {L, reuse_search, mini_infer_size, deterministic, scatter_legal, d_obs, d_latent, d_logits, d_mask, d_policy_mask,
                   d_to_play, d_true_action, d_noise, noise_weight, d_targets, d_child_visits, d_root_values, d_infer_count};
    return sweep(q, a, (cudaStream_t)s);
}

}  // extern "C"
