// gumbel.cu -- Gumbel MuZero trees on the device: sequential halving with Gumbel noise at the root, completed-Q
// improved-policy selection below it (lzero/mcts/ctree/ctree_gumbel_muzero/lib/cnode.cpp), built on the lz_tree storage.
// Compiled with -fmad=false like tree.cu: every fp32 operation is an explicit round-to-nearest intrinsic, the sums run in
// the reference's sequential order, expf / logf are the glibc-exact restatements of lz_exact_math.h.
//
// One warp per tree.  The node pool, legal lists, paths, expand (softmax + noise), the back-up and the read-outs of
// visit counts / values / trajectories are the MuZero tree's; this file adds the completed-Q transform, the two
// selection rules and the improved-policy read-out, with its own state in GumbelParams.
#include <math.h>

#include <algorithm>
#include <cmath>
#include <random>
#include <vector>

#include "lz_common.cuh"
#include "gumbel.cuh"

namespace lz {

constexpr int kGumbelBlock = 64;   // 2 trees per CTA, as k_tree_step
static inline dim3 gumbel_grid(int B) { return dim3(ceil_div(B, kGumbelBlock / 32)); }

// Value at the FIRST position attaining the maximum (MAX) / minimum of the active lanes, folded into (best, have) in
// position order: std::max_element / min_element and csoftmax's running `>` maximum (cnode.cpp:917-922, 979-980).
template <bool MAX>
__device__ __forceinline__ void first_extreme(float x, bool act, float &best, bool &have)
{
    float v = act ? x : (MAX ? -INFINITY : INFINITY);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float w = __shfl_xor_sync(0xffffffffu, v, o);
        v = MAX ? fmaxf(v, w) : fminf(v, w);
    }
    const unsigned m = __ballot_sync(0xffffffffu, act && x == v);
    if (!m) return;
    const float c = __shfl_sync(0xffffffffu, x, __ffs(m) - 1);
    if (!have || (MAX ? c > best : c < best)) { best = c; have = true; }
}

// acc += x over the active lanes in lane order (a sequential fp32 loop of the reference)
__device__ __forceinline__ void seq_sum(float x, bool act, float &acc)
{
    unsigned m = __ballot_sync(0xffffffffu, act);
    while (m) {
        const int l = __ffs(m) - 1;
        m &= m - 1;
        acc = __fadd_rn(acc, __shfl_sync(0xffffffffu, x, l));
    }
}

__device__ __forceinline__ int warp_sum_int(int v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Per-node scalars of qtransform_completed_by_mix_value (cnode.cpp:988-1039, defaults maxvisit_init 50, value_scale 0.1,
// rescale on, epsilon 1e-8) for the n children of node block nb (position k -> action lg[k], or k when lg == nullptr).
struct NodeQ {
    float mp;       // max prior (first maximum)
    float lsum;     // logf of csoftmax's denominator over the priors
    float mixed;    // compute_mixed_value: the completed value of unvisited children
    float minv, gap, scale;
    int vsum;       // sum of child visits
};

__device__ __forceinline__ float child_q(const uint32_t *nb, int A, int a, float discount)
{
    const int vis = (int)nb[F_VISIT * A + a];
    return __fadd_rn(u2f(nb[F_REWARD * A + a]), __fmul_rn(discount, __fdiv_rn(u2f(nb[F_VSUM * A + a]), (float)vis)));
}

// csoftmax of the priors at one child (cnode.cpp:929-931), then std::max(p, -1e8) of compute_mixed_value (:955-957)
__device__ __forceinline__ float soft_prior(float prior, const NodeQ &s)
{
    const float sp = lz_expf_exact(__fsub_rn(__fsub_rn(prior, s.mp), s.lsum));
    return sp < -1e8f ? -1e8f : sp;
}

// completed and rescaled Q of one child (cnode.cpp:1018-1036)
__device__ __forceinline__ float completed_q(int vis, float q, const NodeQ &s)
{
    const float c = vis > 0 ? q : s.mixed;
    return __fmul_rn(__fmul_rn(__fdiv_rn(__fsub_rn(c, s.minv), s.gap), s.scale), 0.1f);
}

__device__ NodeQ node_q(const uint32_t *nb, int A, int n, const int *lg, float raw, float discount, int lane)
{
    NodeQ s;
    bool have = false;
    s.mp = 0.0f;
    for (int c0 = 0; c0 < n; c0 += 32) {
        const int k = c0 + lane;
        const bool act = k < n;
        const float p = act ? u2f(nb[F_PRIOR * A + (lg ? lg[k] : k)]) : 0.0f;
        first_extreme<true>(p, act, s.mp, have);
    }
    float sum = 0.0f;                                       // cnode.cpp:924-927
    for (int c0 = 0; c0 < n; c0 += 32) {
        const int k = c0 + lane;
        const bool act = k < n;
        const float e = act ? lz_expf_exact(__fsub_rn(u2f(nb[F_PRIOR * A + (lg ? lg[k] : k)]), s.mp)) : 0.0f;
        seq_sum(e, act, sum);
    }
    s.lsum = lz_logf_exact(sum);
    // compute_mixed_value (cnode.cpp:934-969)
    int vsum = 0, vmax = 0;
    float probs_sum = 0.0f;
    for (int c0 = 0; c0 < n; c0 += 32) {
        const int k = c0 + lane;
        const bool act = k < n;
        const int a = act ? (lg ? lg[k] : k) : 0;
        const int vis = act ? (int)nb[F_VISIT * A + a] : 0;
        const float sp = act ? soft_prior(u2f(nb[F_PRIOR * A + a]), s) : 0.0f;
        seq_sum(sp, act && vis > 0, probs_sum);
        vsum += warp_sum_int(vis);
        int mv = vis;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mv = max(mv, __shfl_xor_sync(0xffffffffu, mv, o));
        vmax = max(vmax, mv);
    }
    float wsum = 0.0f;
    for (int c0 = 0; c0 < n; c0 += 32) {
        const int k = c0 + lane;
        const bool act = k < n;
        const int a = act ? (lg ? lg[k] : k) : 0;
        const int vis = act ? (int)nb[F_VISIT * A + a] : 0;
        float term = 0.0f;
        if (vis > 0) term = __fdiv_rn(__fmul_rn(soft_prior(u2f(nb[F_PRIOR * A + a]), s), child_q(nb, A, a, discount)), probs_sum);
        seq_sum(term, vis > 0, wsum);
    }
    const float vsf = (float)vsum;                          // a sequential float sum of ints: exact below 2^24
    s.mixed = __fdiv_rn(__fadd_rn(raw, __fmul_rn(vsf, wsum)), __fadd_rn(vsf, 1.0f));
    s.vsum = vsum;
    // rescale_qvalues (cnode.cpp:971-986): first max / first min of the completed values
    float mx = 0.0f, mn = 0.0f;
    bool hx = false, hn = false;
    for (int c0 = 0; c0 < n; c0 += 32) {
        const int k = c0 + lane;
        const bool act = k < n;
        const int a = act ? (lg ? lg[k] : k) : 0;
        const int vis = act ? (int)nb[F_VISIT * A + a] : 0;
        const float c = vis > 0 ? child_q(nb, A, a, discount) : s.mixed;
        first_extreme<true>(c, act, mx, hx);
        first_extreme<false>(c, act, mn, hn);
    }
    const float gap = __fsub_rn(mx, mn);
    s.minv = mn;
    s.gap = gap < 1e-8f ? 1e-8f : gap;
    s.scale = __fadd_rn(50.0f, (float)vmax);
    return s;
}

// cselect_root_child (cnode.cpp:701-745) with score_considered (:1096-1131): the first strict maximum, legal[0] when every
// score is -inf.
__device__ int select_root(const uint32_t *nb, int A, int n, const int *lg, const NodeQ &s, const GumbelParams &g,
                           float discount, int lane)
{
    const int cv = g.considered[min(s.vsum, g.S - 1)];      // vsum < S: the host refuses descents past the table
    float best = -INFINITY;
    int best_k = 0;
    for (int c0 = 0; c0 < n; c0 += 32) {
        const int k = c0 + lane;
        const bool act = k < n;
        float sc = -INFINITY;
        if (act) {
            const int a = lg[k];
            const int vis = (int)nb[F_VISIT * A + a];
            const float cq = completed_q(vis, vis > 0 ? child_q(nb, A, a, discount) : 0.0f, s);
            float x = __fadd_rn(__fadd_rn(g.gumbel[k], __fsub_rn(u2f(nb[F_PRIOR * A + a]), s.mp)), cq);
            x = (-1e9f < x) ? x : -1e9f;
            sc = __fadd_rn(x, vis == cv ? 0.0f : -INFINITY);
        }
        const float cmax = warp_max_exact(sc);
        if (cmax > best) {
            best = cmax;
            best_k = c0 + __ffs(__ballot_sync(0xffffffffu, act && sc == cmax)) - 1;
        }
    }
    return lg[best_k];
}

// cselect_interior_child (cnode.cpp:747-790): argmax of softmax(prior + cq) - visits / (1 + sum visits) over all A children
__device__ int select_interior(const uint32_t *nb, int A, const NodeQ &s, float discount, int lane)
{
    float m = 0.0f;
    bool have = false;
    for (int c0 = 0; c0 < A; c0 += 32) {
        const int a = c0 + lane;
        const bool act = a < A;
        float x = 0.0f;
        if (act) {
            const int vis = (int)nb[F_VISIT * A + a];
            x = __fadd_rn(u2f(nb[F_PRIOR * A + a]), completed_q(vis, vis > 0 ? child_q(nb, A, a, discount) : 0.0f, s));
        }
        first_extreme<true>(x, act, m, have);
    }
    float sum = 0.0f;
    for (int c0 = 0; c0 < A; c0 += 32) {
        const int a = c0 + lane;
        const bool act = a < A;
        float e = 0.0f;
        if (act) {
            const int vis = (int)nb[F_VISIT * A + a];
            const float x = __fadd_rn(u2f(nb[F_PRIOR * A + a]), completed_q(vis, vis > 0 ? child_q(nb, A, a, discount) : 0.0f, s));
            e = lz_expf_exact(__fsub_rn(x, m));
        }
        seq_sum(e, act, sum);
    }
    const float lsum = lz_logf_exact(sum);
    const float denom = (float)(1 + s.vsum);
    float best = -INFINITY;
    int best_a = 0;
    for (int c0 = 0; c0 < A; c0 += 32) {
        const int a = c0 + lane;
        const bool act = a < A;
        float sc = -INFINITY;
        if (act) {
            const int vis = (int)nb[F_VISIT * A + a];
            const float x = __fadd_rn(u2f(nb[F_PRIOR * A + a]), completed_q(vis, vis > 0 ? child_q(nb, A, a, discount) : 0.0f, s));
            const float pr = lz_expf_exact(__fsub_rn(__fsub_rn(x, m), lsum));
            sc = __fsub_rn(pr, __fdiv_rn((float)vis, denom));
        }
        const float cmax = warp_max_exact(sc);
        if (cmax > best) {
            best = cmax;
            best_a = c0 + __ffs(__ballot_sync(0xffffffffu, act && sc == cmax)) - 1;
        }
    }
    return best_a;
}

// cbatch_traverse (cnode.cpp:834-897) for tree b; virtual_to_play passes through unchanged.
__device__ void gumbel_traverse(const TreeParams &p, const GumbelParams &g, int b, int lane, int *out_ix, int *out_action)
{
    const int A = p.A, N = p.N;
    const uint32_t *tree_edges = p.edges + (size_t)b * N * kEdgeFields * A;
    const int *lg = p.legal + (size_t)b * A;
    const int nl = p.nlegal[b];
    int *pslot = p.path_slot + (size_t)b * N, *pact = p.path_action + (size_t)b * N;
    int slot = 0, plen = 0, action = 0;
    while (true) {
        const uint32_t *nb = tree_edges + (size_t)slot * kEdgeFields * A;
        const bool is_root = plen == 0;
        const float raw = g.raw_value[(size_t)b * N + slot];
        const NodeQ s = node_q(nb, A, is_root ? nl : A, is_root ? lg : nullptr, raw, p.discount, lane);
        action = is_root ? select_root(nb, A, nl, lg, s, g, p.discount, lane) : select_interior(nb, A, s, p.discount, lane);
        if (lane == 0) {
            p.n_best[(size_t)b * N + slot] = action;
            pslot[plen] = slot;
            pact[plen] = action;
        }
        ++plen;
        const int cs = (int)nb[F_CSLOT * A + action];
        if (cs < 0 || plen >= N) break;
        slot = cs;
    }
    if (lane == 0) {
        p.path_len[b] = plen;
        p.search_len[b] = plen;
        p.vtp[b] = p.to_play[b];
        if (out_ix) out_ix[b] = slot;
        if (out_action) out_action[b] = action;
    }
    __syncwarp();
}

__global__ void __launch_bounds__(kGumbelBlock)
k_gumbel_root_values(TreeParams p, GumbelParams g, const float *values)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < p.B) g.raw_value[(size_t)b * p.N] = values[b];   // CRoots::prepare: expand(..., values[i], ...) (cnode.cpp:432)
}

__global__ void __launch_bounds__(kGumbelBlock)
k_gumbel_step(TreeParams p, GumbelParams g, TreeStep a)
{
    const int b = blockIdx.x * (kGumbelBlock / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= p.B) return;
    if (a.latent_index > 0) {         // cbatch_back_propagate (cnode.cpp:633-652): expand (raw_value = value), one-player back-up
        const float value = a.value[b];
        if (lane == 0 && p.path_len[b] > 0 && a.latent_index < p.N) g.raw_value[(size_t)b * p.N + a.latent_index] = value;
        tree_backprop<false, false, true>(p, b, lane, a.latent_index, a.reward[b], value, a.logits + (size_t)b * p.A, a.to_play);
    }
    if (a.traverse) {
        gumbel_traverse(p, g, b, lane, a.ix, a.act);
        if (lane == 0) {
            if (a.iy) a.iy[b] = b;
            if (a.len) a.len[b] = p.search_len[b];
            if (a.vtp) a.vtp[b] = p.vtp[b];
        }
    }
}

// get_children_values / get_policies (cnode.cpp:309-385, 506-541): completed Q at the legal positions (-inf elsewhere) and
// csoftmax over all A entries of prior + completed Q (-inf at illegal positions, which come out as 0).
__global__ void __launch_bounds__(kGumbelBlock)
k_gumbel_policies(TreeParams p, GumbelParams g, float *children_values, float *policy)
{
    const int b = blockIdx.x * (kGumbelBlock / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= p.B) return;
    const int A = p.A, N = p.N;
    const uint32_t *nb = p.edges + (size_t)b * N * kEdgeFields * A;
    const int *lg = p.legal + (size_t)b * A;
    const int n = p.nlegal[b];
    const NodeQ s = node_q(nb, A, n, lg, g.raw_value[(size_t)b * N], p.discount, lane);
    float *cv = children_values ? children_values + (size_t)b * A : nullptr;
    float *pol = policy ? policy + (size_t)b * A : nullptr;
    if (cv) {
        for (int a = lane; a < A; a += 32) cv[a] = -INFINITY;
        __syncwarp();
        for (int k = lane; k < n; k += 32) {
            const int a = lg[k], vis = (int)nb[F_VISIT * A + a];
            cv[a] = completed_q(vis, vis > 0 ? child_q(nb, A, a, p.discount) : 0.0f, s);
        }
    }
    if (!pol) return;
    // probs[a] by action id: the legal position of a is found by a scan of the legal list (lane-parallel, A <= a few hundred)
    auto logit = [&](int a) -> float {
        for (int k = 0; k < n; ++k)
            if (lg[k] == a) {
                const int vis = (int)nb[F_VISIT * A + a];
                return __fadd_rn(u2f(nb[F_PRIOR * A + a]), completed_q(vis, vis > 0 ? child_q(nb, A, a, p.discount) : 0.0f, s));
            }
        return -INFINITY;
    };
    float m = 0.0f;
    bool have = false;
    for (int c0 = 0; c0 < A; c0 += 32) {
        const int a = c0 + lane;
        first_extreme<true>(a < A ? logit(a) : 0.0f, a < A, m, have);
    }
    float sum = 0.0f;
    for (int c0 = 0; c0 < A; c0 += 32) {
        const int a = c0 + lane;
        seq_sum(a < A ? lz_expf_exact(__fsub_rn(logit(a), m)) : 0.0f, a < A, sum);
    }
    const float lsum = lz_logf_exact(sum);
    for (int a = lane; a < A; a += 32) pol[a] = lz_expf_exact(__fsub_rn(__fsub_rn(logit(a), m), lsum));
}

int gumbel_launch_step(lz_tree *t, const TreeStep &a, cudaStream_t s)
{
    k_gumbel_step<<<gumbel_grid(t->p.B), kGumbelBlock, 0, s>>>(t->p, t->gumbel->g, a);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

void gumbel_free(lz_tree *t)
{
    if (!t || !t->gumbel) return;
    cudaFree(t->gumbel->alloc);
    delete t->gumbel;
    t->gumbel = nullptr;
}

// get_sequence_of_considered_visits (cnode.cpp:1041-1076) for row min(m, S) of get_table_of_considered_visits, and
// generate_gumbel(10, 0, A) (:1133-1151).  Same integer arithmetic, the double log2 and the float Gumbel draws of libstdc++.
void gumbel_host_tables(int m, int S, int A, int *seq, float *gumbel)
{
    if (seq) {
        const int mm = std::min(m, S);
        std::vector<int> out;
        if (mm <= 1) {
            for (int i = 0; i < S; ++i) out.push_back(i);
        } else {
            const int log2max = (int)std::ceil(std::log2(mm));
            std::vector<int> visits(mm, 0);
            int nc = mm;
            while ((int)out.size() < S) {
                const int extra = std::max(1, S / (log2max * nc));
                for (int i = 0; i < extra; ++i) {
                    out.insert(out.end(), visits.begin(), visits.begin() + nc);
                    for (int j = 0; j < nc; ++j) visits[j] += 1;
                }
                nc = std::max(2, nc / 2);
            }
        }
        std::copy(out.begin(), out.begin() + S, seq);
    }
    if (gumbel) {
        const float scale = 10.0f, rng = 0.0f;            // CNode: gumbel_scale = 10, gumbel_rng = 0
        std::mt19937 gen(static_cast<unsigned int>(rng));
        std::extreme_value_distribution<float> d(0, 1);
        for (int i = 0; i < A; ++i) gumbel[i] = scale * d(gen);
    }
}

}  // namespace lz

using namespace lz;

extern "C" {

int lz_gumbel_tables(int max_num_considered_actions, int num_simulations, int A, int32_t *h_seq, float *h_gumbel)
{
    LZ_REQUIRE(max_num_considered_actions >= 0 && num_simulations > 0 && A >= 0, LZ_EINVAL,
               "lz_gumbel_tables: bad arguments m=%d S=%d A=%d", max_num_considered_actions, num_simulations, A);
    gumbel_host_tables(max_num_considered_actions, num_simulations, A, h_seq, h_gumbel);
    return LZ_OK;
}

int lz_tree_set_gumbel(lz_tree *t, int max_num_considered_actions, int num_simulations)
{
    LZ_REQUIRE(t, LZ_EINVAL, "lz_tree_set_gumbel: null tree");
    if (num_simulations == 0) {                 // back to a MuZero tree
        if (t->gumbel) { gumbel_free(t); ++t->generation; }
        return LZ_OK;
    }
    LZ_REQUIRE(!t->p.ez, LZ_ESTATE, "lz_tree_set_gumbel: tree is in EfficientZero mode (the Gumbel tree is a MuZero tree)");
    LZ_REQUIRE(max_num_considered_actions >= 0 && num_simulations > 0, LZ_EINVAL,
               "lz_tree_set_gumbel: bad arguments max_num_considered_actions=%d num_simulations=%d",
               max_num_considered_actions, num_simulations);
    if (t->gumbel && t->gumbel->g.m == max_num_considered_actions && t->gumbel->g.S == num_simulations) return LZ_OK;
    const int A = t->p.A, S = num_simulations;
    std::vector<int> seq(S);
    std::vector<float> gum(A);
    gumbel_host_tables(max_num_considered_actions, S, A, seq.data(), gum.data());
    gumbel_free(t);
    lz_gumbel *gs = new lz_gumbel();
    memset(gs, 0, sizeof(*gs));
    const size_t o_gum = 0, o_seq = (size_t)((A + 31) & ~31), o_raw = o_seq + (size_t)((S + 31) & ~31);
    const size_t words = o_raw + (size_t)t->p.B * t->p.N;
    uint32_t *base = nullptr;
    int rc = dev_alloc(&base, words);
    if (rc != LZ_OK) { delete gs; return rc; }
    gs->alloc = base;
    t->gumbel = gs;
    gs->g.m = max_num_considered_actions;
    gs->g.S = S;
    gs->g.gumbel = (const float *)(base + o_gum);
    gs->g.considered = (const int *)(base + o_seq);
    gs->g.raw_value = (float *)(base + o_raw);
    LZ_CUDA_CHECK(cudaMemset(base, 0, words * 4));
    LZ_CUDA_CHECK(cudaMemcpy(base + o_gum, gum.data(), A * sizeof(float), cudaMemcpyHostToDevice));
    LZ_CUDA_CHECK(cudaMemcpy(base + o_seq, seq.data(), S * sizeof(int), cudaMemcpyHostToDevice));
    ++t->generation;                             // captured search graphs bake GumbelParams in
    return LZ_OK;
}

int lz_tree_prepare_gumbel(lz_tree *t, const float *d_logits, const float *d_noise, float noise_weight, const float *d_rewards,
                           const float *d_values, const int32_t *d_to_play, lz_stream s)
{
    LZ_REQUIRE(t && d_logits && d_values, LZ_EINVAL, "lz_tree_prepare_gumbel: null argument");
    LZ_REQUIRE(t->gumbel, LZ_ESTATE, "lz_tree_prepare_gumbel: not a Gumbel tree (lz_tree_set_gumbel)");
    int rc = lz_tree_prepare(t, d_logits, d_noise, noise_weight, d_rewards, d_to_play, s);
    if (rc != LZ_OK) return rc;
    k_gumbel_root_values<<<ceil_div(t->p.B, kGumbelBlock), kGumbelBlock, 0, (cudaStream_t)s>>>(t->p, t->gumbel->g, d_values);
    LZ_KERNEL_CHECK();
    t->gumbel->prepared = true;
    t->gumbel->pending = false;
    t->gumbel->traversals = 0;
    return LZ_OK;
}

int lz_tree_traverse_gumbel(lz_tree *t, int32_t *d_ix, int32_t *d_iy, int32_t *d_last_action, int32_t *d_search_len,
                            int32_t *d_virtual_to_play, lz_stream s)
{
    LZ_REQUIRE(t && t->gumbel, LZ_ESTATE, "lz_tree_traverse_gumbel: not a Gumbel tree (lz_tree_set_gumbel)");
    lz_gumbel *gs = t->gumbel;
    LZ_REQUIRE(gs->prepared, LZ_ESTATE, "lz_tree_traverse_gumbel: roots not prepared (call lz_tree_prepare_gumbel first)");
    LZ_REQUIRE(gs->traversals < gs->g.S, LZ_ESTATE,
               "lz_tree_traverse_gumbel: %d descents after one prepare would index past the considered-visit table of "
               "num_simulations = %d", gs->traversals + 1, gs->g.S);
    TreeStep a = {};
    a.traverse = 1;
    a.ix = d_ix; a.iy = d_iy; a.act = d_last_action; a.len = d_search_len; a.vtp = d_virtual_to_play;
    int rc = gumbel_launch_step(t, a, (cudaStream_t)s);
    if (rc != LZ_OK) return rc;
    ++gs->traversals;
    gs->pending = true;
    return LZ_OK;
}

int lz_tree_backpropagate_gumbel(lz_tree *t, int latent_index, const float *d_reward, const float *d_value, const float *d_logits,
                                 const int32_t *d_to_play, lz_stream s)
{
    LZ_REQUIRE(t && d_reward && d_value && d_logits, LZ_EINVAL, "lz_tree_backpropagate_gumbel: null argument");
    LZ_REQUIRE(t->gumbel, LZ_ESTATE, "lz_tree_backpropagate_gumbel: not a Gumbel tree (lz_tree_set_gumbel)");
    LZ_REQUIRE(t->gumbel->pending, LZ_ESTATE, "lz_tree_backpropagate_gumbel: no descent to back up (call lz_tree_traverse_gumbel first)");
    LZ_REQUIRE(latent_index >= 1 && latent_index <= t->max_sims, LZ_EINVAL,
               "lz_tree_backpropagate_gumbel: latent_index %d outside [1, %d]", latent_index, t->max_sims);
    TreeStep a = {};
    a.latent_index = latent_index; a.reward = d_reward; a.value = d_value; a.logits = d_logits; a.to_play = d_to_play;
    int rc = gumbel_launch_step(t, a, (cudaStream_t)s);
    if (rc != LZ_OK) return rc;
    t->gumbel->pending = false;
    return LZ_OK;
}

int lz_tree_gumbel_policies(lz_tree *t, float *d_children_values, float *d_improved_policy, lz_stream s)
{
    LZ_REQUIRE(t && t->gumbel, LZ_ESTATE, "lz_tree_gumbel_policies: not a Gumbel tree (lz_tree_set_gumbel)");
    LZ_REQUIRE(t->gumbel->prepared, LZ_ESTATE, "lz_tree_gumbel_policies: roots not prepared (call lz_tree_prepare_gumbel first)");
    k_gumbel_policies<<<gumbel_grid(t->p.B), kGumbelBlock, 0, (cudaStream_t)s>>>(t->p, t->gumbel->g, d_children_values, d_improved_policy);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

}  // extern "C"
