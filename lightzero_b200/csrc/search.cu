// search.cu -- the whole MuZeroMCTSCtree.search loop (lzero/mcts/tree_search/mcts_ctree.py:267-368) as ONE
// CUDA graph: [traverse] + num_simulations x [recurrent_inference -> backpropagate(+next traverse)].
// The reference's per-simulation host work (Python list gather of latents :323-324, two H2D copies
// :326-329, a duplicated recurrent_inference :338/:345, four blocking D2H copies :347-350 and three
// .tolist() conversions :355-357) has no counterpart here: the tree hands (slot, action) to the
// network through device memory and the network hands (reward, value, logits) back the same way.
#include <string.h>

#include <algorithm>
#include <atomic>

#include "gumbel.cuh"
#include "search.cuh"

using namespace lz;

// recurrent_inference of simulation sim: latents (and EfficientZero LSTM state) gathered at the slots the descent left in d_ix,
// results into pool slot sim + 1 (mcts_ctree.py:352,364) and the tree hand-off buffers
static RecIO rec_io(const lz_search *q, int sim)
{
    RecIO io;
    memset(&io, 0, sizeof(io));
    io.B = q->B; io.latent_base = q->pool; io.ix = q->d_ix; io.slot_stride = q->slot_stride; io.action = q->d_action;
    io.next_latent = q->pool + (size_t)(sim + 1) * q->slot_stride;
    io.reward = q->d_reward; io.value = q->d_value; io.policy_logits = q->d_policy;
    io.skip_scratch = q->d_skip;
    if (q->hpool) {
        io.h_base = q->hpool; io.c_base = q->cpool; io.hslot_stride = q->hslot_stride;
        io.h_out = q->hpool + (size_t)(sim + 1) * q->hslot_stride; io.c_out = q->cpool + (size_t)(sim + 1) * q->hslot_stride;
        io.is_reset = q->d_is_reset;
    }
    return io;
}

// Persistent search: roots never interact, so the CTA that owns up to 8 roots can run their whole search -- tree
// back-up / descent and the network -- for all num_simulations inside ONE launch of the tensor-core kernel.
// EfficientZero stays a multi-kernel graph: its LSTM step is a GEMM over all roots (several launches per simulation).
static bool persistent_search(const lz_search *q, bool reuse)
{
    return !reuse && !q->tree->gumbel && !q->hpool && q->model->family == ModelFamily::Conv && q->tree->p.A <= 32;   // tree_persist.cuh: one lane per child
}

static TcIO persistent_io(const lz_search *q, int deterministic)
{
    TcIO io;
    memset(&io, 0, sizeof(io));
    io.B = q->B; io.npass = q->model->npass;
    io.latent_base = q->pool; io.latent_pool_rw = q->pool; io.slot_stride = q->slot_stride;
    io.ix = q->d_ix; io.ix_rw = q->d_ix; io.action = q->d_action; io.action_rw = q->d_action;
    io.reward = q->d_reward; io.value = q->d_value; io.policy_logits = q->d_policy;
    io.persistent = 1; io.nsims = q->S; io.sim0 = 0; io.deterministic = deterministic;
    io.skip_scratch = q->d_skip;
    io.pool_cl = 1;      // slots >= 1 are written and read only by this kernel: channels-last (vector loads / stores); slot 0 stays NCHW
    return io;
}

// recurrent_inference of simulation sim.  A Stochastic MuZero model runs two programs, each on its own rows and into the same
// pool slot and hand-off buffers: the afterstate program on the rows whose leaf is a chance node (odd depth, search_len in
// d_len), then the dynamics program on the others (mcts_ctree_stochastic.py:171-212).
static int recurrent_step(const lz_search *q, int sim, cudaStream_t s)
{
    RecIO io = rec_io(q, sim);
    if (!q->d_len) return model_recurrent(q->model, io, s);
    io.row_mask = q->d_len; io.policy_stride = q->A;
    for (int chance = 1; chance >= 0; --chance) {
        io.after_program = chance; io.row_mask_on = chance;
        if (int rc = model_recurrent(q->model, io, s)) return rc;
    }
    return LZ_OK;
}

// MuZeroMCTSCtree.search (mcts_ctree.py:267-368), EfficientZeroMCTSCtree.search (:671-876) and their search_with_reuse variants
// (:370-468, :878-1003), GumbelMuZeroMCTSCtree.search (:1076-1172) and StochasticMuZeroMCTSCtree.search
// (mcts_ctree_stochastic.py:117-252): [descent] + S x [recurrent_inference, back-up (+ next descent)], each tree step the
// kernel of the tree's mode (tree_launch_step).  Under reuse every tree goes through the network every simulation (the
// reference compacts the batch on the host; here the rows of "no inference" trees are computed and ignored, which keeps the
// loop one static CUDA graph).  The stochastic reference splits the leaves on the host and backs up the two subsets one
// after the other; the trees are independent, so one back-up of every tree is the same.
static int enqueue_search(lz_search *q, int deterministic, bool reuse, cudaStream_t s)
{
    int rc;
    lz_tree *t = q->tree;
    if (!t->gumbel) t->step_counter = 0;      // the Gumbel descent takes no RNG step and leaves the counter as it is
    if (persistent_search(q, reuse)) return tc_launch(q->model->conv.tc_rec, persistent_io(q, deterministic), s, &t->p);
    TreeStep descent = {};
    descent.traverse = 1; descent.deterministic = deterministic;
    descent.act = q->d_action; descent.is_reset = q->d_is_reset; descent.len = q->d_len;
    if (reuse) {
        descent.true_action = q->d_true_action; descent.reuse_value = q->d_reuse_value;
        descent.ix_net = q->d_ix;
    } else {
        descent.ix = q->d_ix;
    }
    // the EfficientZero reuse back-up and the next descent are separate launches
    const bool fuse = !(reuse && q->hpool);
    if ((rc = tree_launch_step(t, descent, s))) return rc;
    for (int sim = 0; sim < q->S; ++sim) {
        if ((rc = recurrent_step(q, sim, s))) return rc;
        const bool next = sim + 1 < q->S;
        TreeStep step = descent;
        step.traverse = next && fuse;
        step.latent_index = sim + 1;
        step.reward = q->d_reward; step.value = q->d_value; step.logits = q->d_policy; step.leaf_reset = q->d_is_reset;
        if ((rc = tree_launch_step(t, step, s))) return rc;
        if (next && !fuse && (rc = tree_launch_step(t, descent, s))) return rc;
    }
    return LZ_OK;
}

static std::atomic<unsigned long long> g_captures{0};   // lz_debug_graph_captures

int lz::search_run_graph(lz_search *q, int deterministic, bool reuse, cudaStream_t s)
{
    // an EfficientZero plain search breaks ties by p.tie_first (tracked by the tree generation), not by the flag: one graph
    SearchGraph &g = q->graphs[q->tree->gumbel ? 3 : reuse ? 2 : (deterministic || q->hpool) ? 1 : 0];
    // a captured graph bakes in device pointers of the model's tables (passed by value in TcNet / EzNet), the pass count
    // and the tree parameters (TreeParams by value): re-capture when any of them changed since (weight reload, set_math,
    // model_reserve growth, lz_tree_set_params / lz_tree_set_ez / lz_tree_set_tiebreak)
    if (g.exec && (g.gen_model != q->model->generation || g.gen_tree != q->tree->generation)) {
        cudaGraphExecDestroy(g.exec);
        g.exec = nullptr;
    }
    if (!g.exec) {
        g_captures.fetch_add(1, std::memory_order_relaxed);
        g.gen_model = q->model->generation;
        g.gen_tree = q->tree->generation;
        cudaGraph_t graph = nullptr;
        if (!q->capture_stream) LZ_CUDA_CHECK(cudaStreamCreateWithFlags(&q->capture_stream, cudaStreamNonBlocking));
        LZ_CUDA_CHECK(cudaStreamBeginCapture(q->capture_stream, cudaStreamCaptureModeThreadLocal));
        int rc = enqueue_search(q, deterministic, reuse, q->capture_stream);
        cudaError_t e = cudaStreamEndCapture(q->capture_stream, &graph);
        if (rc != LZ_OK) { if (graph) cudaGraphDestroy(graph); return rc; }
        if (e != cudaSuccess) { set_error("cudaStreamEndCapture failed: %s", cudaGetErrorString(e)); return LZ_ECUDA; }
        size_t n = 0;
        LZ_CUDA_CHECK(cudaGraphGetNodes(graph, nullptr, &n));
        g.num_kernels = (int)n;
        e = cudaGraphInstantiate(&g.exec, graph, 0);
        cudaGraphDestroy(graph);
        if (e != cudaSuccess) { set_error("cudaGraphInstantiate failed: %s", cudaGetErrorString(e)); return LZ_ECUDA; }
    }
    LZ_CUDA_CHECK(cudaGraphLaunch(g.exec, s));
    q->num_kernels = g.num_kernels;
    count_launch(g.num_kernels);       // the graph's kernel nodes
    if (lz_gumbel *gs = q->tree->gumbel) {      // the Gumbel graph makes all S descents of the prepared roots and backs each up
        gs->traversals = q->S;
        gs->pending = false;
    }
    return LZ_OK;
}

static int copy_latent_roots(lz_search *q, const float *d_latent_roots, cudaStream_t s)
{
    if (d_latent_roots && d_latent_roots != q->pool)
        LZ_CUDA_CHECK(cudaMemcpyAsync(q->pool, d_latent_roots, q->slot_stride * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return LZ_OK;
}

static int ez_root_hidden(lz_search *q, const float *d_hidden0, const float *d_hidden1, cudaStream_t s)
{
    const size_t bytes = q->hslot_stride * sizeof(float);
    if (d_hidden0) LZ_CUDA_CHECK(cudaMemcpyAsync(q->hpool, d_hidden0, bytes, cudaMemcpyDeviceToDevice, s));
    else LZ_CUDA_CHECK(cudaMemsetAsync(q->hpool, 0, bytes, s));        // efficientzero_model.py:231-236: zeros after initial_inference
    if (d_hidden1) LZ_CUDA_CHECK(cudaMemcpyAsync(q->cpool, d_hidden1, bytes, cudaMemcpyDeviceToDevice, s));
    else LZ_CUDA_CHECK(cudaMemsetAsync(q->cpool, 0, bytes, s));
    return LZ_OK;
}

int lz::search_reuse_buffers(lz_search *q)
{
    if (q->d_true_action) return LZ_OK;
    int rc = dev_alloc(&q->d_true_action, (size_t)q->B);
    if (rc == LZ_OK) rc = dev_alloc(&q->d_reuse_value, (size_t)q->B);
    return rc;
}

// A Gumbel search may not take more simulations than its considered-visit table has (checked before any work is enqueued)
static int gumbel_sims_check(const lz_search *q, const char *fn)
{
    const lz_gumbel *gs = q->tree->gumbel;
    LZ_REQUIRE(!gs || q->S <= gs->g.S, LZ_EINVAL,
               "%s: %d simulations past the considered-visit table of the Gumbel tree's num_simulations = %d", fn, q->S,
               gs ? gs->g.S : 0);
    return LZ_OK;
}

// lz_search_collect*: reset the roots to the legal mask, prepare them from the initial inference's logits (+ noise), then search.
// A Gumbel tree also takes the initial inference's root values d_values (GumbelMuZeroPolicy._forward_collect,
// lzero/policy/gumbel_muzero.py:560-571) and runs the Gumbel search graph.  A stochastic tree runs the stochastic search graph
// (StochasticMuZeroPolicy._forward_collect, lzero/policy/stochastic_muzero.py:578-760); its logits, mask and noise rows are the
// tree's width max(A, C) wide, and the reset bumps the RNG epoch that keys the sampled chance draws of the step.
static int collect_search(lz_search *q, const uint8_t *d_mask, const float *d_logits, const float *d_values, const float *d_noise,
                          float noise_weight, const int32_t *d_to_play, int deterministic, cudaStream_t s)
{
    int rc;
    lz_tree *t = q->tree;
    LZ_REQUIRE((q->d_len != nullptr) == (t->p.nc != 0), LZ_ESTATE,
               "lz_search_collect: the tree's stochastic mode does not match the model (lz_tree_set_stochastic)");
    if ((rc = lz_tree_reset_mask(t, d_mask, s))) return rc;                        // policy/muzero.py:760,769
    const float *values = t->gumbel ? d_values : nullptr;
    if ((rc = lz_tree_prepare(t, d_logits, d_noise, noise_weight, nullptr, values, d_to_play, s))) return rc;   // :774
    if (q->hpool) {      // EfficientZero: zero LSTM state at the roots; the tree has no deterministic argument, the collect call's flag selects its tie-breaking
        if ((rc = ez_root_hidden(q, nullptr, nullptr, s))) return rc;
        if ((rc = lz_tree_set_tiebreak(t, deterministic))) return rc;
    }
    return search_run_graph(q, deterministic, false, s);                                // :775
}

extern "C" {

int lz_search_create(lz_tree *t, lz_model *m, int num_simulations, lz_search **out)
{
    LZ_REQUIRE(t && m && out && num_simulations > 0, LZ_EINVAL, "lz_search_create: bad argument");
    LZ_REQUIRE(m->finalized, LZ_ESTATE, "lz_search_create: model not finalized");
    LZ_REQUIRE(num_simulations <= t->max_sims, LZ_EINVAL, "lz_search_create: num_simulations %d > tree capacity %d", num_simulations, t->max_sims);
    const int C = m->chance;
    LZ_REQUIRE(C == t->p.nc, LZ_EINVAL, "lz_search_create: a Stochastic MuZero model needs a tree in stochastic mode with its "
               "chance_space_size and any other model a tree without chance nodes (lz_tree_set_stochastic; model %d, tree %d)", C, t->p.nc);
    LZ_REQUIRE(t->p.na == m->A && t->p.A == std::max(m->A, C), LZ_EINVAL, "lz_search_create: tree has %d actions (width %d), model %d",
               t->p.na, t->p.A, m->A);
    const bool ez = m->vp;
    LZ_REQUIRE(ez == (t->p.ez != 0), LZ_EINVAL, "lz_search_create: %s model needs a tree in %s mode (lz_tree_set_ez)",
               ez ? "an EfficientZero" : "a MuZero", ez ? "EfficientZero" : "MuZero");
    lz_search *q = new lz_search();
    memset(q, 0, sizeof(*q));
    q->tree = t; q->model = m; q->S = num_simulations; q->B = t->p.B; q->A = t->p.A;
    q->slot_stride = (size_t)q->B * m->latent_floats;
    int rc = dev_alloc(&q->pool, q->slot_stride * (size_t)(q->S + 1));
    if (rc == LZ_OK) rc = dev_alloc(&q->d_ix, (size_t)q->B);
    if (rc == LZ_OK) rc = dev_alloc(&q->d_action, (size_t)q->B);
    if (rc == LZ_OK) rc = dev_alloc(&q->d_reward, (size_t)q->B);
    if (rc == LZ_OK) rc = dev_alloc(&q->d_value, (size_t)q->B);
    if (rc == LZ_OK) rc = dev_alloc(&q->d_policy, (size_t)q->B * q->A);
    if (rc == LZ_OK) rc = dev_alloc(&q->d_root_logits, (size_t)q->B * q->A);
    if (rc == LZ_OK) rc = dev_alloc(&q->d_root_value, (size_t)q->B);
    if (rc == LZ_OK) rc = dev_alloc(&q->d_skip, q->slot_stride);
    if (rc == LZ_OK && C) rc = dev_alloc(&q->d_len, (size_t)q->B);
    if (rc == LZ_OK && ez) {
        q->hslot_stride = (size_t)q->B * m->lstm_hidden;
        rc = dev_alloc(&q->hpool, q->hslot_stride * (size_t)(q->S + 1));
        if (rc == LZ_OK) rc = dev_alloc(&q->cpool, q->hslot_stride * (size_t)(q->S + 1));
        if (rc == LZ_OK) rc = dev_alloc(&q->d_is_reset, (size_t)q->B);
    }
    if (rc == LZ_OK) {      // no stream here: the model's scratch is grown on the setup stream and complete on return
        cudaStream_t ss;
        rc = setup_stream(&ss);
        if (rc == LZ_OK) rc = model_reserve(m, q->B, ss);
        if (rc == LZ_OK) rc = setup_sync();
    }
    if (rc != LZ_OK) { lz_search_destroy(q); return rc; }
    *out = q;
    return LZ_OK;
}

int lz_search_destroy(lz_search *q)
{
    if (!q) return LZ_OK;
    for (SearchGraph &g : q->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
    if (q->capture_stream) cudaStreamDestroy(q->capture_stream);
    if (q->copy_stream) {
        cudaStreamDestroy(q->copy_stream);
        cudaStreamDestroy(q->copy_stream2);
        for (int i = 0; i < 8; ++i) cudaEventDestroy(q->ev_chunk[i]);
        cudaEventDestroy(q->ev_start);
    }
    cudaFree(q->d_obs_stage); cudaFree(q->d_noise_stage); cudaFree(q->d_pre_stage); cudaFree(q->d_mask_stage); cudaFree(q->d_tp_stage);
    cudaFree(q->pool); cudaFree(q->d_ix); cudaFree(q->d_action); cudaFree(q->d_reward); cudaFree(q->d_value);
    cudaFree(q->d_policy); cudaFree(q->d_root_logits); cudaFree(q->d_root_value); cudaFree(q->d_skip);
    cudaFree(q->hpool); cudaFree(q->cpool); cudaFree(q->d_is_reset); cudaFree(q->d_len);
    cudaFree(q->d_true_action); cudaFree(q->d_reuse_value);
    cudaFree(q->rz_latent); cudaFree(q->rz_logits);
    delete q;
    return LZ_OK;
}

int lz_search_run_ez(lz_search *q, const float *d_latent_roots, const float *d_hidden0_roots, const float *d_hidden1_roots, lz_stream s)
{
    LZ_REQUIRE(q && q->hpool, LZ_EINVAL, "lz_search_run_ez: not an EfficientZero search");
    LZ_REQUIRE(!q->tree->gumbel, LZ_ESTATE, "lz_search_run_ez: Gumbel tree, use lz_search_run");
    LZ_REQUIRE(q->tree->prepared, LZ_ESTATE, "lz_search_run_ez: roots not prepared (call lz_tree_prepare first)");
    int rc = copy_latent_roots(q, d_latent_roots, (cudaStream_t)s);
    if (rc == LZ_OK) rc = ez_root_hidden(q, d_hidden0_roots, d_hidden1_roots, (cudaStream_t)s);
    if (rc) return rc;
    return search_run_graph(q, 1, false, (cudaStream_t)s);
}

int lz_search_run_with_reuse(lz_search *q, const float *d_latent_roots, const float *d_hidden0_roots, const float *d_hidden1_roots,
                             const int32_t *d_true_action, const float *d_reuse_value, int32_t *d_infer_count, lz_stream s_)
{
    LZ_REQUIRE(q && d_true_action && d_reuse_value, LZ_EINVAL, "lz_search_run_with_reuse: null argument");
    LZ_REQUIRE(q->hpool || (!d_hidden0_roots && !d_hidden1_roots), LZ_EINVAL,
               "lz_search_run_with_reuse: LSTM state passed to a MuZero search");
    LZ_REQUIRE(q->tree->prepared, LZ_ESTATE, "lz_search_run_with_reuse: roots not prepared (call lz_tree_prepare first)");
    LZ_REQUIRE(!q->tree->gumbel, LZ_ESTATE, "lz_search_run_with_reuse: Gumbel tree (it has no reuse search)");
    LZ_REQUIRE(!q->tree->p.nc, LZ_ESTATE, "lz_search_run_with_reuse: stochastic tree (it has no reuse search)");
    const cudaStream_t s = (cudaStream_t)s_;
    int rc = search_reuse_buffers(q);
    if (rc == LZ_OK) rc = copy_latent_roots(q, d_latent_roots, s);
    if (rc == LZ_OK && q->hpool) rc = ez_root_hidden(q, d_hidden0_roots, d_hidden1_roots, s);
    if (rc) return rc;
    LZ_CUDA_CHECK(cudaMemcpyAsync(q->d_true_action, d_true_action, (size_t)q->B * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
    LZ_CUDA_CHECK(cudaMemcpyAsync(q->d_reuse_value, d_reuse_value, (size_t)q->B * sizeof(float), cudaMemcpyDeviceToDevice, s));
    LZ_CUDA_CHECK(cudaMemsetAsync(q->tree->p.infer_count, 0, (size_t)q->tree->p.N * sizeof(int), s));
    if ((rc = search_run_graph(q, 0, true, s))) return rc;
    if (d_infer_count)      // per simulation: how many trees needed the network (mcts_ctree.py:433,466-467)
        LZ_CUDA_CHECK(cudaMemcpyAsync(d_infer_count, q->tree->p.infer_count, (size_t)q->S * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
    return LZ_OK;
}

int lz_search_run(lz_search *q, const float *d_latent_roots, int deterministic, lz_stream s)
{
    LZ_REQUIRE(q, LZ_EINVAL, "lz_search_run: null search");
    LZ_REQUIRE(!q->hpool, LZ_ESTATE, "lz_search_run: EfficientZero search, use lz_search_run_ez");
    LZ_REQUIRE(q->tree->prepared, LZ_ESTATE, "lz_search_run: roots not prepared (call lz_tree_prepare first)");
    LZ_REQUIRE((q->d_len != nullptr) == (q->tree->p.nc != 0), LZ_ESTATE,
               "lz_search_run: the tree's stochastic mode does not match the model (lz_tree_set_stochastic)");
    if (const lz_gumbel *gs = q->tree->gumbel) {
        LZ_REQUIRE(gs->prepared && gs->traversals == 0, LZ_ESTATE,
                   "lz_search_run: Gumbel roots not freshly prepared (call lz_tree_prepare first)");
        if (int rc = gumbel_sims_check(q, "lz_search_run")) return rc;
    }
    int rc = copy_latent_roots(q, d_latent_roots, (cudaStream_t)s);
    if (rc) return rc;
    return search_run_graph(q, deterministic, false, (cudaStream_t)s);
}

static int collect_device(lz_search *q, const float *d_obs, const uint8_t *d_obs_u8, const uint8_t *d_mask, const float *d_noise,
                          float noise_weight, const int32_t *d_to_play, int deterministic, float *d_pred_value,
                          float *d_policy_logits, lz_stream s)
{
    LZ_REQUIRE(q && (d_obs || d_obs_u8), LZ_EINVAL, "lz_search_collect: bad argument");
    int rc = gumbel_sims_check(q, "lz_search_collect");
    if (rc) return rc;
    TailIO io;
    memset(&io, 0, sizeof(io));
    io.latent2 = q->pool;                                   // latent roots go straight into pool slot 0
    io.policy_logits = d_policy_logits ? d_policy_logits : q->d_root_logits;
    io.value = d_pred_value ? d_pred_value : q->d_root_value;
    io.policy_stride = q->A;                                // the tree's width: max(A, C) on a stochastic tree, else A
    if (d_obs_u8) {
        LZ_REQUIRE(q->model->family == ModelFamily::Conv, LZ_EINVAL, "lz_search_collect_u8: uint8 frames need the conv model");
        if (!q->d_pre_stage && (rc = dev_alloc(&q->d_pre_stage, (size_t)q->B * q->model->latent_floats))) return rc;
        rc = conv_initial_tower(q->model, q->B, nullptr, q->d_pre_stage, (cudaStream_t)s, d_obs_u8);
        if (rc == LZ_OK) rc = conv_initial_tail(q->model, q->B, q->d_pre_stage, io, (cudaStream_t)s);
    } else {
        rc = model_initial(q->model, q->B, d_obs, io, (cudaStream_t)s);          // policy/muzero.py:749
    }
    if (rc) return rc;
    return collect_search(q, d_mask, io.policy_logits, io.value, d_noise, noise_weight, d_to_play, deterministic, (cudaStream_t)s);
}

int lz_search_collect(lz_search *q, const float *d_obs, const uint8_t *d_mask, const float *d_noise, float noise_weight,
                      const int32_t *d_to_play, int deterministic, float *d_pred_value, float *d_policy_logits, lz_stream s)
{
    return collect_device(q, d_obs, nullptr, d_mask, d_noise, noise_weight, d_to_play, deterministic, d_pred_value, d_policy_logits, s);
}

int lz_search_collect_u8(lz_search *q, const uint8_t *d_obs_u8, const uint8_t *d_mask, const float *d_noise, float noise_weight,
                         const int32_t *d_to_play, int deterministic, float *d_pred_value, float *d_policy_logits, lz_stream s)
{
    return collect_device(q, nullptr, d_obs_u8, d_mask, d_noise, noise_weight, d_to_play, deterministic, d_pred_value, d_policy_logits, s);
}

static int collect_host(lz_search *q, const void *h_obs, int obs_u8, const uint8_t *h_mask, const float *h_noise, float noise_weight,
                        const int32_t *h_to_play, int deterministic, int nchunks, float *d_pred_value,
                        float *d_policy_logits, lz_stream s_)
{
    LZ_REQUIRE(q && h_obs, LZ_EINVAL, "lz_search_collect_host: bad argument");
    LZ_REQUIRE(!obs_u8 || q->model->family == ModelFamily::Conv, LZ_EINVAL, "lz_search_collect_host_u8: uint8 frames need the conv model");
    if (int rc = gumbel_sims_check(q, "lz_search_collect_host")) return rc;
    const size_t esz = obs_u8 ? 1 : sizeof(float);         // bytes per observation element on the wire and in the staging buffer
    cudaStream_t s = (cudaStream_t)s_;
    const int B = q->B, A = q->A;
    nchunks = nchunks < 1 ? 1 : (nchunks > 8 ? 8 : nchunks);
    if (!q->copy_stream) {
        q->obs_elems = q->model->obs_elems;
        LZ_CUDA_CHECK(cudaStreamCreateWithFlags(&q->copy_stream, cudaStreamNonBlocking));
        LZ_CUDA_CHECK(cudaStreamCreateWithFlags(&q->copy_stream2, cudaStreamNonBlocking));
        for (int i = 0; i < 8; ++i) LZ_CUDA_CHECK(cudaEventCreateWithFlags(&q->ev_chunk[i], cudaEventDisableTiming));
        LZ_CUDA_CHECK(cudaEventCreateWithFlags(&q->ev_start, cudaEventDisableTiming));
        int rc = dev_alloc(&q->d_obs_stage, q->obs_elems * B);
        if (rc == LZ_OK) rc = dev_alloc(&q->d_noise_stage, (size_t)B * A);
        if (rc == LZ_OK && !q->d_pre_stage) rc = dev_alloc(&q->d_pre_stage, (size_t)B * q->model->latent_floats);
        if (rc == LZ_OK) rc = dev_alloc(&q->d_mask_stage, (size_t)B * A);
        if (rc == LZ_OK) rc = dev_alloc(&q->d_tp_stage, (size_t)B);
        if (rc != LZ_OK) return rc;
    }
    // the copy stream may not overwrite the staging buffer before earlier work on `s` has consumed it
    LZ_CUDA_CHECK(cudaEventRecord(q->ev_start, s));
    LZ_CUDA_CHECK(cudaStreamWaitEvent(q->copy_stream, q->ev_start, 0));
    LZ_CUDA_CHECK(cudaStreamWaitEvent(q->copy_stream2, q->ev_start, 0));
    const int per = (B + nchunks - 1) / nchunks;
    for (int i = 0; i < nchunks; ++i) {
        const int b0 = i * per, bc = std::min(per, B - b0);
        if (bc <= 0) { nchunks = i; break; }
        cudaStream_t cs = (i & 1) ? q->copy_stream2 : q->copy_stream;
        LZ_CUDA_CHECK(cudaMemcpyAsync(reinterpret_cast<unsigned char *>(q->d_obs_stage) + (size_t)b0 * q->obs_elems * esz,
                                      static_cast<const unsigned char *>(h_obs) + (size_t)b0 * q->obs_elems * esz,
                                      (size_t)bc * q->obs_elems * esz, cudaMemcpyHostToDevice, cs));
        LZ_CUDA_CHECK(cudaEventRecord(q->ev_chunk[i], cs));
    }
    if (h_mask) LZ_CUDA_CHECK(cudaMemcpyAsync(q->d_mask_stage, h_mask, (size_t)B * A, cudaMemcpyHostToDevice, s));
    if (h_noise) LZ_CUDA_CHECK(cudaMemcpyAsync(q->d_noise_stage, h_noise, (size_t)B * A * sizeof(float), cudaMemcpyHostToDevice, s));
    if (h_to_play) LZ_CUDA_CHECK(cudaMemcpyAsync(q->d_tp_stage, h_to_play, (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    float *logits = d_policy_logits ? d_policy_logits : q->d_root_logits;
    float *pred = d_pred_value ? d_pred_value : q->d_root_value;
    const bool split = q->model->family == ModelFamily::Conv;   // tower per chunk, tail once
    for (int i = 0; i < nchunks; ++i) {
        const int b0 = i * per, bc = std::min(per, B - b0);
        LZ_CUDA_CHECK(cudaStreamWaitEvent(s, q->ev_chunk[i], 0));
        int rc;
        if (split) {
            const unsigned char *stage = reinterpret_cast<const unsigned char *>(q->d_obs_stage) + (size_t)b0 * q->obs_elems * esz;
            rc = conv_initial_tower(q->model, bc, obs_u8 ? nullptr : reinterpret_cast<const float *>(stage),
                                    q->d_pre_stage + (size_t)b0 * q->model->latent_floats, s, obs_u8 ? stage : nullptr);
        } else {
            TailIO io;
            memset(&io, 0, sizeof(io));
            io.latent2 = q->pool + (size_t)b0 * q->model->latent_floats;
            io.policy_logits = logits + (size_t)b0 * A;     // rows of the tree's width
            io.policy_stride = A;
            io.value = pred + b0;
            rc = model_initial(q->model, bc, q->d_obs_stage + (size_t)b0 * q->obs_elems, io, s);
        }
        if (rc) return rc;
    }
    if (split) {
        TailIO io;
        memset(&io, 0, sizeof(io));
        io.latent2 = q->pool;
        io.policy_logits = logits;
        io.policy_stride = A;
        io.value = pred;
        int rc = conv_initial_tail(q->model, B, q->d_pre_stage, io, s);
        if (rc) return rc;
    }
    return collect_search(q, h_mask ? q->d_mask_stage : nullptr, logits, pred, h_noise ? q->d_noise_stage : nullptr, noise_weight,
                          h_to_play ? q->d_tp_stage : nullptr, deterministic, s);
}

int lz_search_collect_host(lz_search *q, const float *h_obs, const uint8_t *h_mask, const float *h_noise, float noise_weight,
                           const int32_t *h_to_play, int deterministic, int nchunks, float *d_pred_value,
                           float *d_policy_logits, lz_stream s)
{
    return collect_host(q, h_obs, 0, h_mask, h_noise, noise_weight, h_to_play, deterministic, nchunks, d_pred_value, d_policy_logits, s);
}

int lz_search_collect_host_u8(lz_search *q, const uint8_t *h_obs_u8, const uint8_t *h_mask, const float *h_noise, float noise_weight,
                              const int32_t *h_to_play, int deterministic, int nchunks, float *d_pred_value,
                              float *d_policy_logits, lz_stream s)
{
    return collect_host(q, h_obs_u8, 1, h_mask, h_noise, noise_weight, h_to_play, deterministic, nchunks, d_pred_value, d_policy_logits, s);
}

int lz_search_num_kernels(const lz_search *q) { return q ? q->num_kernels : 0; }
unsigned long long lz_debug_graph_captures(void) { return g_captures.load(std::memory_order_relaxed); }

int lz_search_debug_plan(const lz_search *q, int32_t *h_info)
{
    LZ_REQUIRE(q && h_info, LZ_EINVAL, "lz_search_debug_plan: null argument");
    memset(h_info, 0, 8 * sizeof(int32_t));
    h_info[7] = q->tree->p.N;
    if (!persistent_search(q, false)) return LZ_OK;
    h_info[0] = 1;
    tc_describe_search(q->model->conv.tc_rec, persistent_io(q, 1), q->tree->p.N, h_info + 1);
    return LZ_OK;
}
const float *lz_search_latent_pool(const lz_search *q) { return q ? q->pool : nullptr; }
const float *lz_search_hidden_pool(const lz_search *q, int which) { return q ? (which ? q->cpool : q->hpool) : nullptr; }

}  // extern "C"
