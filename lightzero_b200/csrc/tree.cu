// tree.cu -- kernels + C ABI for the device-resident batched MuZero trees (see tree.cuh for the design).
// Compiled with -fmad=false: no fp32 contraction anywhere in this translation unit.
#include <math.h>
#include <stdarg.h>

#include <algorithm>
#include <atomic>
#include <limits.h>
#include <mutex>
#include <vector>

#include "lz_common.cuh"
#include "gumbel.cuh"
#include "tree.cuh"

namespace lz {

static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};
void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// the setup stream of each device (lz_common.cuh), created on first use and kept for the life of the process
int setup_stream(cudaStream_t *s)
{
    static std::mutex mu;
    static cudaStream_t streams[64];
    int dev = 0;
    LZ_CUDA_CHECK(cudaGetDevice(&dev));
    LZ_REQUIRE(dev >= 0 && dev < 64, LZ_ECUDA, "setup stream: device ordinal %d out of range", dev);
    std::lock_guard<std::mutex> lock(mu);
    if (!streams[dev]) LZ_CUDA_CHECK(cudaStreamCreateWithFlags(&streams[dev], cudaStreamNonBlocking));
    *s = streams[dev];
    return LZ_OK;
}

int setup_sync()
{
    cudaStream_t s;
    if (int rc = setup_stream(&s)) return rc;
    LZ_CUDA_CHECK(cudaStreamSynchronize(s));
    return LZ_OK;
}

int setup_memset(void *d, size_t bytes)
{
    cudaStream_t s;
    if (int rc = setup_stream(&s)) return rc;
    LZ_CUDA_CHECK(cudaMemsetAsync(d, 0, bytes, s));
    LZ_CUDA_CHECK(cudaStreamSynchronize(s));
    return LZ_OK;
}

int setup_upload(void *d, const void *h, size_t bytes)
{
    cudaStream_t s;
    if (int rc = setup_stream(&s)) return rc;
    LZ_CUDA_CHECK(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, s));
    LZ_CUDA_CHECK(cudaStreamSynchronize(s));
    return LZ_OK;
}

constexpr int kTreeBlock = 64;   // 2 warps = 2 trees per CTA: latency-bound work, spread over all SMs

__global__ void __launch_bounds__(kTreeBlock)
k_tree_reset(TreeParams p, const int32_t *legal, const int32_t *nlegal, const uint8_t *mask)
{
    const int b = blockIdx.x * (kTreeBlock / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        *p.players_max = INT_MIN;
        *p.rng_epoch += 1ull;
    }
    if (b >= p.B) return;
    const size_t row = (size_t)b * p.A;
    tree_reset_root(p, b, lane, mask ? mask + row : nullptr, (legal && nlegal) ? legal + row : nullptr,
                    (legal && nlegal) ? nlegal[b] : 0);
}

// CRoots::prepare / prepare_no_noise (cnode.cpp:321-358)
__global__ void __launch_bounds__(kTreeBlock)
k_tree_prepare(TreeParams p, const float *logits, const float *noise, float noise_w, const float *rewards,
               const int32_t *to_play)
{
    const int b = blockIdx.x * (kTreeBlock / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= p.B) return;
    const int tp = to_play ? to_play[b] : -1;
    tree_prepare_root(p, b, lane, logits + (size_t)b * p.A, noise ? noise + (size_t)b * p.A : nullptr, noise_w,
                      rewards ? rewards[b] : 0.0f, tp);
    if (lane == 0) atomicMax(p.players_max, tp);
}

// One simulation boundary of every tree: the back-up of the last expansion, then the next descent (see TreeStep).  Fusing
// both into one launch halves the tree launches of a search graph.
template <bool EZ, bool REUSE>
__global__ void __launch_bounds__(kTreeBlock)
k_tree_step(TreeParams p, TreeStep a)
{
    const int b = blockIdx.x * (kTreeBlock / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= p.B) return;
    if (a.latent_index > 0)
        tree_backprop<EZ, REUSE>(p, b, lane, a.latent_index, a.reward[b], a.value[b], a.logits + (size_t)b * p.A, a.to_play,
                                 (EZ && a.leaf_reset) ? a.leaf_reset[b] : 0, REUSE ? a.reuse_value[b] : 0.0f,
                                 (REUSE && a.batch_rank) ? a.batch_rank[b] : -1);
    if (a.traverse) {
        tree_traverse<EZ, REUSE>(p, b, lane, a.deterministic, a.step, a.ix, a.act, a.true_action, a.reuse_value, a.ix_net);
        if (lane == 0) {
            const int len = p.search_len[b];
            // batch_index (cnode.cpp:907-923): recorded on the node the descent ended in (the last path entry), or this tree after a
            // reuse stop on an already expanded child
            if (a.iy)
                a.iy[b] = (REUSE && p.reuse_state[b] != 2) ? p.n_batch[(size_t)b * p.N + p.path_slot[(size_t)b * p.N + len - 1]] : b;
            if (a.len) a.len[b] = len;
            if (a.vtp) a.vtp[b] = p.vtp[b];
            // mcts_ctree.py:856-861 / 1040-1046: the LSTM state of a leaf is reset every lstm_horizon_len steps of depth (per tree)
            if (EZ && a.is_reset) a.is_reset[b] = (len % p.lstm_horizon == 0) ? 1 : 0;
        }
    }
}

// get_distributions / get_values / get_trajectories (cnode.cpp:237-277,369-417)
__global__ void __launch_bounds__(kTreeBlock)
k_tree_results(TreeParams p, int32_t *visits, float *values, int32_t *nlegal, int32_t *traj)
{
    const int b = blockIdx.x * (kTreeBlock / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= p.B) return;
    const int A = p.A, N = p.N;
    const uint32_t *tree_edges = p.edges + (size_t)b * N * kEdgeFields * A;
    const int n = p.nlegal[b];
    if (visits) {
        for (int k = lane; k < A; k += 32)
            visits[(size_t)b * A + k] = k < n ? (int)tree_edges[F_VISIT * A + p.legal[(size_t)b * A + k]] : -1;
    }
    if (lane == 0) {
        if (values) values[b] = tree_root_value(p, b);
        if (nlegal) nlegal[b] = n;
    }
    if (traj) {
        for (int k = lane; k < N; k += 32) traj[(size_t)b * N + k] = -1;
        __syncwarp();
        if (lane == 0) {
            int slot = 0, len = 0;
            while (slot >= 0 && len < N) {
                int a = p.n_best[(size_t)b * N + slot];
                if (a < 0) break;
                traj[(size_t)b * N + len++] = a;
                slot = (int)tree_edges[(size_t)slot * kEdgeFields * A + F_CSLOT * A + a];
            }
        }
    }
}

// select_action (lzero/policy/utils.py:637-661) on the root visit counts of every tree: probabilities
// visit ** (1 / temperature) / sum in fp64 like the reference's Python floats, entropy in bits = -sum p ln p / ln 2 (scipy.stats.entropy(p, base=2), policy/utils.py:660),
// action = arg-max (deterministic, first maximum like np.argmax) or an inverse-CDF draw from a counter-based uniform.
__global__ void __launch_bounds__(kTreeBlock)
k_tree_select_action(TreeParams p, double inv_temperature, int deterministic, unsigned long long seed,
                     int32_t *action, int32_t *action_pos, float *entropy)
{
    const int b = blockIdx.x * (kTreeBlock / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= p.B) return;
    const int A = p.A, n = p.nlegal[b];
    const uint32_t *nb = p.edges + (size_t)b * p.N * kEdgeFields * A;      // root block
    const int *lg = p.legal + (size_t)b * A;
    double total;
    const double ent = root_visit_entropy(nb, lg, A, n, inv_temperature, lane, &total);
    if (lane == 0) {
        int pos = 0;
        if (deterministic) {
            int best = -1;
            for (int k = 0; k < n; ++k) { int v = (int)nb[F_VISIT * A + lg[k]]; if (v > best) { best = v; pos = k; } }
        } else {
            const unsigned long long h = mix64(seed ^ mix64((unsigned long long)b + 0x1234567ull));
            const double u = (double)(h >> 11) * (1.0 / 9007199254740992.0);       // uniform [0, 1)
            double cum = 0.0;
            pos = n - 1;
            for (int k = 0; k < n; ++k) {
                cum += pow((double)(int)nb[F_VISIT * A + lg[k]], inv_temperature) / total;
                if (u < cum) { pos = k; break; }
            }
        }
        if (action_pos) action_pos[b] = pos;
        if (action) action[b] = lg[pos];            // np.where(action_mask == 1)[0][pos], policy/muzero.py:800
        if (entropy) entropy[b] = (float)(ent / 0.69314718055994530942);    // base 2, as scipy divides the natural-log entropy by ln 2
    }
}

static inline dim3 tree_grid(int B) { return dim3(ceil_div(B, kTreeBlock / 32)); }

int tree_launch_step(lz_tree *t, const TreeStep &a_in, cudaStream_t s)
{
    if (t->gumbel) return gumbel_step(t, a_in, s);      // takes no step of the RNG counter
    TreeStep a = a_in;
    const bool reuse = a.reuse_value != nullptr;
    if (a.traverse) {
        if (t->p.ez || reuse) a.deterministic = t->p.tie_first;
        a.step = t->step_counter++;
    }
    const dim3 grid = tree_grid(t->p.B);
    if (t->p.ez) {
        if (reuse) k_tree_step<true, true><<<grid, kTreeBlock, 0, s>>>(t->p, a);
        else k_tree_step<true, false><<<grid, kTreeBlock, 0, s>>>(t->p, a);
    } else {
        if (reuse) k_tree_step<false, true><<<grid, kTreeBlock, 0, s>>>(t->p, a);
        else k_tree_step<false, false><<<grid, kTreeBlock, 0, s>>>(t->p, a);
    }
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

}  // namespace lz

using namespace lz;

extern "C" {

int lz_version(void) { return 200; }
unsigned long long lz_debug_launch_count(void) { return lz::g_launches.load(std::memory_order_relaxed); }
const char *lz_last_error(void) { return lz::g_err; }

int lz_tree_create(int B, int A, int max_sims, lz_tree **out)
{
    LZ_REQUIRE(out && B > 0 && A > 0 && max_sims > 0, LZ_EINVAL, "lz_tree_create: bad arguments B=%d A=%d max_sims=%d", B, A, max_sims);
    int ndev = 0;
    LZ_CUDA_CHECK(cudaGetDeviceCount(&ndev));
    LZ_REQUIRE(ndev > 0, LZ_ECUDA, "lz_tree_create: no CUDA device (this library has no CPU fallback)");
    lz_tree *t = new lz_tree();
    memset(t, 0, sizeof(*t));
    const int N = max_sims + 1;
    TreeParams &p = t->p;
    p.B = B; p.A = A; p.N = N;
    t->max_sims = max_sims;
    // one allocation, carved
    size_t words = 0;
    auto take = [&](size_t n) { size_t o = words; words += (n + 31) & ~(size_t)31; return o; };
    size_t o_edges = take((size_t)B * N * kEdgeFields * A);
    size_t o_ntp = take((size_t)B * N), o_nbest = take((size_t)B * N), o_nreset = take((size_t)B * N), o_nbatch = take((size_t)B * N);
    size_t o_rstate = take(B), o_infer = take(N);
    size_t o_legal = take((size_t)B * A), o_nlegal = take(B);
    size_t o_rvis = take(B), o_rvsum = take(B), o_rrew = take(B), o_mmax = take(B), o_mmin = take(B);
    size_t o_tp = take(B), o_players = take(1), o_pslot = take((size_t)B * N), o_pact = take((size_t)B * N);
    size_t o_plen = take(B), o_vtp = take(B), o_slen = take(B), o_pbc = take(N + 1), o_epoch = take(2);
    uint32_t *base = nullptr;
    int rc = dev_alloc(&base, words);
    if (rc != LZ_OK) { delete t; return rc; }
    if ((rc = setup_memset(base, words * 4)) != LZ_OK) { cudaFree(base); delete t; return rc; }
    t->alloc_base = base;
    p.edges = base + o_edges;
    p.n_to_play = (int *)(base + o_ntp); p.n_best = (int *)(base + o_nbest); p.n_reset = (int *)(base + o_nreset);
    p.n_batch = (int *)(base + o_nbatch); p.reuse_state = (int *)(base + o_rstate); p.infer_count = (int *)(base + o_infer);
    p.ez = 0; p.lstm_horizon = 5; p.tie_first = 1;
    p.na = A; p.nc = 0; p.chance_u = -1.0;
    p.legal = (int *)(base + o_legal); p.nlegal = (int *)(base + o_nlegal);
    p.root_visit = (int *)(base + o_rvis); p.root_vsum = (float *)(base + o_rvsum); p.root_reward = (float *)(base + o_rrew);
    p.mm_max = (float *)(base + o_mmax); p.mm_min = (float *)(base + o_mmin);
    p.to_play = (int *)(base + o_tp); p.players_max = (int *)(base + o_players);
    p.path_slot = (int *)(base + o_pslot); p.path_action = (int *)(base + o_pact); p.path_len = (int *)(base + o_plen);
    p.vtp = (int *)(base + o_vtp); p.search_len = (int *)(base + o_slen);
    t->d_pbc = (float *)(base + o_pbc); p.pbc = t->d_pbc;
    p.rng_epoch = (unsigned long long *)(base + o_epoch);
    p.rng_seed = 0x5eed5eedull;
    *out = t;
    return lz_tree_set_params(t, 19652, 1.25f, 0.997f, 0.01f);
}

int lz_tree_destroy(lz_tree *t)
{
    if (!t) return LZ_OK;
    gumbel_free(t);
    cudaFree(t->alloc_base);
    delete t;
    return LZ_OK;
}

int lz_tree_set_params(lz_tree *t, int pb_c_base, float pb_c_init, float discount, float value_delta_max)
{
    LZ_REQUIRE(t, LZ_EINVAL, "lz_tree_set_params: null tree");
    LZ_REQUIRE(pb_c_base > 0, LZ_EINVAL, "lz_tree_set_params: pb_c_base must be > 0");
    // cucb_score (cnode.cpp:672): pb_c = log((N + base + 1) / base) + init, all fp32, N = visit_count - 1.
    // The argument only depends on the integer visit count, so the S+2 possible values are tabulated
    // once on the host with the same libm logf the reference binary links against.
    const int n = t->p.N + 1;
    std::vector<float> tab(n);
    const float base = (float)pb_c_base;
    for (int i = 0; i < n; ++i) {
        volatile float num = (float)i + base;
        num = num + 1;
        volatile float arg = num / base;
        volatile float lg = logf(arg);
        tab[i] = lg + pb_c_init;
    }
    if (int rc = setup_upload(t->d_pbc, tab.data(), n * sizeof(float))) return rc;
    if (t->p.discount != discount || t->p.delta != value_delta_max) ++t->generation;   // passed BY VALUE into captured search graphs
    t->p.discount = discount;
    t->p.delta = value_delta_max;
    t->params_set = true;
    return LZ_OK;
}

int lz_tree_reset(lz_tree *t, const int32_t *d_legal, const int32_t *d_nlegal, lz_stream s)
{
    LZ_REQUIRE(t, LZ_EINVAL, "lz_tree_reset: null tree");
    LZ_REQUIRE((d_legal == nullptr) == (d_nlegal == nullptr), LZ_EINVAL, "lz_tree_reset: pass both d_legal and d_nlegal or neither");
    k_tree_reset<<<tree_grid(t->p.B), kTreeBlock, 0, (cudaStream_t)s>>>(t->p, d_legal, d_nlegal, nullptr);
    LZ_KERNEL_CHECK();
    t->prepared = false;
    if (t->gumbel) t->gumbel->prepared = false;
    return LZ_OK;
}

int lz_tree_reset_mask(lz_tree *t, const uint8_t *d_mask, lz_stream s)
{
    LZ_REQUIRE(t, LZ_EINVAL, "lz_tree_reset_mask: null tree");
    k_tree_reset<<<tree_grid(t->p.B), kTreeBlock, 0, (cudaStream_t)s>>>(t->p, nullptr, nullptr, d_mask);
    LZ_KERNEL_CHECK();
    t->prepared = false;
    if (t->gumbel) t->gumbel->prepared = false;
    return LZ_OK;
}

int lz_tree_prepare(lz_tree *t, const float *d_logits, const float *d_noise, float noise_weight, const float *d_rewards,
                    const float *d_values, const int32_t *d_to_play, lz_stream s)
{
    LZ_REQUIRE(t && d_logits, LZ_EINVAL, "lz_tree_prepare: null argument");
    LZ_REQUIRE(!t->gumbel == !d_values, LZ_EINVAL, t->gumbel ? "lz_tree_prepare: a Gumbel tree needs the root values d_values"
                                                             : "lz_tree_prepare: d_values is for Gumbel trees only (lz_tree_set_gumbel)");
    k_tree_prepare<<<tree_grid(t->p.B), kTreeBlock, 0, (cudaStream_t)s>>>(t->p, d_logits, d_noise, noise_weight,
                                                                         d_rewards, d_to_play);
    LZ_KERNEL_CHECK();
    t->prepared = true;
    return t->gumbel ? gumbel_prepare(t, d_values, (cudaStream_t)s) : LZ_OK;
}

int lz_tree_traverse(lz_tree *t, int deterministic, const int32_t *d_true_action, const float *d_reuse_value, int32_t *d_ix,
                     int32_t *d_iy, int32_t *d_last_action, int32_t *d_search_len, int32_t *d_virtual_to_play, int32_t *d_is_reset,
                     lz_stream s)
{
    LZ_REQUIRE(t, LZ_EINVAL, "lz_tree_traverse: null tree");
    LZ_REQUIRE(!d_true_action == !d_reuse_value, LZ_EINVAL, "lz_tree_traverse: pass both d_true_action and d_reuse_value or neither");
    LZ_REQUIRE(!d_is_reset || t->p.ez, LZ_EINVAL, "lz_tree_traverse: d_is_reset is an output of EfficientZero trees only");
    LZ_REQUIRE(t->prepared, LZ_ESTATE, "lz_tree_traverse: roots not prepared (call lz_tree_prepare first)");
    LZ_REQUIRE(!t->gumbel || !d_reuse_value, LZ_ESTATE, "lz_tree_traverse: Gumbel tree (it has no reuse descent)");
    LZ_REQUIRE(!t->p.nc || !d_reuse_value, LZ_ESTATE, "lz_tree_traverse: stochastic tree (it has no reuse descent)");
    TreeStep a = {};
    a.traverse = 1; a.deterministic = deterministic; a.true_action = d_true_action; a.reuse_value = d_reuse_value;
    a.ix = d_ix; a.iy = d_iy; a.act = d_last_action; a.len = d_search_len; a.vtp = d_virtual_to_play; a.is_reset = d_is_reset;
    return tree_launch_step(t, a, (cudaStream_t)s);
}

int lz_tree_backpropagate(lz_tree *t, int latent_index, const float *d_reward, const float *d_value, const float *d_logits,
                          const float *d_reuse_value, const int32_t *d_batch_rank, const int32_t *d_is_reset,
                          const int32_t *d_to_play, lz_stream s)
{
    LZ_REQUIRE(t && d_reward && d_value && d_logits, LZ_EINVAL, "lz_tree_backpropagate: null argument");
    LZ_REQUIRE(!d_batch_rank || d_reuse_value, LZ_EINVAL, "lz_tree_backpropagate: d_batch_rank needs d_reuse_value");
    LZ_REQUIRE(!t->p.ez == !d_is_reset, LZ_EINVAL, t->p.ez ? "lz_tree_backpropagate: EfficientZero trees need d_is_reset"
                                                          : "lz_tree_backpropagate: d_is_reset is for EfficientZero trees only");
    LZ_REQUIRE(t->prepared, LZ_ESTATE, "lz_tree_backpropagate: roots not prepared");
    LZ_REQUIRE(!t->gumbel || !d_reuse_value, LZ_ESTATE, "lz_tree_backpropagate: Gumbel tree (it has no reuse back-up)");
    LZ_REQUIRE(!t->p.nc || !d_reuse_value, LZ_ESTATE, "lz_tree_backpropagate: stochastic tree (it has no reuse back-up)");
    LZ_REQUIRE(latent_index >= 1 && latent_index <= t->max_sims, LZ_EINVAL,
               "lz_tree_backpropagate: latent_index %d outside [1, %d]", latent_index, t->max_sims);
    TreeStep a = {};
    a.latent_index = latent_index; a.reward = d_reward; a.value = d_value; a.logits = d_logits; a.to_play = d_to_play;
    a.leaf_reset = d_is_reset; a.batch_rank = d_batch_rank; a.reuse_value = d_reuse_value;
    return tree_launch_step(t, a, (cudaStream_t)s);
}

int lz_tree_set_ez(lz_tree *t, int efficientzero, int lstm_horizon_len)
{
    LZ_REQUIRE(t, LZ_EINVAL, "lz_tree_set_ez: null tree");
    LZ_REQUIRE(!efficientzero || lstm_horizon_len > 0, LZ_EINVAL, "lz_tree_set_ez: lstm_horizon_len must be > 0 (mcts_ctree.py:857)");
    LZ_REQUIRE(!efficientzero || !t->gumbel, LZ_ESTATE, "lz_tree_set_ez: Gumbel tree (lz_tree_set_gumbel(t, m, 0) turns it back into a MuZero tree)");
    LZ_REQUIRE(!efficientzero || !t->p.nc, LZ_ESTATE, "lz_tree_set_ez: stochastic tree (lz_tree_set_stochastic(t, A, 0, -1) turns it back into a MuZero tree)");
    const int ez = efficientzero ? 1 : 0, hor = efficientzero ? lstm_horizon_len : t->p.lstm_horizon;
    if (t->p.ez != ez || t->p.lstm_horizon != hor) ++t->generation;
    t->p.ez = ez;
    t->p.lstm_horizon = hor;
    return LZ_OK;
}

int lz_tree_set_stochastic(lz_tree *t, int action_space_size, int chance_space_size, double chance_u)
{
    LZ_REQUIRE(t, LZ_EINVAL, "lz_tree_set_stochastic: null tree");
    TreeParams &p = t->p;
    int na = p.A, nc = 0;
    double u = -1.0;
    if (chance_space_size) {
        LZ_REQUIRE(!p.ez && !t->gumbel, LZ_ESTATE, "lz_tree_set_stochastic: EfficientZero or Gumbel tree");
        LZ_REQUIRE(action_space_size >= 1 && chance_space_size >= 1 && std::max(action_space_size, chance_space_size) == p.A, LZ_EINVAL,
                   "lz_tree_set_stochastic: a tree of width %d takes max(action_space_size, chance_space_size) == %d (got %d, %d)",
                   p.A, p.A, action_space_size, chance_space_size);
        LZ_REQUIRE(chance_u < 1.0, LZ_EINVAL, "lz_tree_set_stochastic: chance_u %g must be < 1 (or < 0 to sample)", chance_u);
        na = action_space_size;
        nc = chance_space_size;
        u = chance_u < 0.0 ? -1.0 : chance_u;
    }
    if (p.na != na || p.nc != nc || p.chance_u != u) ++t->generation;      // captured graphs bake TreeParams in
    p.na = na;
    p.nc = nc;
    p.chance_u = u;
    return LZ_OK;
}

int lz_tree_set_tiebreak(lz_tree *t, int first_maximum)
{
    LZ_REQUIRE(t, LZ_EINVAL, "lz_tree_set_tiebreak: null tree");
    const int v = first_maximum ? 1 : 0;
    if (t->p.tie_first != v) ++t->generation;       // captured graphs bake TreeParams in
    t->p.tie_first = v;
    return LZ_OK;
}

int lz_tree_select_action(lz_tree *t, float temperature, int deterministic, uint64_t seed, int32_t *d_action,
                          int32_t *d_action_pos, float *d_entropy, lz_stream s)
{
    LZ_REQUIRE(t && temperature > 0.0f, LZ_EINVAL, "lz_tree_select_action: bad argument (temperature must be > 0)");
    k_tree_select_action<<<tree_grid(t->p.B), kTreeBlock, 0, (cudaStream_t)s>>>(t->p, 1.0 / (double)temperature, deterministic,
                                                                               (unsigned long long)seed, d_action, d_action_pos, d_entropy);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

int lz_tree_debug_rng(lz_tree *t, uint64_t *h_seed, uint64_t *h_epoch, uint32_t *h_step_counter)
{
    LZ_REQUIRE(t && h_seed && h_epoch && h_step_counter, LZ_EINVAL, "lz_tree_debug_rng: null argument");
    LZ_CUDA_CHECK(cudaDeviceSynchronize());      // the epoch is bumped on the device by every reset
    unsigned long long epoch = 0;
    LZ_CUDA_CHECK(cudaMemcpy(&epoch, t->p.rng_epoch, sizeof(epoch), cudaMemcpyDeviceToHost));
    *h_seed = t->p.rng_seed;
    *h_epoch = epoch;
    *h_step_counter = t->step_counter;
    return LZ_OK;
}

int lz_tree_results(lz_tree *t, int32_t *d_visits, float *d_values, int32_t *d_nlegal, int32_t *d_traj, lz_stream s)
{
    LZ_REQUIRE(t, LZ_EINVAL, "lz_tree_results: null tree");
    k_tree_results<<<tree_grid(t->p.B), kTreeBlock, 0, (cudaStream_t)s>>>(t->p, d_visits, d_values, d_nlegal, d_traj);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

}  // extern "C"
