// targets.cu -- the replay buffer's reward and value targets (MuZeroGameBuffer._compute_target_reward_value,
// lzero/mcts/buffer/game_buffer_muzero.py:467-575; EfficientZeroGameBuffer, game_buffer_efficientzero.py:167-323) on the device.
//
// The reference runs initial_inference over the N*(K+1) bootstrap observations, copies latents, logits and values to the host,
// and builds the n-step TD targets in nested Python loops; with EfficientZero's use_root_value it first searches those rows and
// bootstraps from the root values.  Here everything is enqueued on the caller's stream with no host synchronisation:
//   initial_inference in mini_infer_size slices (value scalars only; use_root_value: latents and logits into the search)
//   [-> reset + prepare of the T roots -> the search's captured graph -> root values]  -> k_value_targets.
// k_value_targets walks each segment in the reference's order with its float32 / float64 arithmetic spelled out (the NumPy
// promotion rules, DESIGN.md §4.6.2); compiled with -fmad=false so no product is fused into a sum.
#include <string.h>

#include <algorithm>

#include "lz_common.cuh"
#include "search.cuh"

namespace lz {

constexpr int kTargetsBlock = 128;   // one thread per segment

// The reference's accumulation `x += y` of a reward term: float64, or (float32 rewards) a float32 add of the accumulator rounded to
// float32 -- exact after the first add, which turns the Python float into np.float32 (NEP 50: the Python float is weak)
__device__ __forceinline__ double acc_add(double acc, double term, int fp32)
{
    return fp32 ? (double)__fadd_rn(__double2float_rn(acc), __double2float_rn(term)) : __dadd_rn(acc, term);
}

// Segment n, rows n*K1 + k:
//   value = (value_f32 * bootstrap) * value_mask                       (float64 products; -0.0 where a negative value is masked)
//   for i, reward in enumerate(reward_list[pos + k : pos + k + td]):   value += ±reward * discount ** i
//       (float32 rewards: float32 product with the power rounded to float32; the sign compares to_play_list[base_index] with
//       to_play_list[i], i the offset into the window, in two-player mode)
// MuZero: reward target reward_list[pos + k] if pos + k < len(reward_list), else 0.
// EfficientZero: after the window sum, every lstm_horizon_len rows counted across segments (horizon_id == row) the prefix
// restarts at 0.0 and base_index moves to this row; rows inside the segment take the value and prefix += reward_list[pos + k],
// rows past its end take 0 and the running prefix.
__global__ void __launch_bounds__(kTargetsBlock)
k_value_targets(lz_value_tables t, const float *__restrict__ values, double *__restrict__ reward_out, double *__restrict__ value_out)
{
    const int n = blockIdx.x * kTargetsBlock + threadIdx.x;
    if (n >= t.N) return;
    const int K1 = t.K1;
    const double *rw = t.rewards + (size_t)n * t.W;
    const int rlen = t.rlen[n];
    const int seglen = t.value_prefix ? t.seglen[n] : 0;
    const int32_t *tp = t.two_player ? t.to_play + (size_t)n * (t.P + K1) : nullptr;
    const size_t row0 = (size_t)n * K1;
    double prefix = 0.0;
    bool live = false;          // the prefix is an accumulated value (not the Python 0.0 of a reset)
    int chunk0 = 0, base = 0;   // first row of the live prefix; base_index - pos
    for (int k = 0; k < K1; ++k) {
        const size_t r = row0 + k;
        double acc = __dmul_rn(__dmul_rn((double)values[r], t.bootstrap[r]), t.value_mask[r]);
        const int end = min(k + t.td[r], rlen);
        const int tp_base = tp ? tp[t.P + base] : 0;
        for (int i = 0; k + i < end; ++i) {
            const double x = tp && tp[i] != tp_base ? -rw[k + i] : rw[k + i];
            const double term = t.fp32 ? (double)__fmul_rn(__double2float_rn(x), __double2float_rn(t.powers[i]))
                                       : __dmul_rn(x, t.powers[i]);
            acc = acc_add(acc, term, t.fp32);
        }
        if (!t.value_prefix) {
            value_out[r] = acc;
            reward_out[r] = k < rlen ? rw[k] : 0.0;
            continue;
        }
        if (r % (size_t)t.horizon == 0) {
            if (t.alias_prefix && live)
                for (int j = chunk0; j < k; ++j) reward_out[row0 + j] = prefix;
            prefix = 0.0;
            live = false;
            base = k;
        }
        if (k < seglen) {
            value_out[r] = acc;
            prefix = acc_add(prefix, rw[k], t.fp32);
            if (!live) {
                live = true;
                chunk0 = k;
            }
        } else {
            value_out[r] = 0.0;
        }
        reward_out[r] = prefix;
    }
    if (t.alias_prefix && live)
        for (int j = chunk0; j < K1; ++j) reward_out[row0 + j] = prefix;
}

static int check_tables(const char *fn, const lz_value_tables *t, int mini, const float *d_obs, const float *d_values,
                        const double *d_reward_out, const double *d_value_out)
{
    LZ_REQUIRE(t && d_obs && d_values && d_reward_out && d_value_out, LZ_EINVAL, "%s: null argument", fn);
    LZ_REQUIRE(t->N >= 1 && t->K1 >= 1 && t->P >= 1 && t->W == t->K1 - 1 + t->P, LZ_EINVAL,
               "%s: bad table shape N = %d, K1 = %d, P = %d, W = %d (W must be K1 - 1 + P)", fn, t->N, t->K1, t->P, t->W);
    LZ_REQUIRE(t->rewards && t->rlen && t->td && t->bootstrap && t->value_mask && t->powers, LZ_EINVAL, "%s: null table", fn);
    LZ_REQUIRE(!t->value_prefix || (t->seglen && t->horizon >= 1), LZ_EINVAL,
               "%s: value prefixes need the segment lengths and lstm_horizon_len >= 1 (got %d)", fn, t->horizon);
    LZ_REQUIRE(!t->two_player || t->to_play, LZ_EINVAL, "%s: two-player targets need the to_play table", fn);
    LZ_REQUIRE(!t->alias_prefix || t->value_prefix, LZ_EINVAL, "%s: alias_prefix applies to value prefixes only", fn);
    LZ_REQUIRE(mini > 0, LZ_EINVAL, "%s: mini_infer_size %d must be > 0", fn, mini);
    return LZ_OK;
}

static int launch_targets(const lz_value_tables &t, const float *values, double *reward_out, double *value_out, cudaStream_t s)
{
    k_value_targets<<<ceil_div(t.N, kTargetsBlock), kTargetsBlock, 0, s>>>(t, values, reward_out, value_out);
    LZ_KERNEL_CHECK();
    return LZ_OK;
}

}  // namespace lz

using namespace lz;

extern "C" {

int lz_value_targets(lz_model *m, const lz_value_tables *tab, int mini_infer_size, const float *d_obs, float *d_values,
                     double *d_reward_out, double *d_value_out, lz_stream s_)
{
    LZ_REQUIRE(m, LZ_EINVAL, "lz_value_targets: null model");
    LZ_REQUIRE(m->finalized, LZ_ESTATE, "lz_value_targets: model not finalized");
    int rc = check_tables("lz_value_targets", tab, mini_infer_size, d_obs, d_values, d_reward_out, d_value_out);
    if (rc) return rc;
    LZ_REQUIRE((tab->value_prefix != 0) == m->vp, LZ_EINVAL, "lz_value_targets: %s targets need %s model",
               tab->value_prefix ? "value-prefix (EfficientZero)" : "reward (MuZero)", tab->value_prefix ? "an EfficientZero" : "a MuZero");
    const cudaStream_t s = (cudaStream_t)s_;
    const size_t rows = (size_t)tab->N * tab->K1;
    const int slice = (int)std::min<size_t>((size_t)mini_infer_size, rows);
    if ((rc = model_reserve(m, slice, s))) return rc;
    for (size_t beg = 0; beg < rows; beg += (size_t)slice) {      // game_buffer_muzero.py:491-510: the values alone are kept
        TailIO io;
        memset(&io, 0, sizeof(io));
        io.value = d_values + beg;
        if ((rc = model_initial(m, (int)std::min<size_t>((size_t)slice, rows - beg), d_obs + beg * m->obs_elems, io, s))) return rc;
    }
    return launch_targets(*tab, d_values, d_reward_out, d_value_out, s);
}

int lz_value_targets_root(lz_search *q, const lz_value_tables *tab, int mini_infer_size, const float *d_obs, const uint8_t *d_mask,
                          const int32_t *d_to_play, const float *d_noise, float noise_weight, int first_maximum, float *d_values,
                          double *d_reward_out, double *d_value_out, lz_stream s_)
{
    LZ_REQUIRE(q, LZ_EINVAL, "lz_value_targets_root: null search");
    int rc = check_tables("lz_value_targets_root", tab, mini_infer_size, d_obs, d_values, d_reward_out, d_value_out);
    if (rc) return rc;
    lz_tree *t = q->tree;
    lz_model *m = q->model;
    LZ_REQUIRE(q->hpool && tab->value_prefix, LZ_ESTATE,
               "lz_value_targets_root: the root-value search runs EfficientZero searches and value-prefix targets only");
    LZ_REQUIRE(!t->gumbel, LZ_ESTATE, "lz_value_targets_root: Gumbel tree (the root-value search runs EfficientZero trees)");
    const size_t rows = (size_t)tab->N * tab->K1;
    LZ_REQUIRE((size_t)q->B == rows, LZ_EINVAL, "lz_value_targets_root: search of %d roots for %zu rows", q->B, rows);
    const cudaStream_t s = (cudaStream_t)s_;
    // game_buffer_efficientzero.py:192-215: initial_inference in slices, latents straight into the search's pool slot 0
    const int slice = (int)std::min<size_t>((size_t)mini_infer_size, rows);
    if ((rc = model_reserve(m, slice, s))) return rc;
    for (size_t beg = 0; beg < rows; beg += (size_t)slice) {
        TailIO io;
        memset(&io, 0, sizeof(io));
        io.latent = q->pool + beg * m->latent_floats;
        io.policy_logits = q->d_root_logits + beg * q->A;
        if ((rc = model_initial(m, (int)std::min<size_t>((size_t)slice, rows - beg), d_obs + beg * m->obs_elems, io, s))) return rc;
    }
    // :220-239: roots from the legal actions, zero value prefixes, the logits, noise and to_play; the search on zero LSTM state
    if ((rc = lz_tree_reset_mask(t, d_mask, s_))) return rc;
    if ((rc = lz_tree_prepare(t, q->d_root_logits, d_noise, noise_weight, nullptr, d_to_play, s_))) return rc;
    LZ_CUDA_CHECK(cudaMemsetAsync(q->hpool, 0, q->hslot_stride * sizeof(float), s));
    LZ_CUDA_CHECK(cudaMemsetAsync(q->cpool, 0, q->hslot_stride * sizeof(float), s));
    if ((rc = lz_tree_set_tiebreak(t, first_maximum))) return rc;
    if ((rc = search_run_graph(q, 1, false, s))) return rc;
    if ((rc = lz_tree_results(t, nullptr, d_values, nullptr, nullptr, s_))) return rc;     // :240 roots.get_values()
    return launch_targets(*tab, d_values, d_reward_out, d_value_out, s);
}

}  // extern "C"
