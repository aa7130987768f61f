/*
 * lzb200.h -- C ABI of the H100-native batched MuZero MCTS + inference engine.
 *
 * This is the drop-in boundary for ONE hot path of opendilab/LightZero (file:line relative to the
 * reference repository root):
 *
 *   lzero/mcts/ctree/ctree_muzero/mz_tree.pyx:5-107   (the Cython surface: Roots, MinMaxStatsList,
 *        ResultsWrapper, batch_traverse, batch_backpropagate)  -> lz_tree_*
 *   lzero/mcts/ctree/ctree_muzero/lib/cnode.cpp:83-147,169-203,301-358,387-500,551-595,654-698,754-825
 *        (expand / compute_mean_q / prepare / results / backpropagate / select / ucb / traverse)
 *   lzero/mcts/ctree/common_lib/cminimax.cpp:7-66      (MinMaxStats)          -> folded into lz_tree
 *   lzero/model/muzero_model.py:210-272                (initial/recurrent_inference) -> lz_model_*
 *   lzero/policy/scaling_transform.py:64-92            (InverseScalarTransform) -> fused in lz_model_*
 *   lzero/mcts/tree_search/mcts_ctree.py:267-368       (MuZeroMCTSCtree.search loop) -> lz_search_*
 *   lzero/policy/muzero.py:749-779                     (_forward_collect inner part) -> lz_search_collect
 *
 * Conventions
 *   - every function returns 0 on success or a negative LZ_E* code; lz_last_error() gives the
 *     message of the last failure on the calling thread.  No C++ exception crosses this boundary.
 *   - pointers named d_* are DEVICE pointers, h_* are HOST pointers.  Plain pointers and sizes only.
 *   - every compute call takes the cudaStream_t (passed as void*) it is enqueued on and performs
 *     NO host<->device synchronisation; results are valid once the stream reaches that point.
 *   - a handle must be used from one stream at a time (thread-compatible, no global state).
 *   - there is no CPU fallback: without a CUDA device every create call fails with LZ_ECUDA.
 *   - tie-breaking: `deterministic != 0` picks the first legal action attaining the exact maximum
 *     (cnode.cpp:592 front()); 0 draws uniformly among the reference's epsilon-tie list with a
 *     counter-based device RNG (the reference reseeds rand() from the wall clock, cnode.cpp:770).
 */
#ifndef LZB200_H
#define LZB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LZ_OK 0
#define LZ_EINVAL (-1)   /* bad argument */
#define LZ_ECUDA (-2)    /* CUDA runtime error (message has the cudaError string) */
#define LZ_ESTATE (-3)   /* call order violated (e.g. search before prepare) */
#define LZ_ENOMEM (-4)

typedef struct lz_tree lz_tree;
typedef struct lz_model lz_model;
typedef struct lz_search lz_search;
typedef struct lz_frames lz_frames;       /* device-resident observation frame stacks of B environments */
typedef struct lz_segments lz_segments;   /* device-resident search statistics of B game segments */
typedef void *lz_stream;   /* cudaStream_t */

int lz_version(void);
/* Launch accounting: kernels this library has enqueued since load (kernel nodes of launched graphs included). */
unsigned long long lz_debug_launch_count(void);
const char *lz_last_error(void);

/* ------------------------------------------------------------------ tree (mz_tree / cnode.cpp) */

/* B trees, A actions, room for max_sims expansions per tree (node slot k == latent index k). */
int lz_tree_create(int B, int A, int max_sims, lz_tree **out);
int lz_tree_destroy(lz_tree *t);

/* Search constants (mcts_ctree.py:286,292): PUCT constants, discount, MinMax value_delta_max.
 * Precomputes the per-visit-count exploration table on the host with libm logf (cnode.cpp:672). */
int lz_tree_set_params(lz_tree *t, int pb_c_base, float pb_c_init, float discount, float value_delta_max);

/* CRoots::CRoots (cnode.cpp:301-317).  d_legal: int32 [B,A] legal action ids in the caller's order,
 * -1 padded; d_nlegal: int32 [B] (0 == all actions, cnode.cpp:101-107).  Both NULL == all legal.
 * Also resets MinMax stats (a fresh MinMaxStatsList per search, mcts_ctree.py:291-292). */
int lz_tree_reset(lz_tree *t, const int32_t *d_legal, const int32_t *d_nlegal, lz_stream s);
/* Same from a mask uint8 [B,A] (legal ids ascending == np.nonzero order, policy/muzero.py:760). */
int lz_tree_reset_mask(lz_tree *t, const uint8_t *d_mask, lz_stream s);

/* CRoots::prepare / prepare_no_noise (cnode.cpp:321-358).  d_logits f32 [B,A] by action id;
 * d_noise f32 [B,A] rows in LEGAL ORDER (first nlegal[b] used) or NULL for prepare_no_noise;
 * d_rewards f32 [B] or NULL (zeros); d_to_play int32 [B] (-1 == single player).
 * d_values f32 [B]: the roots' value estimates, required on a Gumbel tree (ctree_gumbel_muzero cnode.cpp:418-455; it also
 * starts a fresh round of at most num_simulations descents) and NULL on any other tree (LZ_EINVAL otherwise). */
int lz_tree_prepare(lz_tree *t, const float *d_logits, const float *d_noise, float noise_weight,
                    const float *d_rewards, const float *d_values, const int32_t *d_to_play, lz_stream s);

/* cbatch_traverse: one descent per tree, the one of the tree's mode.  Outputs (each int32 [B], may be NULL): latent-pool slot
 * of the leaf's parent (== its current_latent_state_index), batch index (== tree index), last action, search length, virtual
 * to_play after the descent.
 *   MuZero tree (cnode.cpp:754-825): PUCT; ties by `deterministic`.
 *   EfficientZero tree (ctree_efficientzero cnode.cpp:876-958): ties by lz_tree_set_tiebreak; d_is_reset int32 [B] out (may be
 *     NULL; only EfficientZero trees take it, LZ_EINVAL otherwise) = (search_len % lstm_horizon_len == 0).
 *   Reuse descent (ReZero search_with_reuse, cnode.cpp:597-652, 701-752, 828-932; EfficientZero :699-754, 960-1072), selected
 *     by a non-NULL d_true_action int32 [B] / d_reuse_value f32 [B] pair (both or neither, LZ_EINVAL otherwise): the action
 *     taken in the stored trajectory and the value to reuse for it.  The root scores that child with carm_score and the
 *     descent stops right after the root when it is selected.  d_ix reports -1 for trees that stopped on an already expanded
 *     child ("no inference"); d_iy is the batch_index recorded when the parent was expanded (the compact inference row).  Ties
 *     by lz_tree_set_tiebreak.
 *   Gumbel tree (ctree_gumbel_muzero cnode.cpp:834-897): sequential halving at the root; `deterministic` is ignored, the virtual
 *     to_play is the root's, unchanged.  No reuse descent (LZ_ESTATE); at most num_simulations descents per prepare (one more
 *     would index past the considered-visit table): LZ_ESTATE. */
int lz_tree_traverse(lz_tree *t, int deterministic, const int32_t *d_true_action, const float *d_reuse_value, int32_t *d_ix,
                     int32_t *d_iy, int32_t *d_last_action, int32_t *d_search_len, int32_t *d_virtual_to_play, int32_t *d_is_reset,
                     lz_stream s);

/* cbatch_backpropagate: expand the leaves found by the last traverse into slot `latent_index` (simulation_index + 1) and back
 * up, the back-up of the tree's mode.  d_reward/d_value f32 [B] (scalars, after the inverse transform), d_logits f32 [B,A];
 * d_to_play int32 [B] or NULL (use the virtual to_play the last traverse produced, which is what mcts_ctree.py:365-368 passes).
 *   MuZero tree (cnode.cpp:480-500).
 *   EfficientZero tree (ctree_efficientzero cnode.cpp:577-601): d_reward carries the value prefixes; d_is_reset int32 [B]
 *     (is_reset_list) is required.  Any other tree takes d_is_reset == NULL (LZ_EINVAL otherwise).
 *   Reuse back-up (cbatch_backpropagate_with_reuse, cnode.cpp:502-549; EfficientZero :603-650), selected by a non-NULL
 *     d_reuse_value f32 [B]: rows are indexed BY TREE (not compacted; rows of "no inference" trees are ignored).  d_batch_rank
 *     int32 [B] or NULL, only with d_reuse_value (LZ_EINVAL otherwise): compact row of each tree in the caller's inference
 *     batch, stored as the batch_index of the node it expands.  Which trees skip the expansion / back up the reuse value is
 *     the state the last traverse left.
 *   Gumbel tree (ctree_gumbel_muzero cnode.cpp:633-652): the one-player back-up for every to_play; d_value is also the new
 *     node's raw value.  It must follow a descent, and there is no reuse back-up (LZ_ESTATE). */
int lz_tree_backpropagate(lz_tree *t, int latent_index, const float *d_reward, const float *d_value, const float *d_logits,
                          const float *d_reuse_value, const int32_t *d_batch_rank, const int32_t *d_is_reset,
                          const int32_t *d_to_play, lz_stream s);

/* ---- EfficientZero tree (lzero/mcts/ctree/ctree_efficientzero/lib/cnode.cpp, ez_tree.pyx) ----
 * lz_tree_set_ez switches a tree to value-prefix semantics before lz_tree_prepare: the reward slot carries the child's
 * value prefix, every expanded node carries is_reset, the reward of a step is the prefix difference unless the parent
 * was reset (cnode.cpp:185-195, 496-573, 786-790).  lstm_horizon_len (mcts_ctree.py:857) is used by the fused search
 * and by lz_tree_traverse to derive is_reset = (search_len % lstm_horizon_len == 0).
 * The reference tie-break is rand() % len(ties) with no deterministic switch (cnode.cpp:691); these trees use the rule of
 * lz_tree_set_tiebreak, by default the first maximum, which is that draw with rand() == 0 (how the parity oracle builds the
 * reference). */
int lz_tree_set_ez(lz_tree *t, int efficientzero, int lstm_horizon_len);
/* ---- Stochastic MuZero tree (lzero/mcts/ctree/ctree_stochastic_muzero/lib/cnode.cpp, stochastic_mz_tree.pyx) ----
 * lz_tree_set_stochastic puts a MuZero tree in stochastic mode before lz_tree_prepare: the root is a decision node, the children
 * of a decision node are chance nodes and those of a chance node decision nodes (cnode.cpp:96-165), so a node is a chance node
 * exactly when its depth is odd.  The tree must have been created with A = max(action_space_size, chance_space_size): every
 * logits, noise, mask, legal and visit row of the tree has that width.  An inner decision node has action_space_size children,
 * a chance node chance_space_size, and a chance node's reward is 0.  A chance node's child is drawn as
 * std::discrete_distribution(priors) (cnode.cpp:610-630, libstdc++'s arithmetic in double) at a uniform u: every selection
 * uses chance_u when it is in [0, 1) (the reference's draw from std::mt19937(s) when std::random_device returns s), and a fresh
 * u from the counter-based RNG of the tie draws (seed, epoch, step, depth) when chance_u < 0.  Decision nodes select as a
 * MuZero tree (lz_tree_traverse's deterministic flag).  The traverse's d_search_len is the leaf's depth: the leaf is a chance
 * node (leaf_node_is_chance) when it is odd.  lz_tree_backpropagate takes, per tree, the afterstate program's chance logits
 * (the first chance_space_size entries of the row) for a chance leaf and the dynamics program's action logits otherwise.
 * chance_space_size = 0 turns the tree back into a MuZero tree (the other arguments are then ignored).  Refused on EfficientZero
 * and Gumbel trees (LZ_ESTATE); the reuse descent, back-up and search (lz_search_run_with_reuse) are refused on a stochastic
 * tree. */
int lz_tree_set_stochastic(lz_tree *t, int action_space_size, int chance_space_size, double chance_u);
/* Tie-breaking of the EfficientZero and reuse descents, which have no deterministic switch in the reference (they draw
 * rand() % len(ties) after reseeding from the wall clock, ctree_efficientzero/lib/cnode.cpp:691, ctree_muzero cnode.cpp:610-640):
 * first_maximum = 1 (default; the reference's draw with rand() == 0, what the parity tests pin) or 0 = a uniform draw from the same tie
 * list with the counter-based device RNG of the MuZero lz_tree_traverse(deterministic = 0). */
int lz_tree_set_tiebreak(lz_tree *t, int first_maximum);
/* get_distributions / get_values / get_trajectories (cnode.cpp:237-277,369-417).
 * d_visits int32 [B,A] in legal order, -1 padded; d_values f32 [B]; d_nlegal int32 [B];
 * d_traj int32 [B, max_sims+1] -1 padded.  Any pointer may be NULL. */
int lz_tree_results(lz_tree *t, int32_t *d_visits, float *d_values, int32_t *d_nlegal,
                    int32_t *d_traj, lz_stream s);
/* Test hook: the key of the tree's tie-break draws, hash(seed, epoch, tree, step, depth) (tree.cuh).  h_epoch is the
 * epoch the next descent uses (every reset advances it; it lives in device memory, so this synchronises the device and
 * copies it); h_step_counter is the step the next step-wise descent takes (each one consumes a step; a fused search
 * uses steps 0 ... num_simulations - 1). */
int lz_tree_debug_rng(lz_tree *t, uint64_t *h_seed, uint64_t *h_epoch, uint32_t *h_step_counter);

/* select_action (lzero/policy/utils.py:637-661) on the device, from the root visit counts of the finished search:
 * p = visit ** (1 / temperature) / sum (fp64), d_entropy = -sum p log2 p (scipy.stats.entropy(p, base=2)), d_action_pos = arg-max (deterministic != 0; the
 * eval path, policy/muzero.py:935) or one draw from p (inverse CDF of a counter-based uniform keyed by seed and tree index;
 * the reference draws with np.random.choice), d_action = the action id at that legal position (policy/muzero.py:800).
 * Outputs int32 [B] / f32 [B], any may be NULL.  SURVEY 8(f) row f-3: keeps the collector's action choice on the GPU. */
int lz_tree_select_action(lz_tree *t, float temperature, int deterministic, uint64_t seed, int32_t *d_action,
                          int32_t *d_action_pos, float *d_entropy, lz_stream s);

/* ---- Gumbel MuZero tree (lzero/mcts/ctree/ctree_gumbel_muzero/lib/cnode.cpp, gmz_tree.pyx) ----
 * lz_tree_set_gumbel turns a MuZero tree into a Gumbel tree: sequential halving with Gumbel noise at the root
 * (cselect_root_child, cnode.cpp:701-745) and completed-Q improved-policy selection below it (cselect_interior_child,
 * :747-790); the back-up is the one-player recurrence for every to_play (:605-631).  It builds the root Gumbel vector
 * (10 * Gumbel(0, 1) from std::mt19937(0), the first n draws for a root with n legal actions) and row min(m, S) of the
 * considered-visit table on the host.  num_simulations == 0 turns the tree back into a MuZero tree.  Refused on an
 * EfficientZero tree.  On a Gumbel tree lz_tree_prepare, lz_tree_traverse, lz_tree_backpropagate and lz_search_run run the
 * Gumbel prepare, descent, back-up and search; the reuse descent and search are refused.
 * Descents use the discount of lz_tree_set_params. */
int lz_tree_set_gumbel(lz_tree *t, int max_num_considered_actions, int num_simulations);
/* get_children_values / get_policies (cnode.cpp:309-385, 506-541) with the tree's discount: d_children_values f32 [B,A]
 * completed Q by action id (-inf at illegal actions), d_improved_policy f32 [B,A] softmax(prior + completed Q) by action id.
 * Either may be NULL.  Visit counts, values and trajectories: lz_tree_results. */
int lz_tree_gumbel_policies(lz_tree *t, float *d_children_values, float *d_improved_policy, lz_stream s);
/* What GumbelMuZeroPolicy._forward_collect / _forward_eval (lzero/policy/gumbel_muzero.py:573-605, 685-700) take from the
 * searched roots, in the one pass of lz_tree_gumbel_policies: d_action int32 [B] = np.argmax(np.where(action_mask,
 * improved_policy, 0)) (the first maximum; the same in collect and eval), d_entropy f32 [B] = select_action's visit-count
 * entropy at this temperature (the arithmetic of lz_tree_select_action; it does not depend on the draw), d_children_values
 * f32 [B,A] = np.where(action_mask, completed Q, 0) (roots_completed_value), d_improved_policy f32 [B,A] as
 * lz_tree_gumbel_policies.  Any output may be NULL. */
int lz_tree_gumbel_select_action(lz_tree *t, float temperature, int32_t *d_action, float *d_entropy, float *d_children_values,
                                 float *d_improved_policy, lz_stream s);
/* Host only (no device needed): row min(m, S) of get_table_of_considered_visits(m, S) into h_seq int32 [S] and
 * generate_gumbel(10, 0, A) into h_gumbel f32 [A] (cnode.cpp:1041-1094, 1133-1151).  Either may be NULL. */
int lz_gumbel_tables(int max_num_considered_actions, int num_simulations, int A, int32_t *h_seq, float *h_gumbel);

/* ------------------------------------------------------------------ model (muzero_model.py, efficientzero_model.py) */

typedef struct lz_model_config {
    int obs_c, obs_h, obs_w;       /* observation planes and size: (4|12, 64|84|96, same) */
    int action_space_size;
    int num_res_blocks;            /* per network (reference default 1) */
    int num_channels;              /* 64 */
    int reward_head_channels, value_head_channels, policy_head_channels;   /* 16 */
    int reward_hidden, value_hidden, policy_hidden;                         /* one hidden layer: 32 */
    float support_min, support_max, support_step;                           /* -300, 301, 1 (value == reward) */
    /* EfficientZeroModel (lzero/model/efficientzero_model.py:20-272): the reward head becomes conv1x1 -> BN -> ReLU ->
     * LSTM(hc*h*w -> lstm_hidden_size) -> BN1d -> ReLU -> MLP and predicts a VALUE PREFIX; 0 = MuZeroModel */
    int efficientzero;
    int lstm_hidden_size;          /* 512 (must be a multiple of 16, <= 512) */
    /* 1 = DownSample representation (the Atari network); 0 = the full-resolution board network of downsample=False
     * (common.py:764-787; tictactoe, connect4, gomoku), every layer at the observation's H x W */
    int downsample;
} lz_model_config;

/* downsample = 1, conv models (DownSample representation, common.py:334-366): 84x84 and 96x96 observations give a 6x6 latent
 * grid; 64x64 (the shipped Atari configs) gives 8x8, with no pooling2 (common.py:357-359).  Other sizes: LZ_EINVAL.
 * downsample = 0, board models: latent [num_channels, obs_h, obs_w] with num_channels in {16, 32, 64}, 1 <= obs_h, obs_w <= 8,
 * 1 <= obs_c <= 16, 1 <= action_space_size <= 64, MuZero only (efficientzero = 0); other configs: LZ_EINVAL.  Same head and
 * support limits as the conv models.  The uint8 collect entry points take conv models only. */
int lz_model_create(const lz_model_config *cfg, lz_model **out);

/* MuZeroModelMLP (lzero/model/muzero_model_mlp.py:21-295; vector observations, BASELINE config 1).  The
 * handle is used with the same lz_model_* / lz_search_* calls: d_obs is f32 [B, obs_dim], latents are
 * f32 [B, latent_dim].  State-dict names follow muzero_model_mlp.py / common.py:790-850,1218-1292.
 * Two kernels run it, chosen from the config alone:
 *   - the fp32 CUDA-core kernels take latent_dim 8-128, obs_dim 1-160, latent_dim + action_space_size <= 160 and head hidden
 *     sizes <= 160 (no math mode: lz_model_set_math is LZ_EINVAL);
 *   - every other config with latent_dim a multiple of 32 in [32, 256], obs_dim 1-4096, action_space_size 1-608 and head
 *     hidden sizes 1-32 runs on the tensor-core kernel of EfficientZeroModelMLP (math modes tc3 / tc1; latent buffers in and
 *     out 16-byte aligned).
 * Support size <= 608; anything else is LZ_EINVAL. */
typedef struct lz_mlp_config {
    int obs_dim, action_space_size, latent_dim;         /* 4, 2, 128 for CartPole */
    int reward_hidden, value_hidden, policy_hidden;     /* one hidden layer each: 32 */
    int res_connection_in_dynamics;                     /* policy default True (policy/muzero.py:68) */
    float support_min, support_max, support_step;
} lz_mlp_config;
int lz_model_create_mlp(const lz_mlp_config *cfg, lz_model **out);
/* EfficientZeroModelMLP (lzero/model/efficientzero_model_mlp.py:150-300; vector observations): the MLP representation /
 * prediction networks of MuZeroModelMLP, a dynamics MLP (fc_dynamics, or fc_dynamics_1 + latent -> fc_dynamics_2 with
 * res_connection_in_dynamics) whose output feeds nn.LSTM(latent_dim -> lstm_hidden_size) and fc_reward_head (a VALUE PREFIX,
 * no norm_value_prefix).  Same lz_model_* / lz_search_* calls as EfficientZeroModel: d_obs is f32 [B, obs_dim], latents
 * f32 [B, latent_dim], the reward hidden state f32 [B, lstm_hidden_size] x 2.  Accepted: latent_dim a multiple of 32 in
 * [32, 256], lstm_hidden_size a multiple of 16 in [16, 512], obs_dim 1-4096, action_space_size 1-608, head hidden sizes 1-32,
 * support size <= 608; anything else is LZ_EINVAL.  Math modes tc3 / tc1 as the conv models (lz_model_set_math).  Latent
 * buffers (in and out) must be 16-byte aligned: the kernel moves latent rows as vectors. */
typedef struct lz_mlp_ez_config {
    int obs_dim, action_space_size, latent_dim, lstm_hidden_size;
    int reward_hidden, value_hidden, policy_hidden;     /* one hidden layer each: 32 */
    int res_connection_in_dynamics;
    float support_min, support_max, support_step;
} lz_mlp_ez_config;
int lz_model_create_mlp_ez(const lz_mlp_ez_config *cfg, lz_model **out);
/* StochasticMuZeroModelMLP (lzero/model/stochastic_muzero_model_mlp.py; vector observations): MuZeroModelMLP's representation,
 * dynamics and prediction networks, the dynamics network over [afterstate | one-hot chance outcome], plus
 * afterstate_dynamics_network (a MuZeroModelMLP dynamics network over [latent | one-hot action]) and
 * afterstate_prediction_network (a prediction network with chance_space_size policy outputs).  State-dict names follow the
 * reference class; chance_encoder.* and the SSL projection entries are ignored.  Runs on the tensor-core MLP kernel: latent_dim a
 * multiple of 32 in [32, 256], obs_dim 1-4096, action_space_size and chance_space_size 1-608, head hidden sizes 1-32, support
 * size <= 608; anything else is LZ_EINVAL.  Math modes tc3 / tc1.  initial_inference is lz_model_initial_inference;
 * recurrent_inference is lz_model_recurrent_inference_stochastic.  Its searches run on stochastic trees
 * (lz_tree_set_stochastic) through lz_search_run. */
typedef struct lz_mlp_stochastic_config {
    int obs_dim, action_space_size, chance_space_size, latent_dim;
    int reward_hidden, value_hidden, policy_hidden;     /* one hidden layer each: 32 */
    int res_connection_in_dynamics;
    float support_min, support_max, support_step;
} lz_mlp_stochastic_config;
int lz_model_create_mlp_stochastic(const lz_mlp_stochastic_config *cfg, lz_model **out);
/* StochasticMuZeroModel.recurrent_inference(state, option, afterstate) (stochastic_muzero_model.py:233-273) on B rows:
 * afterstate = 0: afterstate dynamics over [latent d_state | one-hot action d_option] and the afterstate prediction, so
 *   d_next_state is the afterstate and d_policy_logits f32 [B, chance_space_size] the chance logits;
 * afterstate = 1: dynamics over [afterstate d_state | one-hot chance outcome d_option] and the prediction, so d_next_state is
 *   the next latent and d_policy_logits f32 [B, action_space_size].
 * Reward and value as lz_model_recurrent_inference (logits f32 [B, K], scalars f32 [B]); outputs may be NULL.  d_row_mask
 * int32 [B] or NULL: row b is computed only when (d_row_mask[b] & 1) == (row_mask_on & 1), and the other rows are neither
 * read nor written (the fused search splits its leaves this way).  Latent buffers 16-byte aligned. */
int lz_model_recurrent_inference_stochastic(lz_model *m, int afterstate, int B, const float *d_state, const int32_t *d_option,
                                            const int32_t *d_row_mask, int row_mask_on, float *d_next_state,
                                            float *d_reward_logits, float *d_value_logits, float *d_policy_logits,
                                            float *d_reward, float *d_value, lz_stream s);
int lz_model_destroy(lz_model *m);
/* Feed one tensor of the reference state_dict (names as produced by MuZeroModel.state_dict(),
 * SURVEY.md App. B.4; fp32, contiguous, HOST memory).  Unknown names are ignored (returns 1). */
int lz_model_set_tensor(lz_model *m, const char *name, const float *h_data, int64_t numel);
/* Folds eval-mode BatchNorm into per-channel scale/shift, packs weights for the kernels, uploads. */
int lz_model_finalize(lz_model *m);
/* Arithmetic of the conv model's tensor-core kernels (the DownSample tower and the latent-grid networks; the
 * EfficientZeroModelMLP network and its LSTM likewise):
 *   1 = tc3: fp16 hi/lo operand splitting (3 MMAs per product, fp32 accumulate in registers): fp32-accurate, the default
 *       and the mode parity is stated for;
 *   2 = tc1: single fp16 pass (fp32 accumulate): ~3x fewer MMAs, logits accurate to ~1e-3.
 * Any other mode, and any mode on a MuZeroModelMLP that runs on the fp32 MLP kernels, is LZ_EINVAL. */
int lz_model_set_math(lz_model *m, int mode);
/* Test hook: overrides the layer program of the tensor-core kernels (see net_tc.cuh LF_* flags). */
int lz_model_debug_tc_program(lz_model *m, int which, int nlayers, const int *layer_w, const int *layer_flags,
                              int has_reward);
/* Test hook: 64 clock64 stamps of CTA 0 of the last tensor-core launch made with env LZ_TC_DEBUG=1. */
int lz_debug_tc_stamps(unsigned long long *h_out);
/* Test hook: runs the tensor-core DownSample tower on d_obs (f32) or d_obs_u8 (uint8; exactly one non-NULL) through
 * stage `stage` and copies that stage's output tensor, byte for byte, to d_out (out_bytes must be large enough).
 * Stages: 0 stem -> T0, 1 resblocks1 -> T1 (phase-split), 2 / 3 downsample conv1 / conv3 (one launch) -> U0 / U1,
 * 4 downsample conv2 + identity -> U2, 5 resblocks2 -> U0, 6 pooling1 -> V0, 7 resblocks3 -> V1, 8 pooling2 -> the
 * f32 NCHW pre-latent [B][64][6][6] (84 / 96 px); at 64 px the tower has no pooling2 and stage 8 is the conversion of V1 to
 * the f32 NCHW pre-latent [B][64][8][8] (each value hi + lo, summed in fp32).  Stages 0-7 copy the tensor-core layout (conv_tc.cuh):
 * [B][nphase][hi | lo][C / 8][plane_rows][8] fp16.
 * h_info (int32[10]) receives the tensor geometry and the plan of the launch that wrote it:
 * C, H, W, nphase, plane_rows (nphase = plane_rows = 0 for stage 8), then G (images per CTA; 1 for the pools and the
 * conversion), band_h (output rows per CTA; 0 where the launch has no bands), stages (weight ring depth; 0 off the wgmma kernels) and the CTA count of the
 * launch, then npass (3 = tc3, 1 = tc1).  Needs a finalized conv model (LZ_ESTATE otherwise). */
int lz_model_debug_tower_stage(lz_model *m, int B, const float *d_obs, const uint8_t *d_obs_u8, int stage,
                               void *d_out, size_t out_bytes, int32_t *h_info, lz_stream s);
/* Test hook: runs a copy of the latent-grid tensor-core program (`which` 0: recurrent_inference on d_latent f32 [B,64,h,w]
 * NCHW and d_action int32 [B]; 1: the tail of initial_inference on the pre-latent d_latent, d_action unused) cut off after
 * layer `stage`, and writes that layer's f32 output [B,64,h,w] NCHW to d_out (h = w = lz_model_latent_hw: 6 or 8).  The model's own programs are not changed.
 * stage == nlayers runs the whole program twice and writes, f32: reward logits [B,K], value logits [B,K], policy logits
 * [B,A], reward [B], value [B] with the raw logits requested, then policy logits [B,A], reward [B], value [B] without raw
 * reward / value logits (the joint categorical read-out of the search), then for EfficientZero (`which` 0) the reward-head
 * features [B, reward_head_channels*h*w] the LSTM consumes (h*w = 36 or 64).  Sections a program does not produce are zero.
 * h_info (int32[8]) receives the launch plan: roots per CTA R (<= 8 on the 6x6 grid, <= 4 on 8x8), row tiles NT (<= 3), CTA count, roots of the last CTA, layers of
 * the launched program, MMA passes, 1 if the FC2 biases are staged in shared memory, FC2 tiles.
 * Board models (downsample = 0): `which` 1 is the whole initial_inference program on the observations d_latent
 * f32 [B,obs_c,H,W]; outputs as above without the EfficientZero section, latents [B,C,H,W]; h_info: roots per CTA R, 64-row tiles
 * NT, CTA count, roots of the last CTA, layers, MMA passes, shared memory bytes, 0.
 * EfficientZeroModelMLP: `which` 0 is recurrent_inference's dense program on d_latent f32 [B, latent_dim] and d_action, `which` 1
 * initial_inference's on the observations d_latent f32 [B, obs_dim].  stage < D (D = the L-wide layers before the heads: 4 for
 * `which` 1, 4 or 6 for `which` 0) writes that layer's output f32 [B, latent_dim] (after the LayerNorm for the representation's
 * second layer, after the residual for fc_dynamics_1); stage == D runs the whole program and writes latent [B, latent_dim], the
 * LSTM input [B, latent_dim] (`which` 0; zeros for `which` 1; no LSTM runs), value logits [B,K], policy logits [B,A], value [B].
 * h_info: roots per CTA, CTA count, roots of the last CTA, layers of the launched program, MMA passes, shared memory bytes, weight
 * ring stages, D.
 * MuZeroModelMLP on the fp32 kernels (latent_dim <= 128): `which` as for EfficientZeroModelMLP.  stage < D cuts the program after
 * its dense layer `stage` and writes that layer's f32 output [B, width]: for `which` 1 (D = 9) fc_representation.0 with BN and
 * GELU, fc_representation.3, the LayerNorm, then the prediction network; for `which` 0 fc_dynamics_1.0 (one-hot rows included),
 * fc_dynamics_1.3, the residual add, fc_dynamics_2.0, fc_dynamics_2.3 (D = 13; without res_connection_in_dynamics fc_dynamics.0,
 * fc_dynamics.3, D = 10), the reward head's two layers, then the prediction network.  The prediction network's stages are
 * fc_prediction_common.0 and .3, the value head's two layers, the policy head's two layers; every layer with its BN and
 * activation.  width is latent_dim, a head's hidden size, the support size or A.  stage == D runs the whole program and writes
 * latent [B, latent_dim], value logits [B,K], policy logits [B,A], value [B], and for `which` 0 reward logits [B,K], reward [B].
 * h_info: roots per CTA (4), CTA count, roots of the last CTA, D, width (0 for stage D), 0, 0, 0.
 * MuZeroModelMLP and StochasticMuZeroModelMLP on the tensor cores: stages as for EfficientZeroModelMLP; stage == D writes latent
 * [B, latent_dim], a zero section [B, latent_dim], value logits [B,K], policy logits [B,P], value [B], and for the recurrent
 * programs reward logits [B,K], reward [B].  StochasticMuZeroModelMLP's `which` 0 is its dynamics program on afterstates
 * d_latent and chance outcomes d_action (P = A); `which` 2 is its afterstate program on latents d_latent and actions d_action:
 * the afterstate dynamics, its reward head and the afterstate prediction (P = chance_space_size).  Any other model refuses
 * `which` 2 (LZ_EINVAL). */
int lz_model_debug_net_stage(lz_model *m, int which, int B, const float *d_latent, const int32_t *d_action, int stage,
                             void *d_out, size_t out_bytes, int32_t *h_info, lz_stream s);
int lz_model_latent_hw(const lz_model *m);   /* 6 for 84/96, 8 for 64; a square board's side; 0 for a non-square board */
/* Shape of one root's latent: channels, height, width (h_c / h_h / h_w may be NULL).  The MLP model reports (latent_dim, 1, 1). */
int lz_model_latent_shape(const lz_model *m, int32_t *h_c, int32_t *h_h, int32_t *h_w);
int lz_model_support_size(const lz_model *m);

/* initial_inference (muzero_model.py:210-240).  d_obs f32 [B,obs_c,H,W].  Outputs (NULL to skip):
 * d_latent f32 [B,C,h,w] (NCHW, as the reference returns), d_policy_logits f32 [B,A],
 * d_value_logits f32 [B,support], d_value f32 [B] (inverse-transformed scalar). */
int lz_model_initial_inference(lz_model *m, int B, const float *d_obs, float *d_latent,
                               float *d_policy_logits, float *d_value_logits, float *d_value,
                               lz_stream s);
/* recurrent_inference (muzero_model.py:242-272).  d_latent f32 [B,C,h,w], d_action int32 [B].
 * Outputs (NULL to skip): d_next_latent [B,C,h,w], d_reward_logits/d_value_logits [B,support],
 * d_policy_logits [B,A], d_reward/d_value f32 [B] scalars after the inverse transform. */
int lz_model_recurrent_inference(lz_model *m, int B, const float *d_latent, const int32_t *d_action,
                                 float *d_next_latent, float *d_reward_logits, float *d_value_logits,
                                 float *d_policy_logits, float *d_reward, float *d_value, lz_stream s);
/* EfficientZeroModel.recurrent_inference (efficientzero_model.py:240-272).  The reward hidden state is the tuple the
 * reference passes to nn.LSTM: d_hidden0 = element 0 (LSTM h), d_hidden1 = element 1 (LSTM c), each f32 [B, lstm_hidden_size]
 * (the leading sequence dimension of 1 dropped).  Outputs as lz_model_recurrent_inference with the value prefix in place of
 * the reward, plus the next hidden state (un-reset: resetting every lstm_horizon_len steps is the search driver's job,
 * mcts_ctree.py:856-861).  initial_inference is lz_model_initial_inference (the hidden state starts as zeros). */
int lz_model_recurrent_inference_ez(lz_model *m, int B, const float *d_latent, const float *d_hidden0, const float *d_hidden1,
                                    const int32_t *d_action, float *d_next_latent, float *d_next_hidden0, float *d_next_hidden1,
                                    float *d_value_prefix_logits, float *d_value_logits, float *d_policy_logits,
                                    float *d_value_prefix, float *d_value, lz_stream s);
int lz_model_lstm_hidden_size(const lz_model *m);   /* 0 for a MuZero model */

/* InverseScalarTransform (scaling_transform.py:82-92) on its own: logits f32 [B,support] -> f32 [B]. */
int lz_inverse_scalar_transform(lz_model *m, int B, const float *d_logits, float *d_out, lz_stream s);

/* ------------------------------------------------------------------ fused search (mcts_ctree.py) */

/* Binds a tree and a model; owns the latent pool [(num_simulations+1), B, C, h, w] and the CUDA
 * graph holding [traverse -> recurrent_inference -> backpropagate] x num_simulations. */
int lz_search_create(lz_tree *t, lz_model *m, int num_simulations, lz_search **out);
int lz_search_destroy(lz_search *q);
/* MuZeroMCTSCtree.search (mcts_ctree.py:267-368) on roots already prepared with lz_tree_prepare.
 * d_latent_roots f32 [B,C,h,w].  One graph launch, zero host syncs.  An EfficientZero search runs with lz_search_run_ez.
 * On a Gumbel tree (lz_tree_set_gumbel) with a MuZero conv or MLP model: GumbelMuZeroMCTSCtree.search (mcts_ctree.py:1076-1172),
 * one CUDA graph of [Gumbel descent] + num_simulations x [recurrent_inference, Gumbel back-up + next descent]; `deterministic`
 * is ignored, the roots must be freshly prepared (no descent since lz_tree_prepare; LZ_ESTATE) and the search's
 * num_simulations may not exceed the tree's Gumbel num_simulations (LZ_EINVAL).
 * On a stochastic tree (lz_tree_set_stochastic) with a StochasticMuZeroModelMLP: StochasticMuZeroMCTSCtree.search
 * (mcts_ctree_stochastic.py:117-252), one CUDA graph of [descent] + num_simulations x [the afterstate program on the leaves that
 * are chance nodes, the dynamics program on the others (one row mask, its two parities), back-up + next descent]; both programs
 * write the same latent pool slot.  `deterministic` is the decision nodes' tie rule.  lz_search_collect* runs the same graph
 * (see there). */
int lz_search_run(lz_search *q, const float *d_latent_roots, int deterministic, lz_stream s);
/* MuZeroMCTSCtree.search_with_reuse (mcts_ctree.py:370-468; ReZero) and EfficientZeroMCTSCtree.search_with_reuse (:878-1003).
 * d_true_action int32 [B], d_reuse_value f32 [B] as for the reuse lz_tree_traverse; d_infer_count int32 [num_simulations] or
 * NULL receives, per simulation, how many trees needed the network (the reference returns the last count and the mean).  One
 * CUDA graph; "no inference" rows are computed and ignored instead of compacted on the host.  Ties by lz_tree_set_tiebreak.
 * An EfficientZero search takes the roots' LSTM state d_hidden{0,1}_roots as lz_search_run_ez (NULL = zeros); its graph has
 * 5 x num_simulations kernels and is_reset is taken per TREE from the descent (search_len % lstm_horizon_len; the
 * reference indexes a compacted list by tree at :1040-1046 / cnode.cpp:646, see DESIGN.md 4.6).  A MuZero search takes
 * NULL hidden pointers (LZ_EINVAL otherwise).  Refused on a Gumbel or a stochastic tree (LZ_ESTATE). */
int lz_search_run_with_reuse(lz_search *q, const float *d_latent_roots, const float *d_hidden0_roots, const float *d_hidden1_roots,
                             const int32_t *d_true_action, const float *d_reuse_value, int32_t *d_infer_count, lz_stream s);
/* EfficientZeroMCTSCtree.search (mcts_ctree.py:671-876) for a search created from an EfficientZero model and a tree in
 * EfficientZero mode.  d_hidden{0,1}_roots: f32 [B, lstm_hidden_size] = reward_hidden_state_roots[0] / [1] (NULL = zeros,
 * what initial_inference returns).  The LSTM state of a leaf is zeroed every lstm_horizon_len steps of depth (:856-861). */
int lz_search_run_ez(lz_search *q, const float *d_latent_roots, const float *d_hidden0_roots, const float *d_hidden1_roots, lz_stream s);
/* The search-feeding part of _forward_collect (policy/muzero.py:749-779): initial_inference ->
 * reset(mask) -> prepare(noise) -> search.  d_obs f32 [B,obs_c,H,W]; d_mask uint8 [B,A] or NULL;
 * d_noise f32 [B,A] legal-order rows or NULL; d_to_play int32 [B] or NULL (-1).
 * Optional outputs: d_pred_value f32 [B] (root value prediction), d_policy_logits f32 [B,A].
 * On a Gumbel tree (lz_tree_set_gumbel) lz_tree_prepare takes the root value prediction as the roots' values
 * (GumbelMuZeroPolicy._forward_collect, gumbel_muzero.py:560-571) and the search is the Gumbel graph of lz_search_run; the
 * search's num_simulations may not exceed the tree's Gumbel num_simulations (LZ_EINVAL).  The same holds for the three
 * entry points below.  Read the results with lz_tree_results and lz_tree_gumbel_select_action.
 * On a stochastic tree (lz_tree_set_stochastic) with a StochasticMuZeroModelMLP (StochasticMuZeroPolicy._forward_collect /
 * _forward_eval, lzero/policy/stochastic_muzero.py:578-760) the search is the stochastic graph of lz_search_run, and every row
 * of d_mask, d_noise and d_policy_logits is the tree's width W = max(action_space_size, chance_space_size) wide: d_policy_logits
 * receives initial_inference's policy in the first action_space_size columns of each row (the others are not written), mask
 * columns at action_space_size and beyond are ignored and noise columns past the legal count are not read.  The step's reset
 * advances the tree's RNG epoch, so with chance_u < 0 successive collects (and replays of one captured graph) draw their chance
 * outcomes independently; with chance_u in [0, 1) every draw is the pinned one.  lz_tree_select_action then reads the root's
 * legal children and returns action ids < action_space_size.  The same holds for the host entry points below. */
int lz_search_collect(lz_search *q, const float *d_obs, const uint8_t *d_mask, const float *d_noise,
                      float noise_weight, const int32_t *d_to_play, int deterministic,
                      float *d_pred_value, float *d_policy_logits, lz_stream s);
/* Same with HOST buffers (pinned memory recommended): h_obs f32 [B,obs_c,H,W], h_mask uint8 [B,A] or NULL,
 * h_noise f32 [B,A] or NULL, h_to_play int32 [B] or NULL.  The observation batch is copied in `nchunks`
 * (1..8) pieces on an internal copy stream so that the copy of chunk i+1 overlaps the representation
 * network of chunk i; everything else is ordered on `s`.  The host buffers must stay valid until `s`
 * reaches the end of the call's work. */
int lz_search_collect_host(lz_search *q, const float *h_obs, const uint8_t *h_mask, const float *h_noise,
                           float noise_weight, const int32_t *h_to_play, int deterministic, int nchunks,
                           float *d_pred_value, float *d_policy_logits, lz_stream s);
/* The same two entry points for uint8 frames [B,obs_c,H,W] (Atari frames as the emulator delivers them; a quarter of the
 * bytes on the wire).  The [0, 1] scaling of the reference's env wrapper (ScaledFloatFrameWrapper: obs / 255 -> float32,
 * zoo/atari/envs/atari_wrappers.py:219-220, atari_lightzero_env.py:87-88) is applied inside the first conv kernel, bit-identical
 * to that host arithmetic.  Conv model only; 64x64, 84x84 and 96x96 frames. */
int lz_search_collect_u8(lz_search *q, const uint8_t *d_obs_u8, const uint8_t *d_mask, const float *d_noise,
                         float noise_weight, const int32_t *d_to_play, int deterministic,
                         float *d_pred_value, float *d_policy_logits, lz_stream s);
int lz_search_collect_host_u8(lz_search *q, const uint8_t *h_obs_u8, const uint8_t *h_mask, const float *h_noise,
                              float noise_weight, const int32_t *h_to_play, int deterministic, int nchunks,
                              float *d_pred_value, float *d_policy_logits, lz_stream s);
/* ---- ReZero policy reanalyze (ReZeroMZGameBuffer._compute_target_policy_reanalyzed, lzero/mcts/buffer/game_buffer_rezero_mz.py:194-404;
 * ReZeroEZGameBuffer, game_buffer_rezero_ez.py:126-330; SURVEY 8(f) row f-4) ----
 * The whole sweep over N sampled segments of L positions, for a search q created for N roots (B = N).  Every [N*L] input is in the
 * reference's flat order, row i = segment * L + position:
 *   d_obs f32 [N*L, obs...] (initial_inference runs over all rows in mini_infer_size slices), or instead d_latent f32 [N*L, latent]
 *   and d_logits f32 [N*L, A] of a prior initial_inference (d_obs NULL);
 *   d_mask uint8 [N*L, A] (legal actions; an all-zero row is every action), d_to_play int32 [N*L] or NULL (-1),
 *   d_true_action int32 [N*L] (the reference's -2 for a segment's last step and for padding), d_policy_mask uint8 [N*L],
 *   d_noise f32 [N*L, A] in legal order or NULL (reanalyze_noise = False), noise_weight.
 * q may be a MuZero or an EfficientZero search (the LSTM state at every root is zero, as initial_inference returns it); a
 * Gumbel or a stochastic search is refused (LZ_ESTATE).
 * The searches run backward from position L - 1: a plain search (MuZero: ties by `deterministic`; EfficientZero: first maximum,
 * `deterministic` is ignored),
 * then, with reuse_search, L - 1 search_with_reuse calls each reusing the root values of the position searched before it (ties:
 * first maximum, the reference's rand() == 0); without reuse_search L plain searches.  Outputs:
 *   d_targets f64 [N, L, A]: visit / sum(visits) by legal position (scatter_legal = 0, fixed_action_space) or by action id
 *   (scatter_legal != 0), zeros where policy_mask == 0; d_root_values f32 [N, L]; d_child_visits f64 [N, L, A]: visit / sum in
 *   legal order, zero padded (what the buffer stores back); d_infer_count int32 [L - 1, S] (reuse_search, L > 1; else may be NULL):
 *   per reuse search and simulation, how many trees needed the network.
 * Everything is enqueued on s with no host synchronisation: initial_inference, then L x [handoff kernel, the search's captured
 * graph, targets kernel].  The graphs are those of lz_search_run(_ez) / lz_search_run_with_reuse, captured once and replayed
 * along the sweep.
 * Sets the tree's tie-break rule to first maximum (lz_tree_set_tiebreak). */
int lz_rezero_reanalyze(lz_search *q, int L, int reuse_search, int mini_infer_size, const float *d_obs, const float *d_latent,
                        const float *d_logits, const uint8_t *d_mask, const int32_t *d_to_play, const int32_t *d_true_action,
                        const uint8_t *d_policy_mask, const float *d_noise, float noise_weight, int deterministic, int scatter_legal,
                        double *d_targets, float *d_root_values, double *d_child_visits, int32_t *d_infer_count, lz_stream s);
/* ---- Replay-buffer reward and value targets (MuZeroGameBuffer._compute_target_reward_value,
 * lzero/mcts/buffer/game_buffer_muzero.py:467-575; EfficientZeroGameBuffer, game_buffer_efficientzero.py:167-323) ----
 * N sampled segments of K1 = num_unroll_steps + 1 rows, T = N * K1 rows, row = segment * K1 + position (the reference's
 * value_obs_list order).  The host packs the ragged reward and to_play windows and the discount powers into the device tables
 * below (lightzero_b200.reanalyze.compute_target_reward_value); every power is computed on the host with the reference's own
 * expression, the device only multiplies and adds. */
typedef struct lz_value_tables {
    int N, K1;                     /* segments, rows per segment */
    int W, P;                      /* reward window width (K1 - 1 + P), power-table length (the largest td) */
    int value_prefix;              /* 1: EfficientZero value prefixes and targets; 0: MuZero rewards and targets */
    int fp32;                      /* 1: float32 rewards (float32 products, float32 sums after the first add); 0: float64 */
    int two_player;                /* env_type == 'board_games' and to_play_segment[0][0] in [1, 2] */
    int horizon;                   /* lstm_horizon_len (value_prefix) */
    int alias_prefix;              /* value_prefix with (n, 1) rewards: the reference appends one array per horizon chunk, added
                                      to in place, so every row of a chunk reads the chunk's last prefix */
    const double *rewards;         /* [N][W]: reward_list[pos + w] (exact float64 of the float32 rewards), 0 past rlen */
    const int32_t *rlen;           /* [N]: clip(len(reward_list) - pos, 0, W) */
    const int32_t *seglen;         /* [N]: clip(game_segment_len - pos, 0, K1) (value_prefix) */
    const int32_t *td;             /* [T]: td_steps_list */
    const double *bootstrap;       /* [T]: discount ** td, negated for odd td in two_player mode */
    const double *value_mask;      /* [T] */
    const double *powers;          /* [P]: discount ** i */
    const int32_t *to_play;        /* two_player: [N][P + K1], to_play_list[i] for i < P then to_play_list[pos + k]; else NULL */
} lz_value_tables;
/* initial_inference over the T observations d_obs f32 [T, obs...] in mini_infer_size slices (value scalars only, into d_values
 * f32 [T]), then one thread per segment writes d_reward_out f64 [N, K1] (rewards, or value prefixes) and d_value_out f64 [N, K1]
 * (value targets).  The model must be an EfficientZero model exactly when tab->value_prefix.  Enqueued on s, no host sync. */
int lz_value_targets(lz_model *m, const lz_value_tables *tab, int mini_infer_size, const float *d_obs, float *d_values,
                     double *d_reward_out, double *d_value_out, lz_stream s);
/* EfficientZero with use_root_value: for an EfficientZero search q of B = T roots, initial_inference in mini_infer_size slices
 * (latents into the search's pool, policy logits), the roots reset to d_mask uint8 [T, A] and prepared with zero value prefixes,
 * d_noise f32 [T, A] in legal order (NULL: prepare_no_noise), noise_weight and d_to_play int32 [T] (NULL: -1), the search's
 * captured graph on zero LSTM state (ties: first maximum when first_maximum, lz_tree_set_tiebreak), its root values into
 * d_values f32 [T], then the targets as lz_value_targets.  A repeated call of the same shapes captures no graph. */
int lz_value_targets_root(lz_search *q, const lz_value_tables *tab, int mini_infer_size, const float *d_obs, const uint8_t *d_mask,
                          const int32_t *d_to_play, const float *d_noise, float noise_weight, int first_maximum, float *d_values,
                          double *d_reward_out, double *d_value_out, lz_stream s);
/* Test hook: search graphs this library has captured since load (a capture happens on a search's first run and after a change of
 * the model, the tree parameters or the tie rule). */
unsigned long long lz_debug_graph_captures(void);
/* Number of kernel nodes of the search graph this search launched last (any lz_search_run* / lz_search_collect* call). */
int lz_search_num_kernels(const lz_search *q);
/* Test hook: the launch plan of lz_search_run, host only.  h_info int32[8]: 1 if the search is one persistent launch of the
 * tensor-core kernel (else 0 and the next six entries are 0), roots per CTA R, CTAs, roots of the last CTA, 1 if the
 * exploration-rate table pbc[] is staged in shared memory, 1 if the FC2 biases are, layers of the recurrent program, and the
 * node slots N of the tree (max_sims + 1). */
int lz_search_debug_plan(const lz_search *q, int32_t *h_info);
/* Device pointer of the latent pool (NCHW per slot) for inspection in tests. */
const float *lz_search_latent_pool(const lz_search *q);
/* EfficientZero: device LSTM-state pool [(S+1)][B][H], which = 0 / 1 for tuple element 0 / 1 (NULL for MuZero). */
const float *lz_search_hidden_pool(const lz_search *q, int which);


/* ---- collector state on the device (SURVEY 8(f) row f-3) ----
 * Observation frame stacks: what the reference collector rebuilds on the host every step with
 * GameSegment.get_obs() = obs_segment[t : t + frame_stack_num] (lzero/mcts/buffer/game_segment.py:140-156), seeded with
 * frame_stack_num copies of the first frame (lzero/worker/muzero_collector.py:451-457) and fed one new frame per step
 * (GameSegment.append, game_segment.py:158-181; muzero_collector.py:520-545).  Here only the NEW uint8 frame of every environment
 * crosses PCIe (B*H*W bytes instead of B*stack*H*W*4); lz_frames_stacked() is the [B, stack, H, W] uint8 batch (oldest frame
 * first) that lz_search_collect_u8 consumes.  H*W must be a multiple of 16. */
int lz_frames_create(int B, int stack, int H, int W, lz_frames **out);
int lz_frames_destroy(lz_frames *f);
/* d_new_frames uint8 [B,H,W]; d_reset uint8 [B] or NULL: 1 = the environment was reset, its whole stack becomes the new frame. */
int lz_frames_push(lz_frames *f, const uint8_t *d_new_frames, const uint8_t *d_reset, lz_stream s);
/* The same from HOST buffers (pinned memory recommended); they must stay valid until `s` reaches the copies. */
int lz_frames_push_host(lz_frames *f, const uint8_t *h_new_frames, const uint8_t *h_reset, lz_stream s);
/* Device pointer of the current stacks; valid until the next push. */
const uint8_t *lz_frames_stacked(lz_frames *f);
/* GameSegment.store_search_stats (game_segment.py:241-263, idx=None) for B segments of capacity T: appends
 * child_visits[b][len[b]][k] = visit_counts[k] / sum(visit_counts) (computed in float64 as Python does, 1e-6 denominator when every
 * count is 0; k = position in the root's legal-action list, 0 beyond it) and root_values[b][len[b]].  d_visits int32 [B,A] / d_values
 * f32 [B] as lz_tree_results returns them (-1 beyond the legal list); d_active uint8 [B] or NULL selects the environments that
 * stepped.  A full segment (len == T) is left unchanged. */
int lz_segments_create(int B, int T, int A, lz_segments **out);
int lz_segments_destroy(lz_segments *g);
int lz_segments_store_search_stats(lz_segments *g, const int32_t *d_visits, const float *d_values, const uint8_t *d_active, lz_stream s);
/* GameSegment.reset (game_segment.py:340-362) of the statistics: len = 0 where d_done[b] != 0 (NULL: everywhere). */
int lz_segments_reset(lz_segments *g, const uint8_t *d_done, lz_stream s);
/* Device pointers: child_visits f32 [B,T,A], root_values f32 [B,T], len int32 [B] (any may be NULL). */
int lz_segments_data(lz_segments *g, float **d_child_visits, float **d_root_values, int32_t **d_len);
/* The improved_policy argument of store_search_stats (Gumbel MuZero, game_segment.py:258-259): d_improved_policy f32 [B,A] by
 * action id is stored at position len[b], the one the NEXT lz_segments_store_search_stats fills, with the same d_active and
 * full-segment rule: call it first for the step.  The f32 [B,T,A] array is allocated (zeroed) by the first call; lz_segments_reset
 * zeroes the rows of the segments it resets. */
int lz_segments_store_improved_policy(lz_segments *g, const float *d_improved_policy, const uint8_t *d_active, lz_stream s);
/* Device pointer of the improved-policy array f32 [B,T,A]; NULL before the first lz_segments_store_improved_policy. */
int lz_segments_improved_policy(lz_segments *g, float **d_improved_policy);

#ifdef __cplusplus
}
#endif
#endif /* LZB200_H */
