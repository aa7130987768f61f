"""Mirror of the reanalyze call site of the search, ``MuZeroGameBuffer._compute_target_policy_reanalyzed``
(lzero/mcts/buffer/game_buffer_muzero.py:578-730): the replay buffer re-searches
``batch_size * (num_unroll_steps + 1)`` stored observations with the latest model and turns the root
visit counts into policy targets.  This is the second caller of ``MuZeroMCTSCtree.search`` in the
reference and its largest natural batch (1536 roots by default).  With an ``EfficientZeroMCTSCtree`` it follows
``EfficientZeroGameBuffer._compute_target_policy_reanalyzed`` (game_buffer_efficientzero.py:325-440): the same flow with
the (zero) reward hidden state of ``initial_inference`` handed to the value-prefix search.

Everything between the observation batch and the visit counts stays on the GPU: ``initial_inference``
in ``mini_infer_size`` slices (:612-633), root preparation with/without Dirichlet noise (:644-652), one
CUDA-graph search (:654-658); the per-segment target assembly (:676-730) is host-side bookkeeping on
the small [roots, A] result and follows the reference line by line.

``compute_target_reward_value`` mirrors the other target computation of ``GameBuffer.sample()``,
``_compute_target_reward_value`` of the MuZero and EfficientZero buffers, as one device call (csrc/targets.cu).
"""
from typing import List, Optional, Sequence

import numpy as np
import torch

from .mcts_ctree import EfficientZeroMCTSCtree, MuZeroMCTSCtree


def compute_target_policy_reanalyzed(
        model, mcts: MuZeroMCTSCtree, policy_obs: torch.Tensor, action_mask: np.ndarray, to_play: Sequence[int],
        policy_mask: Sequence[int], pos_in_game_segment_list: Sequence[int], child_visits: Optional[List[list]] = None,
        num_unroll_steps: int = 5, action_space_size: Optional[int] = None, action_type: str = "fixed_action_space",
        reanalyze_noise: bool = True, mini_infer_size: int = 10240, noises: Optional[np.ndarray] = None,
        return_roots: bool = False):
    """policy_obs: [transition_batch_size, ...] observations (host or device); action_mask [T, A] 0/1;
    to_play [T]; policy_mask [T] (0 = padding beyond the episode end); pos_in_game_segment_list [segments];
    child_visits: per segment, the list the reference updates in place with the fresh distributions.
    Returns np.ndarray [segments, num_unroll_steps + 1, A] (game_buffer_muzero.py:728)."""
    cfg = mcts._cfg
    T = policy_obs.shape[0]
    action_mask = np.asarray(action_mask)
    A = action_space_size or action_mask.shape[1]
    legal_actions = [np.nonzero(action_mask[j])[0].tolist() for j in range(T)]          # :610
    dev = model.device
    lat, logits, hid0, hid1 = [], [], [], []
    ez = isinstance(mcts, EfficientZeroMCTSCtree)      # EfficientZeroGameBuffer._compute_target_policy_reanalyzed, game_buffer_efficientzero.py:325-440
    for beg in range(0, T, mini_infer_size):                                              # :612-633
        out = model.initial_inference(policy_obs[beg:beg + mini_infer_size].to(dev, non_blocking=True))
        lat.append(out.latent_state)
        logits.append(out.policy_logits)
        if ez:                                                                            # game_buffer_efficientzero.py:365-372
            hid0.append(out.reward_hidden_state[0])
            hid1.append(out.reward_hidden_state[1])
    latent_state_roots = torch.cat(lat) if len(lat) > 1 else lat[0]
    policy_logits_pool = torch.cat(logits) if len(logits) > 1 else logits[0]
    if noises is None:                                                                    # :638-641 (A entries per root)
        noises = np.stack([np.random.dirichlet([cfg.root_dirichlet_alpha] * A).astype(np.float32) for _ in range(T)])
    roots = mcts.roots(T, legal_actions)                                                  # :644
    reward_pool = [0.] * T                                                                # initial_inference rewards
    if reanalyze_noise:
        roots.prepare(cfg.root_noise_weight, noises, reward_pool, policy_logits_pool, list(to_play))   # :646
    else:
        roots.prepare_no_noise(reward_pool, policy_logits_pool, list(to_play))            # :648
    if ez:
        hidden_roots = (torch.cat(hid0, dim=1), torch.cat(hid1, dim=1))                   # game_buffer_efficientzero.py:375-376
        mcts.search(roots, model, latent_state_roots, hidden_roots, list(to_play))        # :398-400
    else:
        mcts.search(roots, model, latent_state_roots, list(to_play))                      # :654-658
    roots_distributions = roots.get_distributions()                                       # :674
    roots_values = roots.get_values()

    batch_target_policies_re = []
    policy_index = 0
    if child_visits is None:
        child_visits = [dict() for _ in pos_in_game_segment_list]
    for state_index, child_visit in zip(pos_in_game_segment_list, child_visits):         # :679
        target_policies = []
        for current_index in range(state_index, state_index + num_unroll_steps + 1):
            distributions = roots_distributions[policy_index]
            if policy_mask[policy_index] == 0:                                            # :686-688
                target_policies.append([0 for _ in range(A)])
            else:
                sum_visits = sum(distributions)
                child_visit[current_index] = [v / sum_visits for v in distributions]      # :691,704-705
                if action_type == "fixed_action_space":                                   # :707-711
                    target_policies.append([v / sum_visits for v in distributions])
                else:                                                                     # :712-721 (board games)
                    policy_tmp = [0 for _ in range(A)]
                    for index, legal_action in enumerate(legal_actions[policy_index]):
                        policy_tmp[legal_action] = distributions[index] / sum_visits
                    target_policies.append(policy_tmp)
            policy_index += 1
        batch_target_policies_re.append(target_policies)
    out = np.array(batch_target_policies_re)
    if return_roots:
        return out, roots_values, roots
    roots.clear()
    return out


def rezero_write_back(child_visits, root_values, pos_in_game_segment_list, length, policy_mask, action_mask, visits, values):
    """The buffer-side write-back of the sweep (game_buffer_rezero_mz.py:378-392): where policy_mask is 1, segment n's
    ``child_visits[n][pos + p]`` becomes the legal-order distribution visits[n, p, :nlegal] and ``root_values[n][pos + p]`` the
    searched value (a Python float of the fp32 value, as get_values() returns it).  Either list may be None."""
    action_mask = np.asarray(action_mask)
    nlegal = np.count_nonzero(action_mask, axis=1)
    nlegal[nlegal == 0] = action_mask.shape[1]          # an empty legal list is every action (cnode.cpp:101-107)
    pm = np.asarray(policy_mask)
    for n, state_index in enumerate(pos_in_game_segment_list):
        for p in range(length):
            i = n * length + p
            if pm[i] == 0:
                continue
            if child_visits is not None:
                child_visits[n][state_index + p] = visits[n, p, :nlegal[i]].tolist()
            if root_values is not None:
                root_values[n][state_index + p] = float(values[n, p])


def rezero_reuse_stats(infer_count: np.ndarray, num_simulations: int):
    """What ReZeroMZGameBuffer adds to ``active_root_num`` / ``average_infer`` (game_buffer_rezero_mz.py:352-359) from the
    per-simulation inference counts [L - 1, S] of the reuse searches: the mean over them of the last count and of
    ``sum / num_simulations`` (mcts_ctree.py:464-467); (0, 0.0) without reuse searches."""
    if len(infer_count) == 0:
        return 0, 0.0
    temp_length, temp_infer = 0, 0
    for c in infer_count:
        temp_length += int(c[-1])
        temp_infer += int(c.sum()) / num_simulations
    return temp_length / len(infer_count), temp_infer / len(infer_count)


def compute_target_policy_reanalyzed_rezero(
        model, mcts: MuZeroMCTSCtree, policy_obs, action_mask, to_play, true_action, policy_mask,
        pos_in_game_segment_list: Sequence[int], length: int, child_visits: Optional[List[list]] = None,
        root_values: Optional[List[list]] = None, action_space_size: Optional[int] = None,
        action_type: str = "fixed_action_space", reanalyze_noise: bool = True, reuse_search: bool = True,
        mini_infer_size: int = 10240, noises: Optional[np.ndarray] = None):
    """Mirror of ``ReZeroMZGameBuffer._compute_target_policy_reanalyzed`` (lzero/mcts/buffer/game_buffer_rezero_mz.py:194-404;
    with an ``EfficientZeroMCTSCtree``, ``ReZeroEZGameBuffer``'s, game_buffer_rezero_ez.py:126-330) as one device call
    (``lz_rezero_reanalyze`` / ``_ez``): initial_inference over every row, the plain search of the last position, then
    ``length - 1`` search_with_reuse calls walking backward, each reusing the previous search's root values, and the targets.

    policy_obs [N * length, ...] (row = segment * length + position), action_mask [N * length, A] 0/1, to_play, true_action
    (-2 past a segment's end) and policy_mask [N * length]; pos_in_game_segment_list [N].  ``child_visits`` / ``root_values``:
    per segment, the lists the reference rewrites in place at ``pos + position`` where policy_mask is 1.
    Returns ``(targets, (active_root_num, average_infer))``: the np.ndarray [N, length, A] the reference returns and what it adds
    to those two statistics.  Ties: the first search by the config's ``deterministic`` (MuZero), the reuse searches and every
    EfficientZero search by the first maximum (the reference's rand() % len(ties) with rand() == 0).  ``noises`` [N * length, A]
    (legal order) are drawn with np.random.dirichlet like the reference only when None."""
    from . import mz_tree
    from .efficientzero_model import EfficientZeroModel
    from .efficientzero_model_mlp import EfficientZeroModelMLP
    from .mcts_ctree import GumbelMuZeroMCTSCtree, UniZeroMCTSCtree
    from .muzero_model import MuZeroModel
    from .muzero_model_mlp import MuZeroModelMLP
    from . import cabi

    L = int(length)
    if L < 1:
        raise ValueError(f"compute_target_policy_reanalyzed_rezero: length must be >= 1 (got {length}); the reference builds no "
                         "rows for length < 1")
    if isinstance(mcts, (GumbelMuZeroMCTSCtree, UniZeroMCTSCtree)) or not isinstance(mcts, MuZeroMCTSCtree):
        raise TypeError(f"compute_target_policy_reanalyzed_rezero: {type(mcts).__name__} has no ReZero sweep "
                        "(MuZeroMCTSCtree or EfficientZeroMCTSCtree)")
    ez = isinstance(mcts, EfficientZeroMCTSCtree)
    ez_model = isinstance(model, (EfficientZeroModel, EfficientZeroModelMLP))
    if ez and not ez_model:
        raise TypeError(f"EfficientZeroMCTSCtree: the ReZero sweep needs an EfficientZeroModel or EfficientZeroModelMLP, "
                        f"not a {type(model).__name__}")
    if not ez and (ez_model or not isinstance(model, (MuZeroModel, MuZeroModelMLP))):
        raise TypeError(f"MuZeroMCTSCtree: the ReZero sweep needs a MuZeroModel or MuZeroModelMLP, not a {type(model).__name__}")
    if ez and not mcts.deterministic:
        raise ValueError("EfficientZeroMCTSCtree: the ReZero sweep breaks every tie by the first maximum (the reference's "
                         "EfficientZero tree has no other rule); deterministic=False is not available")
    cfg = mcts._cfg
    S = int(cfg.num_simulations)
    N = len(pos_in_game_segment_list)
    rows = N * L
    action_mask = np.asarray(action_mask)
    A = int(action_space_size or action_mask.shape[1])
    if policy_obs.shape[0] != rows or action_mask.shape != (rows, A):
        raise ValueError(f"compute_target_policy_reanalyzed_rezero: {N} segments x length {L} = {rows} rows, got policy_obs "
                         f"{tuple(policy_obs.shape)} and action_mask {action_mask.shape}")
    if noises is None:        # game_buffer_rezero_mz.py:266-270 (drawn whether or not reanalyze_noise uses them)
        noises = np.stack([np.random.dirichlet([cfg.root_dirichlet_alpha] * A).astype(np.float32) for _ in range(rows)])
    dev = model.device
    H = int(cfg.lstm_horizon_len) if ez else 5
    t = mz_tree.acquire_tree(dev, N, A, S)
    try:
        t.set_params(*mcts._params())
        cabi.check(t.lib.lz_tree_set_gumbel(t.h, 0, 0), "lz_tree_set_gumbel")     # a pooled tree a Gumbel collect left behind
        cabi.check(t.lib.lz_tree_set_ez(t.h, int(ez), H), "lz_tree_set_ez")
        q = t.search_for(model, S, (1, H) if ez else ())
        with torch.cuda.device(dev):
            s = cabi.stream_ptr()
            obs = mz_tree._to_dev(policy_obs, torch.float32, dev)
            mask = mz_tree._to_dev(action_mask, torch.uint8, dev, (rows, A))
            tp = mz_tree._to_dev(np.asarray(to_play, np.int32), torch.int32, dev, (rows,))
            ta = mz_tree._to_dev(np.asarray(true_action, np.int32), torch.int32, dev, (rows,))
            pm = mz_tree._to_dev(np.asarray(policy_mask, np.uint8), torch.uint8, dev, (rows,))
            nz = mz_tree._to_dev(noises, torch.float32, dev, (rows, A)) if reanalyze_noise else None
            targets = torch.empty((N, L, A), dtype=torch.float64, device=dev)
            visits = torch.empty((N, L, A), dtype=torch.float64, device=dev)
            values = torch.empty((N, L), dtype=torch.float32, device=dev)
            nreuse = L - 1 if reuse_search else 0
            counts = torch.empty((nreuse, S), dtype=torch.int32, device=dev)
            head = (q, L, int(bool(reuse_search)), int(mini_infer_size), obs.data_ptr(), None, None, mask.data_ptr(),
                    tp.data_ptr(), ta.data_ptr(), pm.data_ptr(), cabi.ptr(nz), float(cfg.root_noise_weight))
            tail = (int(action_type != "fixed_action_space"), targets.data_ptr(), values.data_ptr(), visits.data_ptr(),
                    counts.data_ptr() if nreuse else None, s)
            if ez:
                cabi.check(t.lib.lz_rezero_reanalyze_ez(*head, *tail), "lz_rezero_reanalyze_ez")
            else:
                cabi.check(t.lib.lz_rezero_reanalyze(*head, int(mcts.deterministic), *tail), "lz_rezero_reanalyze")
            mcts.last_num_kernels = t.lib.lz_search_num_kernels(q)
            out, vis, val, cnt = targets.cpu().numpy(), visits.cpu().numpy(), values.cpu().numpy(), counts.cpu().numpy()
    finally:
        t.release()

    mcts.last_infer_count = cnt       # [L - 1, S] per reuse search and simulation: trees that needed the network
    rezero_write_back(child_visits, root_values, pos_in_game_segment_list, L, policy_mask, action_mask, vis, val)
    return out, rezero_reuse_stats(cnt, S)


# ---------------------------------------------------------------------------------------------- reward and value targets
def _section_bytes(sections):
    """Packs host arrays into one uint8 buffer, each section 8-byte aligned -> (buffer, byte offsets)."""
    offs, total = [], 0
    for a in sections:
        offs.append(total)
        total += max(8, (a.nbytes + 7) // 8 * 8)
    buf = np.zeros(total, np.uint8)
    for a, o in zip(sections, offs):
        buf[o:o + a.nbytes] = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    return buf, offs


def pack_value_targets(value_mask, pos_in_game_segment_list, rewards_list, game_segment_lens, td_steps_list, to_play_segment,
                       num_unroll_steps: int = 5, discount_factor: float = 0.997, env_type: str = "not_board_games",
                       efficientzero: bool = False, lstm_horizon_len: int = 5):
    """The host side of ``lz_value_targets``: the reference's ragged reward and to_play windows as flat padded arrays (vectorised
    NumPy, no per-element loop) and the discount powers, each computed with the reference's own expression.

    Returns ``(fields, tables)``: the scalar fields of ``lz_value_tables`` and its arrays by name (rewards f64 [N, W], rlen i32 [N],
    seglen i32 [N], td i32 [T], bootstrap f64 [T], value_mask f64 [T], powers f64 [P], to_play i32 [N, P + K1] or None).
    Raises ValueError for empty or mismatched inputs and for windows the reference would index past a list's end, TypeError for
    rewards that are not float32 or float64."""
    N = len(pos_in_game_segment_list)
    K1 = int(num_unroll_steps) + 1
    if N < 1 or K1 < 1:
        raise ValueError(f"compute_target_reward_value: no rows ({N} segments, num_unroll_steps = {num_unroll_steps})")
    T = N * K1
    if len(rewards_list) != N or len(game_segment_lens) != N or len(to_play_segment) != N:
        raise ValueError(f"compute_target_reward_value: {N} segments, but {len(rewards_list)} reward lists, {len(game_segment_lens)} "
                         f"segment lengths and {len(to_play_segment)} to_play lists")
    if len(value_mask) != T or len(td_steps_list) != T:
        raise ValueError(f"compute_target_reward_value: {N} segments x {K1} rows = {T}, got {len(value_mask)} value_mask and "
                         f"{len(td_steps_list)} td_steps entries")
    arrs = [np.asarray(r) for r in rewards_list]
    kinds = {(a.dtype, a.ndim) for a in arrs if a.size}
    dtypes = {d for d, _ in kinds}
    if not dtypes <= {np.dtype(np.float32), np.dtype(np.float64)} or len(dtypes) > 1:
        raise TypeError(f"compute_target_reward_value: rewards must all be float32 or all float64 (got {sorted(map(str, dtypes))})")
    if any(a.size and not (a.ndim == 1 or (a.ndim == 2 and a.shape[1] == 1)) for a in arrs) or len({n for _, n in kinds}) > 1:
        raise ValueError("compute_target_reward_value: every reward segment must be shaped (n,) or every one (n, 1)")
    fp32 = dtypes == {np.dtype(np.float32)}
    alias = bool(efficientzero) and {n for _, n in kinds} == {2}
    pos = np.asarray(pos_in_game_segment_list, np.int64)
    td = np.asarray(td_steps_list)
    if not np.issubdtype(td.dtype, np.integer) or (td < 0).any() or (pos < 0).any():
        raise ValueError("compute_target_reward_value: td_steps_list and pos_in_game_segment_list must be integers >= 0")
    P = max(1, int(td.max()))
    W = K1 - 1 + P
    lens = np.asarray([a.shape[0] for a in arrs], np.int64)
    flat = np.concatenate([a.reshape(-1) for a in arrs]).astype(np.float64) if lens.sum() else np.zeros(1)
    start = np.concatenate(([0], np.cumsum(lens)[:-1]))
    idx = pos[:, None] + np.arange(W)[None, :]
    valid = idx < lens[:, None]
    rewards = np.where(valid, flat[np.where(valid, start[:, None] + idx, 0)], 0.0)
    rlen = np.clip(lens - pos, 0, W).astype(np.int32)
    seglen = np.clip(np.asarray(game_segment_lens, np.int64) - pos, 0, K1).astype(np.int32)
    if efficientzero and (seglen > np.clip(lens - pos, 0, None)).any():
        raise ValueError("compute_target_reward_value: a segment's reward list is shorter than its game_segment_len (the reference "
                         "raises IndexError reading the value prefix)")
    d = discount_factor
    two_player = env_type == "board_games" and to_play_segment[0][0] in [1, 2]
    if two_player:       # game_buffer_muzero.py:520-527: the scalar power of every distinct td, as the reference writes it
        uniq, first = np.unique(td, return_index=True)
        fac = np.array([d ** td_steps_list[j] if int(td_steps_list[j]) % 2 == 0 else -d ** td_steps_list[j] for j in first],
                       np.float64)
        bootstrap = fac[np.searchsorted(uniq, td)]
    else:                # :529-531
        bootstrap = np.asarray(np.array([d]).repeat(T) ** td, np.float64)
    powers = np.array([d ** i for i in range(P)], np.float64)      # :545-552: a Python float to a Python int power
    to_play = None
    if two_player:
        tps = [np.asarray(x).reshape(-1) for x in to_play_segment]
        tlen = np.asarray([x.shape[0] for x in tps], np.int64)
        tflat = np.concatenate(tps).astype(np.int32)
        tstart = np.concatenate(([0], np.cumsum(tlen)[:-1]))
        tidx = np.concatenate((np.broadcast_to(np.arange(P), (N, P)), pos[:, None] + np.arange(K1)[None, :]), axis=1)
        tvalid = tidx < tlen[:, None]
        to_play = np.where(tvalid, tflat[np.where(tvalid, tstart[:, None] + tidx, 0)], 0).astype(np.int32)
        # the entries the window sums read: to_play_list[i] for i < the row's reward count, and to_play_list[base_index]
        k = np.arange(K1)[None, :]
        cnt = np.clip(np.minimum(k + td.reshape(N, K1), rlen[:, None]) - k, 0, None)
        base = np.zeros((N, K1), np.int64)
        if efficientzero:          # base_index moves at every horizon reset (horizon_id == row), after that row's sum
            r = np.arange(T).reshape(N, K1)
            last = (r - 1) // int(lstm_horizon_len) * int(lstm_horizon_len)
            seg0 = (np.arange(N) * K1)[:, None]
            base = np.where((r > 0) & (last >= seg0), last - seg0, 0)
        read = cnt > 0
        if (read & ((cnt > tlen[:, None]) | (pos[:, None] + base >= tlen[:, None]))).any():
            raise ValueError("compute_target_reward_value: a to_play list is shorter than the entries the two-player window sums "
                             "read (the reference raises IndexError)")
    fields = dict(N=N, K1=K1, W=W, P=P, value_prefix=int(bool(efficientzero)), fp32=int(fp32), two_player=int(two_player),
                  horizon=int(lstm_horizon_len), alias_prefix=int(alias))
    tables = dict(rewards=rewards, rlen=rlen, seglen=seglen, td=td.astype(np.int32), bootstrap=bootstrap,
                  value_mask=np.asarray(value_mask, np.float64), powers=powers, to_play=to_play)
    return fields, tables


_TABLE_ORDER = ("rewards", "rlen", "seglen", "td", "bootstrap", "value_mask", "powers", "to_play")


def compute_target_reward_value(
        model, value_obs, value_mask, pos_in_game_segment_list: Sequence[int], rewards_list, game_segment_lens,
        td_steps_list, to_play_segment, num_unroll_steps: int = 5, discount_factor: float = 0.997,
        env_type: str = "not_board_games", efficientzero: bool = False, lstm_horizon_len: int = 5, use_root_value: bool = False,
        mcts=None, action_mask=None, to_play=None, reanalyze_noise: bool = True, root_noise_weight: Optional[float] = None,
        root_dirichlet_alpha: Optional[float] = None, noises: Optional[np.ndarray] = None, mini_infer_size: int = 10240,
        device: bool = False, return_values: bool = False):
    """Mirror of ``MuZeroGameBuffer._compute_target_reward_value`` (lzero/mcts/buffer/game_buffer_muzero.py:467-575) and, with
    ``efficientzero=True``, ``EfficientZeroGameBuffer._compute_target_reward_value`` (game_buffer_efficientzero.py:167-323), as
    one device call (``lz_value_targets`` / ``lz_value_targets_root``).  The ReZero and Gumbel MuZero buffers inherit these.

    The arguments are the fields of the reference's ``reward_value_context``: value_obs [N * (K + 1), ...] (host or device; row =
    segment * (K + 1) + position), value_mask, pos_in_game_segment_list [N], rewards_list (per segment the reward segment,
    float32 or float64, shaped (n,) or (n, 1)), game_segment_lens, td_steps_list [N * (K + 1)], to_play_segment; and the config
    values.  EfficientZero with ``use_root_value`` also takes ``mcts`` (an EfficientZeroMCTSCtree: num_simulations, pb_c, tie
    rule), ``action_mask`` [N * (K + 1), A] and ``to_play`` [N * (K + 1)] as ``_preprocess_to_play_and_action_mask`` returns
    them, and ``noises`` [N * (K + 1), A] in legal order (drawn with np.random.dirichlet like the reference when None).

    Returns ``(batch_rewards, batch_target_values)``: float64 [N, K + 1] each (value prefixes in place of rewards for
    EfficientZero, whose object arrays hold the same numbers), bit for bit the reference's given the same fp32 values.  With
    ``device=True`` they are CUDA float64 tensors and nothing waits for the device.  ``return_values=True`` appends the fp32
    bootstrap values [N * (K + 1)] (initial_inference's value scalars, or the searched root values)."""
    from . import cabi, mz_tree
    from .efficientzero_model import EfficientZeroModel
    from .efficientzero_model_mlp import EfficientZeroModelMLP
    from .mcts_ctree import EfficientZeroMCTSCtree
    from .muzero_model import MuZeroModel
    from .muzero_model_mlp import MuZeroModelMLP

    if use_root_value and not efficientzero:
        raise ValueError("compute_target_reward_value: use_root_value=True is not available for the MuZero buffer: the reference "
                         "reads np.array(root_values) from a list _prepare_reward_value_context never fills, and the product with "
                         "the td discounts fails with a broadcast error")
    fields, tables = pack_value_targets(value_mask, pos_in_game_segment_list, rewards_list, game_segment_lens, td_steps_list,
                                        to_play_segment, num_unroll_steps, discount_factor, env_type, efficientzero,
                                        lstm_horizon_len)
    N, K1 = fields["N"], fields["K1"]
    T = N * K1
    if value_obs.shape[0] != T:
        raise ValueError(f"compute_target_reward_value: {T} rows, got value_obs {tuple(value_obs.shape)}")
    ez_model = isinstance(model, (EfficientZeroModel, EfficientZeroModelMLP))
    if not isinstance(model, (MuZeroModel, MuZeroModelMLP, EfficientZeroModelMLP)):
        raise TypeError(f"compute_target_reward_value: {type(model).__name__} has no CUDA initial_inference (MuZeroModel, "
                        "MuZeroModelMLP, EfficientZeroModel or EfficientZeroModelMLP)")
    if bool(efficientzero) != ez_model:
        raise TypeError(f"compute_target_reward_value: the {'EfficientZero' if efficientzero else 'MuZero'} buffer's targets need "
                        f"{'an EfficientZero' if efficientzero else 'a MuZero'} model, not a {type(model).__name__}")
    sections = [tables[k] for k in _TABLE_ORDER if tables[k] is not None]
    if use_root_value:
        if not isinstance(mcts, EfficientZeroMCTSCtree):
            raise TypeError(f"compute_target_reward_value: the root-value search needs an EfficientZeroMCTSCtree, not a "
                            f"{type(mcts).__name__}")
        if action_mask is None or to_play is None:
            raise ValueError("compute_target_reward_value: use_root_value needs action_mask and to_play")
        cfg = mcts._cfg
        action_mask = np.asarray(action_mask)
        A = model.action_space_size
        if action_mask.shape != (T, A) or len(to_play) != T:
            raise ValueError(f"compute_target_reward_value: {T} rows of {A} actions, got action_mask {action_mask.shape} and "
                             f"{len(to_play)} to_play")
        if noises is None:        # game_buffer_efficientzero.py:223-226
            alpha = cfg.root_dirichlet_alpha if root_dirichlet_alpha is None else root_dirichlet_alpha
            noises = np.stack([np.random.dirichlet([alpha] * A).astype(np.float32) for _ in range(T)])
        sections += [np.ascontiguousarray(action_mask, np.uint8), np.asarray(to_play, np.int32)]
        if reanalyze_noise:
            sections.append(np.ascontiguousarray(noises, np.float32).reshape(T, A))
    dev = model.device
    buf, offs = _section_bytes(sections)
    with torch.cuda.device(dev):
        s = cabi.stream_ptr()
        obs = mz_tree._to_dev(value_obs, torch.float32, dev)
        d_buf = torch.from_numpy(buf).to(dev, non_blocking=True)
        ptrs = [d_buf.data_ptr() + o for o in offs]
        named = dict(zip([k for k in _TABLE_ORDER if tables[k] is not None], ptrs))     # the tables, then the root-search inputs
        tab = cabi.ValueTables(**fields, **named)
        out = torch.empty((2, N, K1), dtype=torch.float64, device=dev)
        values = torch.empty(T, dtype=torch.float32, device=dev)
        if not use_root_value:
            cabi.check(model._lib.lz_value_targets(model._h, tab, int(mini_infer_size), obs.data_ptr(), values.data_ptr(),
                                                   out[0].data_ptr(), out[1].data_ptr(), s), "lz_value_targets")
        else:
            S, H = int(cfg.num_simulations), int(cfg.lstm_horizon_len)
            rest = ptrs[len(named):]        # action mask, to_play, noise
            mask_p, tp_p = rest[0], rest[1]
            nz_p = rest[2] if reanalyze_noise else None
            w = float(cfg.root_noise_weight if root_noise_weight is None else root_noise_weight)
            t = mz_tree.acquire_tree(dev, T, A, S)
            try:
                t.set_params(*mcts._params())
                cabi.check(t.lib.lz_tree_set_gumbel(t.h, 0, 0), "lz_tree_set_gumbel")     # a pooled tree a Gumbel collect left behind
                cabi.check(t.lib.lz_tree_set_ez(t.h, 1, H), "lz_tree_set_ez")
                q = t.search_for(model, S, (1, H))
                cabi.check(t.lib.lz_value_targets_root(q, tab, int(mini_infer_size), obs.data_ptr(), mask_p, tp_p, nz_p, w,
                                                       int(mcts.deterministic), values.data_ptr(), out[0].data_ptr(),
                                                       out[1].data_ptr(), s), "lz_value_targets_root")
                mcts.last_num_kernels = t.lib.lz_search_num_kernels(q)
            finally:
                t.release()
        if device:
            res = (out[0], out[1])
        else:
            host = out.cpu().numpy()
            res = (host[0], host[1])
    if return_values:
        return res + (values,)
    return res
