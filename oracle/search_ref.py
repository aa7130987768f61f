"""oracle/search_ref.py -- restatement of the reference's per-simulation host loop
``MuZeroMCTSCtree.search`` (lzero/mcts/tree_search/mcts_ctree.py:267-368) and of the part of
``MuZeroPolicy._forward_collect`` that feeds it (lzero/policy/muzero.py:749-779).

TEST INFRASTRUCTURE ONLY.  `lzero.mcts.tree_search.mcts_ctree` cannot be imported here (it pulls
lzero.policy -> ding/easydict, absent), so the ~60-line loop is restated; the tree module it drives
is either the compiled UNMODIFIED reference (oracle/_ref/mz_tree, preferred) or oracle/ctree_port.

Differences from the reference loop, all deliberate and stated in DESIGN.md:
  * ``deterministic=True`` is passed to batch_traverse (the parity contract, SURVEY.md s.0 fact 2);
  * ``duplicate_inference`` reproduces the reference's discarded first recurrent_inference call
    (mcts_ctree.py:338 then :345) when timing the reference arm; parity runs set it False;
  * an optional ``recorder`` captures per-simulation (ix, iy, last_action, reward, value, logits)
    for replay-mode tree parity tests.
"""
import copy
import os
import sys

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))


def load_tree_module(prefer_ref: bool = True, name: str = "mz_tree"):
    """Returns (module, kind) with kind in {'reference', 'port'}.  name: 'mz_tree' (MuZero) or 'ez_tree' (EfficientZero;
    the compiled reference is linked with the rand() == 0 shim, see oracle/build_ref.py)."""
    if prefer_ref:
        ref_dir = os.path.join(_HERE, "_ref")
        if os.path.isdir(ref_dir) and any(f.startswith(name) for f in os.listdir(ref_dir)):
            if ref_dir not in sys.path:
                sys.path.insert(0, ref_dir)
            try:
                return __import__(name), "reference"
            except ImportError:
                pass
    if name == "ez_tree":
        from oracle import ctree_port_ez
        return ctree_port_ez, "port"
    from oracle import ctree_port
    return ctree_port, "port"


class SearchRef:
    def __init__(self, tree_module, num_simulations=50, pb_c_base=19652, pb_c_init=1.25,
                 discount_factor=0.997, value_delta_max=0.01, env_type="not_board_games",
                 value_support_range=(-300., 301., 1.), reward_support_range=(-300., 301., 1.),
                 deterministic=True, duplicate_inference=False):
        from oracle.model_ref import DiscreteSupport, InverseScalarTransform
        self.tree = tree_module
        self.num_simulations = num_simulations
        self.pb_c_base, self.pb_c_init = pb_c_base, pb_c_init
        self.discount_factor, self.value_delta_max = discount_factor, value_delta_max
        self.env_type = env_type
        self.deterministic = deterministic
        self.duplicate_inference = duplicate_inference
        self.value_inv = InverseScalarTransform(DiscreteSupport(*value_support_range))
        self.reward_inv = InverseScalarTransform(DiscreteSupport(*reward_support_range))

    def roots(self, n, legal_actions, action_space_size=None):
        if "ctree_port" in self.tree.__name__:
            return self.tree.Roots(n, legal_actions, action_space_size=action_space_size,
                                   max_sims=self.num_simulations)
        return self.tree.Roots(n, legal_actions)

    def search(self, roots, model, latent_state_roots, to_play_batch, recorder=None):
        """mcts_ctree.py:281-368.  latent_state_roots: np.ndarray [B,C,H,W]."""
        tree = self.tree
        with torch.no_grad():
            if model is not None:
                model.eval()
            batch_size = roots.num
            latent_pool = [latent_state_roots]
            mm = tree.MinMaxStatsList(batch_size)
            mm.set_delta(self.value_delta_max)
            for simulation_index in range(self.num_simulations):
                results = tree.ResultsWrapper(batch_size)
                tp_arg = to_play_batch if self.env_type == "not_board_games" else copy.deepcopy(to_play_batch)
                ix_l, iy_l, last_actions, virtual_to_play = tree.batch_traverse(
                    roots, self.pb_c_base, self.pb_c_init, self.discount_factor, mm, results,
                    list(tp_arg), self.deterministic)
                latent_states = [latent_pool[ix][iy] for ix, iy in zip(ix_l, iy_l)]
                latent_states = torch.from_numpy(np.asarray(latent_states))
                actions = torch.from_numpy(np.asarray(last_actions)).long()
                if self.duplicate_inference:
                    model.recurrent_inference(latent_states, actions)   # mcts_ctree.py:338 (discarded)
                out = model.recurrent_inference(latent_states, actions)
                latent_pool.append(out.latent_state.detach().cpu().numpy())
                value = self.value_inv(out.value).detach().cpu().numpy()
                reward = self.reward_inv(out.reward).detach().cpu().numpy()
                reward_batch = reward.reshape(-1).tolist()
                value_batch = value.reshape(-1).tolist()
                policy_logits_batch = out.policy_logits.detach().cpu().numpy().tolist()
                if recorder is not None:
                    recorder.append(dict(ix=list(ix_l), iy=list(iy_l), last_action=list(last_actions),
                                         search_len=list(results.get_search_len()),
                                         reward=list(reward_batch), value=list(value_batch),
                                         policy=[list(p) for p in policy_logits_batch]))
                tree.batch_backpropagate(simulation_index + 1, self.discount_factor, reward_batch,
                                         value_batch, policy_logits_batch, mm, results, virtual_to_play)
        return latent_pool


def unizero_search_ref(search: SearchRef, roots, model, latent_state_roots, to_play_batch, timestep=None, task_id=None):
    """``UniZeroMCTSCtree.search`` (mcts_ctree.py:77-208) restated on the same tree module: the MuZero tree unchanged, the
    world model called as ``model.recurrent_inference(state_action_history, simulation_index, search_depth[, timestep])``
    (:160-176), returns ``first_action_latent_map`` (:90, 183-189).  TEST INFRASTRUCTURE ONLY."""
    tree = search.tree
    with torch.no_grad():
        if hasattr(model, "eval"):
            model.eval()
        batch_size = roots.num
        first_action_latent_map = {env_id: {} for env_id in range(batch_size)}
        latent_pool = [latent_state_roots]
        mm = tree.MinMaxStatsList(batch_size)
        mm.set_delta(search.value_delta_max)
        state_action_history = []
        for simulation_index in range(search.num_simulations):
            results = tree.ResultsWrapper(batch_size)
            tp_arg = to_play_batch if search.env_type == "not_board_games" else copy.deepcopy(to_play_batch)
            ix_l, iy_l, last_actions, virtual_to_play = tree.batch_traverse(
                roots, search.pb_c_base, search.pb_c_init, search.discount_factor, mm, results, list(tp_arg), search.deterministic)
            latent_states = torch.from_numpy(np.asarray([latent_pool[ix][iy] for ix, iy in zip(ix_l, iy_l)]))
            actions = torch.from_numpy(np.asarray(last_actions)).long()
            state_action_history.append((latent_states.detach().cpu().numpy(), actions))
            search_depth = results.get_search_len()
            if timestep is None:
                if task_id is not None:
                    out = model.recurrent_inference(state_action_history, simulation_index, search_depth, task_id=task_id)
                else:
                    out = model.recurrent_inference(state_action_history, simulation_index, search_depth)
            else:
                if task_id is not None:
                    out = model.recurrent_inference(state_action_history, simulation_index, search_depth, task_id=task_id)
                else:
                    out = model.recurrent_inference(state_action_history, simulation_index, search_depth, timestep)
            latent = out.latent_state.detach().cpu().numpy()
            value = search.value_inv(out.value).detach().cpu().numpy()
            reward = search.reward_inv(out.reward).detach().cpu().numpy()
            for env_id in range(batch_size):
                if search_depth[env_id] == 1 and int(actions[env_id].item()) not in first_action_latent_map[env_id]:
                    first_action_latent_map[env_id][int(actions[env_id].item())] = latent[env_id]
            latent_pool.append(latent)
            tree.batch_backpropagate(simulation_index + 1, search.discount_factor, reward.reshape(-1).tolist(),
                                     value.reshape(-1).tolist(), out.policy_logits.detach().cpu().numpy().tolist(), mm, results,
                                     virtual_to_play)
    return first_action_latent_map


def collect_step_ref(search: SearchRef, model, obs, action_mask, to_play, noise_weight=0.25,
                     noises=None, recorder=None):
    """The search-feeding part of MuZeroPolicy._forward_collect (policy/muzero.py:749-779)."""
    with torch.no_grad():
        model.eval()
        out = model.initial_inference(obs)
        pred_values = search.value_inv(out.value).detach().cpu().numpy()
        latent_roots = out.latent_state.detach().cpu().numpy()
        policy_logits = out.policy_logits.detach().cpu().numpy()
    B = obs.shape[0]
    legal_actions = [np.nonzero(action_mask[j])[0].tolist() for j in range(B)]
    roots = search.roots(B, legal_actions, action_space_size=policy_logits.shape[1])
    if noises is not None:
        roots.prepare(noise_weight, noises, [0.] * B, policy_logits.tolist(), list(to_play))
    else:
        roots.prepare_no_noise([0.] * B, policy_logits.tolist(), list(to_play))
    search.search(roots, model, latent_roots, list(to_play), recorder=recorder)
    return dict(distributions=roots.get_distributions(), values=roots.get_values(),
                pred_values=pred_values, policy_logits=policy_logits, latent_roots=latent_roots,
                roots=roots)


class SearchRefEZ(SearchRef):
    """``EfficientZeroMCTSCtree.search`` (mcts_ctree.py:729-876) restated: value prefixes, the LSTM state pools and the
    reset of that state every ``lstm_horizon_len`` steps of depth (:856-863).  No duplicate inference in this driver."""

    def __init__(self, tree_module, lstm_horizon_len=5, **kw):
        kw.pop("deterministic", None)
        super().__init__(tree_module, **kw)
        self.lstm_horizon_len = lstm_horizon_len

    def search(self, roots, model, latent_state_roots, reward_hidden_state_roots, to_play_batch, recorder=None):
        tree = self.tree
        with torch.no_grad():
            if model is not None:
                model.eval()
            batch_size = roots.num
            latent_pool = [latent_state_roots]
            pool0 = [reward_hidden_state_roots[0]]          # "reward_hidden_state_c_batch" in the reference = tuple element 0
            pool1 = [reward_hidden_state_roots[1]]
            mm = tree.MinMaxStatsList(batch_size)
            mm.set_delta(self.value_delta_max)
            for simulation_index in range(self.num_simulations):
                results = tree.ResultsWrapper(batch_size)
                tp_arg = to_play_batch if self.env_type == "not_board_games" else copy.deepcopy(to_play_batch)
                ix_l, iy_l, last_actions, virtual_to_play = tree.batch_traverse(
                    roots, self.pb_c_base, self.pb_c_init, self.discount_factor, mm, results, list(tp_arg))
                search_lens = results.get_search_len()
                reset_idx = (np.array(search_lens) % self.lstm_horizon_len == 0)
                latent_states = torch.from_numpy(np.asarray([latent_pool[ix][iy] for ix, iy in zip(ix_l, iy_l)]))
                s0 = torch.from_numpy(np.asarray([pool0[ix][0][iy] for ix, iy in zip(ix_l, iy_l)])).unsqueeze(0)
                s1 = torch.from_numpy(np.asarray([pool1[ix][0][iy] for ix, iy in zip(ix_l, iy_l)])).unsqueeze(0)
                actions = torch.from_numpy(np.asarray(last_actions)).long()
                out = model.recurrent_inference(latent_states, (s0, s1), actions)
                latent_pool.append(out.latent_state.detach().cpu().numpy())
                value = self.value_inv(out.value).detach().cpu().numpy()
                vp = self.value_inv(out.value_prefix).detach().cpu().numpy()      # :840-842 (value transform handle)
                n0 = out.reward_hidden_state[0].detach().cpu().numpy()
                n1 = out.reward_hidden_state[1].detach().cpu().numpy()
                n0[:, reset_idx, :] = 0
                n1[:, reset_idx, :] = 0
                pool0.append(n0)
                pool1.append(n1)
                vp_batch = vp.reshape(-1).tolist()
                value_batch = value.reshape(-1).tolist()
                policy_logits_batch = out.policy_logits.detach().cpu().numpy().tolist()
                is_reset_list = reset_idx.astype(np.int32).tolist()
                if recorder is not None:
                    recorder.append(dict(ix=list(ix_l), iy=list(iy_l), last_action=list(last_actions),
                                         search_len=list(search_lens), is_reset=is_reset_list,
                                         reward=list(vp_batch), value=list(value_batch),
                                         policy=[list(p) for p in policy_logits_batch]))
                tree.batch_backpropagate(simulation_index + 1, self.discount_factor, vp_batch, value_batch,
                                         policy_logits_batch, mm, results, is_reset_list, virtual_to_play)
        return latent_pool


def collect_step_ref_ez(search: SearchRefEZ, model, obs, action_mask, to_play, noise_weight=0.25, noises=None, recorder=None):
    """The search-feeding part of EfficientZeroPolicy._forward_collect (policy/efficientzero.py:575-610)."""
    with torch.no_grad():
        model.eval()
        out = model.initial_inference(obs)
        pred_values = search.value_inv(out.value).detach().cpu().numpy()
        latent_roots = out.latent_state.detach().cpu().numpy()
        hidden_roots = (out.reward_hidden_state[0].detach().cpu().numpy(), out.reward_hidden_state[1].detach().cpu().numpy())
        policy_logits = out.policy_logits.detach().cpu().numpy()
    B = obs.shape[0]
    legal_actions = [np.nonzero(action_mask[j])[0].tolist() for j in range(B)]
    roots = search.roots(B, legal_actions, action_space_size=policy_logits.shape[1])
    if noises is not None:
        roots.prepare(noise_weight, noises, [0.] * B, policy_logits.tolist(), list(to_play))
    else:
        roots.prepare_no_noise([0.] * B, policy_logits.tolist(), list(to_play))
    search.search(roots, model, latent_roots, hidden_roots, list(to_play), recorder=recorder)
    return dict(distributions=roots.get_distributions(), values=roots.get_values(), pred_values=pred_values,
                policy_logits=policy_logits, latent_roots=latent_roots, hidden_roots=hidden_roots, roots=roots)
