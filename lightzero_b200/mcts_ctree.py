"""Mirror of ``lzero.mcts.tree_search.mcts_ctree.MuZeroMCTSCtree`` (mcts_ctree.py:211-368): same
class-level ``config``, ``default_config()``, ``__init__(cfg)``, ``roots(n, legal_actions)`` and
``search(roots, model, latent_state_roots, to_play_batch, task_id=None)``.

``search`` has two execution modes, both entirely on the GPU:
  * fused (``model`` is a ``lightzero_b200.MuZeroModel``): the whole num_simulations loop is one CUDA
    graph launch (``lz_search_run``) -- zero host<->device synchronisations inside the search;
  * step-wise (any other object with ``recurrent_inference``, e.g. the user's own torch module on
    CUDA): the device trees are driven one simulation at a time around the caller's model; the tree
    hands the gather indices to torch on device, so this mode also never syncs with the host.

Parity contract: ``deterministic=True`` reproduces the reference C++ ctree bit for bit (first legal
action attaining the maximum, cnode.cpp:592); the reference's default mode seeds rand() from the wall
clock on every traverse (cnode.cpp:770, utils.cpp:12-26) and is not reproducible by construction, so
``deterministic=False`` draws from the same tie list with a counter-based device RNG instead.
"""
import copy
from typing import Any, List, Optional, Union

import numpy as np
import torch

from . import cabi, ez_tree, gmz_tree, mz_tree, stochastic_mz_tree
from .model_base import LzModel, StochasticLzModel
from .scaling_transform import DiscreteSupport, InverseScalarTransform


def _dev_f32(x, dev):
    """A latent or hidden-state batch (np.ndarray or tensor) as a contiguous float32 tensor on dev."""
    if isinstance(x, torch.Tensor):
        return x.to(dev, torch.float32, non_blocking=True).contiguous()
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(dev, non_blocking=True)


def _value_prefix_model(model):
    """True for a lightzero_b200 EfficientZero model, False for a MuZero one, None for any other object (step-wise)."""
    return model.value_prefix if isinstance(model, LzModel) else None


class ConfigDict(dict):
    """Minimal attribute dict (the reference uses easydict.EasyDict, not installed here)."""

    def __init__(self, d=None, **kw):
        super().__init__()
        for k, v in dict(d or {}, **kw).items():
            self[k] = v

    def __setitem__(self, k, v):
        if isinstance(v, dict) and not isinstance(v, ConfigDict):
            v = ConfigDict(v)
        super().__setitem__(k, v)

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v

    def update(self, other=None, **kw):
        for k, v in dict(other or {}, **kw).items():
            self[k] = v


class MuZeroMCTSCtree(object):
    # mcts_ctree.py:220-232
    config = dict(
        root_dirichlet_alpha=0.3,
        root_noise_weight=0.25,
        pb_c_base=19652,
        pb_c_init=1.25,
        value_delta_max=0.01,
        env_type='not_board_games',
    )
    # extension: tie-breaking mode (the reference MuZero search passes no flag, i.e. False)
    deterministic_default = False

    @classmethod
    def default_config(cls) -> ConfigDict:
        cfg = ConfigDict(copy.deepcopy(cls.config))
        cfg.cfg_type = cls.__name__ + 'Dict'
        return cfg

    def __init__(self, cfg=None) -> None:
        default_config = self.default_config()
        default_config.update(cfg or {})
        self._cfg = default_config
        self._cfg.setdefault("num_simulations", 50)
        self._cfg.setdefault("discount_factor", 0.997)
        self._cfg.setdefault("device", "cuda")
        self.deterministic = bool(self._cfg.get("deterministic", self.deterministic_default))
        self._inv = self._inv_reward = None    # lazily: InverseScalarTransforms for the step-wise mode (mcts_ctree.py:249-253)

    @classmethod
    def roots(cls, active_collect_env_num: int, legal_actions: List[Any]) -> "mz_tree.Roots":
        """mcts_ctree.py:255-265"""
        return mz_tree.Roots(active_collect_env_num, legal_actions)

    def _params(self):
        c = self._cfg
        return (c.pb_c_base, c.pb_c_init, c.discount_factor, c.value_delta_max)

    def search(self, roots: "mz_tree.Roots", model, latent_state_roots, to_play_batch: Union[int, List[Any]],
               task_id: Optional[int] = None) -> None:
        """mcts_ctree.py:267-368.  ``latent_state_roots``: np.ndarray or CUDA tensor [B,C,H,W]."""
        family = _value_prefix_model(model)
        if family:
            raise TypeError(f"MuZeroMCTSCtree.search: an {type(model).__name__} needs EfficientZeroMCTSCtree")
        S = int(self._cfg.num_simulations)
        roots._materialize(S, self._params(), self.deterministic)     # reset + prepare on device, MinMax stats fresh (:291-292)
        lat = _dev_f32(latent_state_roots, roots.device)
        if family is None:
            self._search_stepwise(roots, model, S, lat)
        else:
            self._run_fused(roots, model, S, (), "lz_search_run", lat.data_ptr(), int(self.deterministic))

    def search_with_reuse(self, roots: "mz_tree.Roots", model, latent_state_roots, to_play_batch: Union[int, List[Any]],
                          true_action_list=None, reuse_value_list=None):
        """mcts_ctree.py:370-468 (ReZero): the root child of ``true_action`` is scored with the stored ``reuse_value`` and the
        descent stops there.  Returns ``(length, average_infer)`` like the reference: how many trees needed the network in
        the last simulation and on average.  One CUDA graph with a ``lightzero_b200`` model."""
        if _value_prefix_model(model) is not False:
            raise NotImplementedError("search_with_reuse is fused only: pass a lightzero_b200 MuZeroModel / MuZeroModelMLP "
                                      "(or drive mz_tree.batch_traverse_with_reuse / batch_backpropagate_with_reuse yourself)")
        S = int(self._cfg.num_simulations)
        return self._run_with_reuse(roots, model, S, (), (_dev_f32(latent_state_roots, roots.device), None, None),
                                    true_action_list, reuse_value_list)

    def _run_with_reuse(self, roots, model, S, mode, roots_state, true_action_list, reuse_value_list):
        """The fused search_with_reuse (lz_search_run_with_reuse) of either tree family from ``roots_state`` = (latents, LSTM
        h, LSTM c; None for MuZero); returns the reference's ``(length, average_infer)``."""
        roots._materialize(S, self._params(), self.deterministic)     # the reference draws rand() % len(ties) (cnode.cpp:610-640)
        dev, B = roots.device, roots.num
        ta = mz_tree._to_dev(true_action_list, torch.int32, dev, (B,))
        rv = mz_tree._to_dev(reuse_value_list, torch.float32, dev, (B,))
        counts = torch.empty(S, dtype=torch.int32, device=dev)
        self._run_fused(roots, model, S, mode, "lz_search_run_with_reuse", *(cabi.ptr(x) for x in roots_state), ta.data_ptr(),
                        rv.data_ptr(), counts.data_ptr())
        c = counts.cpu().numpy()
        return int(c[-1]), float(c.sum()) / S

    def _run_fused(self, roots, model, S, mode, fn, *args):
        """One fused search on the roots' tree: the lz_search handle of (model, S, mode), then the library call
        ``fn(handle, *args, stream)``; records the kernel count of its search graph in ``last_num_kernels``."""
        t = roots._tree
        q = t.search_for(model, S, mode)
        with torch.cuda.device(roots.device):
            cabi.check(getattr(t.lib, fn)(q, *args, cabi.stream_ptr()), fn)
        self.last_num_kernels = t.lib.lz_search_num_kernels(q)

    def _make_inverse_transforms(self, dev):
        """mcts_ctree.py:249-253: separate value and reward supports, both categorical (the only representation the CUDA
        transform implements)."""
        if self._inv is not None:
            return
        m = self._cfg.get("model", None)

        def rng(key):
            return tuple(m[key]) if m is not None and key in m else (-300., 301., 1.)
        if m is not None and not m.get("categorical_distribution", True):
            raise NotImplementedError("model.categorical_distribution=False: only the categorical (support) representation is implemented")
        self._inv = InverseScalarTransform(DiscreteSupport(*rng("value_support_range"), device=dev))
        vr, rr = rng("value_support_range"), rng("reward_support_range")
        self._inv_reward = self._inv if vr == rr else InverseScalarTransform(DiscreteSupport(*rr, device=dev))

    def _search_stepwise(self, roots, model, S, *states):
        """The search driven one simulation at a time around any model object, on the descent and back-up of the tree's mode:
        per simulation one descent, the model call ``_recurrent`` on the leaves it reached and one back-up.  ``states``: the
        roots' latents, then an EfficientZero search's LSTM state h and c [B, lstm_hidden_size]; each has a pool of S + 1
        slots, slot sim + 1 written by simulation sim.  An EfficientZero tree also hands the leaves' is_reset to the model
        call and the back-up."""
        t, dev, B = roots._tree, roots.device, roots.num
        self._make_inverse_transforms(dev)
        pools = [torch.empty((S + 1,) + tuple(x.shape), device=dev, dtype=torch.float32) for x in states]
        for pool, x in zip(pools, states):
            pool[0] = x
        rows = torch.arange(B, device=dev)
        reset = torch.empty(B, dtype=torch.int32, device=dev) if len(states) > 1 else None
        with torch.no_grad(), torch.cuda.device(dev):
            if hasattr(model, "eval"):
                model.eval()
            for sim in range(S):
                cabi.check(t.lib.lz_tree_traverse(t.h, int(self.deterministic), None, None, t.ix.data_ptr(), t.iy.data_ptr(),
                                                  t.action.data_ptr(), t.search_len.data_ptr(), t.vtp.data_ptr(),
                                                  cabi.ptr(reset), cabi.stream_ptr()), "lz_tree_traverse")
                ix = t.ix.long()
                new_states, reward, value, logits = self._recurrent(model, t, [pool[ix, rows] for pool in pools],  # :323-324
                                                                    t.action.long(), reset)
                for pool, x in zip(pools, new_states):
                    pool[sim + 1] = x
                value = self._inv(value).reshape(-1).contiguous()            # :349 (value support)
                reward = self._inv_reward(reward).reshape(-1).contiguous()   # :350 (reward support)
                pol = logits.to(torch.float32).contiguous()
                cabi.check(t.lib.lz_tree_backpropagate(t.h, sim + 1, reward.data_ptr(), value.data_ptr(), pol.data_ptr(), None,
                                                       None, cabi.ptr(reset), None, cabi.stream_ptr()), "lz_tree_backpropagate")

    def _recurrent(self, model, t, states, action, reset):
        """One simulation's model call on the gathered states of the leaves; returns (their new states, reward logits, value
        logits, policy logits), every row of the batch."""
        out = model.recurrent_inference(states[0], action)
        return (out.latent_state,), out.reward, out.value, out.policy_logits


class EfficientZeroMCTSCtree(MuZeroMCTSCtree):
    """Mirror of ``lzero.mcts.tree_search.mcts_ctree.EfficientZeroMCTSCtree`` (mcts_ctree.py:671-876): same config keys
    (+ ``lstm_horizon_len``, read at :857), ``roots(n, legal_actions)`` and
    ``search(roots, model, latent_state_roots, reward_hidden_state_roots, to_play_batch)``.

    With a ``lightzero_b200.EfficientZeroModel`` or ``EfficientZeroModelMLP`` the whole loop is one CUDA-graph launch (``lz_search_run_ez``): per
    simulation the descent (which also derives ``is_reset = search_len % lstm_horizon_len == 0``, :856-861), the conv
    trunk + prediction heads, the LSTM value-prefix head over all roots, and the back-up.  Any other model object is
    driven step-wise around the device trees.  Ties: first maximum (the reference's ``rand() % len(ties)`` with
    ``rand() == 0``; the EfficientZero tree has no deterministic switch, cnode.cpp:691)."""

    def __init__(self, cfg=None) -> None:
        super().__init__(cfg)
        self._cfg.setdefault("lstm_horizon_len", 5)
        # the reference tree has no deterministic switch (always rand() % len(ties)); here first maximum is the default (what the
        # parity tests pin) and ``deterministic=False`` in the config selects the uniform draw (lz_tree_set_tiebreak)
        self.deterministic = bool(self._cfg.get("deterministic", True))

    @classmethod
    def roots(cls, active_collect_env_num: int, legal_actions: List[Any]) -> "ez_tree.Roots":
        """mcts_ctree.py:715-727"""
        return ez_tree.Roots(active_collect_env_num, legal_actions)

    def search(self, roots: "ez_tree.Roots", model, latent_state_roots, reward_hidden_state_roots,
               to_play_batch: Union[int, List[Any]]) -> None:
        S, H = int(self._cfg.num_simulations), int(self._cfg.lstm_horizon_len)
        assert H > 0                                   # mcts_ctree.py:857
        roots._ez, roots._lstm_horizon = True, H
        roots._materialize(S, self._params(), self.deterministic)
        lat, h0, h1 = self._ez_inputs(roots, latent_state_roots, reward_hidden_state_roots)
        if not _value_prefix_model(model):
            self._search_stepwise(roots, model, S, lat, h0, h1)
        else:
            self._run_fused(roots, model, S, (1, H), "lz_search_run_ez", lat.data_ptr(), h0.data_ptr(), h1.data_ptr())

    def search_with_reuse(self, roots: "ez_tree.Roots", model, latent_state_roots, reward_hidden_state_roots,
                          to_play_batch: Union[int, List[Any]], true_action_list=None, reuse_value_list=None):
        """mcts_ctree.py:878-1003 (ReZero on the EfficientZero trees) as one CUDA graph (``lz_search_run_with_reuse``); returns
        ``(length, average_infer)`` like the reference.  Fused only: other model objects drive
        ``ez_tree.batch_traverse_with_reuse`` / ``batch_backpropagate_with_reuse`` themselves."""
        S, H = int(self._cfg.num_simulations), int(self._cfg.lstm_horizon_len)
        assert H > 0
        if not _value_prefix_model(model):
            raise NotImplementedError("EfficientZeroMCTSCtree.search_with_reuse is fused only: pass a lightzero_b200 EfficientZeroModel "
                                      "or EfficientZeroModelMLP")
        roots._ez, roots._lstm_horizon = True, H
        return self._run_with_reuse(roots, model, S, (1, H), self._ez_inputs(roots, latent_state_roots, reward_hidden_state_roots),
                                    true_action_list, reuse_value_list)

    @staticmethod
    def _ez_inputs(roots, latent_state_roots, reward_hidden_state_roots):
        """The roots' latents and LSTM state (h, c) as float32 on the device, the state as [B, lstm_hidden_size]."""
        dev, B = roots.device, roots.num
        return (_dev_f32(latent_state_roots, dev), _dev_f32(reward_hidden_state_roots[0], dev).reshape(B, -1),
                _dev_f32(reward_hidden_state_roots[1], dev).reshape(B, -1))

    def _recurrent(self, model, t, states, action, reset):
        """mcts_ctree.py:819-863: the leaves' LSTM state goes in, and the new state comes out zeroed where the leaf is reset."""
        latent, h, c = states
        out = model.recurrent_inference(latent, (h.unsqueeze(0), c.unsqueeze(0)), action)
        keep = (reset == 0).to(torch.float32).unsqueeze(1)
        B = latent.shape[0]
        hidden = tuple(x.reshape(B, -1) * keep for x in out.reward_hidden_state)
        return (out.latent_state,) + hidden, out.value_prefix, out.value, out.policy_logits


class UniZeroMCTSCtree(MuZeroMCTSCtree):
    """Mirror of ``lzero.mcts.tree_search.mcts_ctree.UniZeroMCTSCtree`` (mcts_ctree.py:19-208): the MuZero tree unchanged
    (``mz_tree.Roots``, :64-75), ``deterministic`` taken from the config (default False, :41-42, passed to ``batch_traverse``
    at :128-137), and a world model that is called with the whole search history:
    ``model.recurrent_inference(state_action_history, simulation_index, search_depth[, timestep | task_id=...])`` (:160-176),
    where ``state_action_history`` is the list of ``(latent_states ndarray, last_actions LongTensor)`` of every simulation so far
    (:147) -- the UniZero transformer re-derives its KV cache from it.  ``search`` returns ``first_action_latent_map`` (:90, :183-189).

    The DRIVER is what this class provides: the trees stay on the GPU (device ``batch_traverse`` / ``batch_backpropagate``), the
    history hand-off follows the reference's host-array contract (one D2H of the gathered latents / actions / search depths per
    simulation, exactly what the reference's own loop does at :144-147).  The transformer world model itself (``WorldModel`` with
    its KV cache, lzero/model/unizero_world_models/) is NOT part of this library: pass the reference's model object, or any
    object with that ``recurrent_inference`` signature."""

    config = dict(MuZeroMCTSCtree.config, deterministic=False)     # mcts_ctree.py:28-43

    def search(self, roots: "mz_tree.Roots", model, latent_state_roots, to_play_batch: Union[int, List[Any]],
               timestep: Union[int, List[Any]] = None, task_id: Optional[int] = None) -> dict:
        S = int(self._cfg.num_simulations)
        roots._materialize(S, self._params(), self.deterministic)
        t = roots._tree
        dev = roots.device
        self._make_inverse_transforms(dev)
        B = roots.num
        lat0 = latent_state_roots.detach().cpu().numpy() if isinstance(latent_state_roots, torch.Tensor) else np.asarray(latent_state_roots)
        latent_pool = [np.ascontiguousarray(lat0, dtype=np.float32)]
        first_action_latent_map = {env_id: {} for env_id in range(B)}
        state_action_history = []
        with torch.no_grad(), torch.cuda.device(dev):
            if hasattr(model, "eval"):
                model.eval()
            for simulation_index in range(S):
                cabi.check(t.lib.lz_tree_traverse(t.h, int(self.deterministic), None, None, t.ix.data_ptr(), t.iy.data_ptr(),
                                                  t.action.data_ptr(), t.search_len.data_ptr(), t.vtp.data_ptr(), None,
                                                  cabi.stream_ptr()), "lz_tree_traverse")
                ix, iy = t.ix.cpu().numpy(), t.iy.cpu().numpy()
                last_actions = t.action.cpu().long()
                search_depth = t.search_len.cpu().numpy().tolist()
                latent_states = np.stack([latent_pool[x][y] for x, y in zip(ix, iy)])          # :141-144
                state_action_history.append((latent_states, last_actions.to(self._cfg.device)))  # :147
                if timestep is None:                                                            # :160-176
                    if task_id is not None:
                        out = model.recurrent_inference(state_action_history, simulation_index, search_depth, task_id=task_id)
                    else:
                        out = model.recurrent_inference(state_action_history, simulation_index, search_depth)
                else:
                    if task_id is not None:
                        out = model.recurrent_inference(state_action_history, simulation_index, search_depth, task_id=task_id)
                    else:
                        out = model.recurrent_inference(state_action_history, simulation_index, search_depth, timestep)
                latent = out.latent_state.detach().cpu().numpy() if isinstance(out.latent_state, torch.Tensor) else np.asarray(out.latent_state)
                value = self._inv(out.value.to(dev)).reshape(-1).contiguous()                   # :180
                reward = self._inv_reward(out.reward.to(dev)).reshape(-1).contiguous()          # :181
                pol = out.policy_logits.to(dev, torch.float32).contiguous()
                for env_id in range(B):                                                         # :183-189
                    a = int(last_actions[env_id].item())
                    if search_depth[env_id] == 1 and a not in first_action_latent_map[env_id]:
                        first_action_latent_map[env_id][a] = latent[env_id]
                latent_pool.append(latent)
                cabi.check(t.lib.lz_tree_backpropagate(t.h, simulation_index + 1, reward.data_ptr(), value.data_ptr(),
                                                       pol.data_ptr(), None, None, None, None, cabi.stream_ptr()),
                           "lz_tree_backpropagate")
        return first_action_latent_map


class GumbelMuZeroMCTSCtree(MuZeroMCTSCtree):
    """Mirror of ``lzero.mcts.tree_search.mcts_ctree.GumbelMuZeroMCTSCtree`` (mcts_ctree.py:1005-1172): same config keys
    (+ ``max_num_considered_actions``, the policy config key read at :1124; default: every action), ``roots(n,
    legal_actions)`` and ``search(roots, model, latent_state_roots, to_play_batch)``.  The roots are ``gmz_tree.Roots``
    prepared with the 6-argument ``prepare`` (or ``prepare_no_noise``).

    With a ``lightzero_b200`` ``MuZeroModel`` / ``MuZeroModelMLP`` the whole loop is one CUDA-graph launch (``lz_search_run``
    on the Gumbel tree): Gumbel descent, recurrent_inference and back-up for every simulation.  Any other model object is
    driven step-wise around the device trees.  The search is deterministic like the reference's (no rand() on its path)."""
    config = dict(
        num_simulations=50,
        root_dirichlet_alpha=0.3,
        root_noise_weight=0.25,
        value_delta_max=0.01,
    )

    @classmethod
    def roots(cls, active_collect_env_num: int, legal_actions: List[Any]) -> "gmz_tree.Roots":
        """mcts_ctree.py:1062-1074"""
        return gmz_tree.Roots(active_collect_env_num, legal_actions)

    def _params(self):
        c = self._cfg
        return (19652, 1.25, c.discount_factor, c.value_delta_max)

    def search(self, roots: "gmz_tree.Roots", model, latent_state_roots, to_play_batch: Union[int, List[Any]]) -> None:
        """mcts_ctree.py:1076-1172.  ``latent_state_roots``: np.ndarray or CUDA tensor."""
        family = _value_prefix_model(model)
        if family:
            raise TypeError(f"GumbelMuZeroMCTSCtree.search: the Gumbel search runs MuZero models, not an {type(model).__name__}")
        S = int(self._cfg.num_simulations)
        if roots._pending is None:
            raise RuntimeError("Roots: prepare()/prepare_no_noise() has not been called")
        m = self._cfg.get("max_num_considered_actions", None)
        m = roots._pending["A"] if m is None else int(m)
        roots._materialize_gumbel((m, S), self._params())   # reset + prepare on device: a fresh search
        lat = _dev_f32(latent_state_roots, roots.device)
        if family is None:
            self._search_stepwise(roots, model, S, lat)
        else:
            self._run_fused(roots, model, S, ("gumbel",), "lz_search_run", lat.data_ptr(), 1)


class StochasticMuZeroMCTSCtree(MuZeroMCTSCtree):
    """Mirror of ``lzero.mcts.tree_search.mcts_ctree_stochastic.StochasticMuZeroMCTSCtree``: ``roots(n, legal_actions,
    chance_space_size)`` and ``search(roots, model, latent_state_roots, to_play_batch)``.  With a
    ``lightzero_b200`` Stochastic MuZero model (``StochasticMuZeroModelMLP`` or ``StochasticMuZeroModel``) the whole search is
    one CUDA graph (``lz_search_run`` on a stochastic tree); any other model is driven step by step on the same device trees.

    Config key ``chance_seed``: an integer s makes every chance selection the draw of ``std::mt19937(s)``, which is what the
    reference draws when ``std::random_device`` returns s (its chance draws are otherwise not reproducible); None (the
    default) samples each selection from the tree's counter-based RNG.  ``deterministic`` is the decision nodes' tie rule,
    as in MuZeroMCTSCtree."""
    config = dict(MuZeroMCTSCtree.config, chance_seed=None)

    @classmethod
    def roots(cls, active_collect_env_num: int, legal_actions: List[Any], chance_space_size: int = 2) -> "stochastic_mz_tree.Roots":
        """mcts_ctree_stochastic.py:72-85"""
        return stochastic_mz_tree.Roots(active_collect_env_num, legal_actions, chance_space_size)

    def search(self, roots: "stochastic_mz_tree.Roots", model, latent_state_roots, to_play_batch: Union[int, List[Any]]) -> None:
        """mcts_ctree_stochastic.py:87-252.  ``latent_state_roots``: np.ndarray or CUDA tensor [B, latent_state_dim] or [B, C, H, W]."""
        S = int(self._cfg.num_simulations)
        roots.set_chance_seed(self._cfg.chance_seed)
        roots._materialize(S, self._params(), self.deterministic)
        lat = _dev_f32(latent_state_roots, roots.device)
        if not isinstance(model, StochasticLzModel):
            self._search_stepwise(roots, model, S, lat)
        else:
            self._run_fused(roots, model, S, (), "lz_search_run", lat.data_ptr(), int(self.deterministic))

    def search_with_reuse(self, *args, **kwargs):
        """Refused: the reference's Stochastic MuZero has no search_with_reuse, and stochastic trees have no reuse descent."""
        raise NotImplementedError("StochasticMuZeroMCTSCtree has no search_with_reuse (stochastic trees have no reuse descent)")

    def _recurrent(self, model, t, states, action, reset):
        """The model with the reference's ``recurrent_inference(state, option, afterstate)``: chance leaves (odd depth) take
        the afterstate program (afterstate=False), the others the dynamics program (mcts_ctree_stochastic.py:171-212); the
        policy logits are padded to the tree's width max(A, C)."""
        latent = states[0]
        B, dev = latent.shape[0], latent.device
        new = torch.empty_like(latent)
        reward = torch.empty(B, self._inv_reward.support.size, device=dev)
        value = torch.empty(B, self._inv.support.size, device=dev)
        logits = torch.zeros(B, t.A, device=dev)
        chance = (t.search_len & 1).bool()
        for is_chance in (True, False):
            sel = torch.nonzero(chance == is_chance).reshape(-1)
            if sel.numel() == 0:
                continue
            out = model.recurrent_inference(latent[sel], action[sel], afterstate=not is_chance)
            new[sel], reward[sel], value[sel] = out.latent_state, out.reward, out.value
            logits[sel, :out.policy_logits.shape[1]] = out.policy_logits.to(torch.float32)
        return (new,), reward, value, logits
