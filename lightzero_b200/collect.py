"""Mirror of the search-driving part of ``MuZeroPolicy._forward_collect`` / ``_forward_eval``
(lzero/policy/muzero.py:705-829, 872-956) and of ``select_action`` (lzero/policy/utils.py:637-661).

``MuZeroCollectPolicy.forward_collect(obs, action_mask, temperature, to_play)`` takes what the
reference's collector passes (a stacked observation batch, a 0/1 action mask, to_play) and returns
the same per-environment output dict.  Observations may live in (pinned) HOST memory: the copy to the
device, the representation+prediction networks, root preparation with Dirichlet noise, the whole
num_simulations search (one CUDA graph) and the result read-back are issued back to back on one
stream; the only host synchronisation is the final read of the results.
"""
from typing import Dict, List, Optional, Union

import numpy as np
import torch

from . import cabi, mz_tree
from .efficientzero_model import EfficientZeroModel
from .efficientzero_model_mlp import EfficientZeroModelMLP
from .mcts_ctree import EfficientZeroMCTSCtree, GumbelMuZeroMCTSCtree, MuZeroMCTSCtree, StochasticMuZeroMCTSCtree
from .model_base import LzModel, StochasticLzModel
from .muzero_model import MuZeroModel
from .muzero_model_mlp import MuZeroModelMLP
from .stochastic_mz_tree import chance_uniform

_NP = {torch.uint8: np.uint8, torch.float32: np.float32, torch.int32: np.int32}


def select_action(visit_counts: np.ndarray, temperature: float = 1, deterministic: bool = True):
    """lzero/policy/utils.py:637-661 (same arithmetic, fp64 numpy)."""
    action_probs = [visit_count_i ** (1 / temperature) for visit_count_i in visit_counts]
    action_probs = [x / sum(action_probs) for x in action_probs]
    if deterministic:
        action_pos = int(np.argmax([v for v in visit_counts]))
    else:
        action_pos = int(np.random.choice(len(visit_counts), p=action_probs))
    p = np.asarray(action_probs, np.float64)
    nz = p[p > 0]
    entropy = float(-(nz * np.log(nz)).sum() / np.log(2.0))   # scipy.stats.entropy(action_probs, base=2): natural-log entropy / ln 2
    return action_pos, entropy


def _as_tensor(x, dtype):
    """A mask, noise or to_play argument (tensor, array or list) as a tensor of dtype where it already lives: arrays and
    lists on the host."""
    if isinstance(x, torch.Tensor):
        return x.to(dtype)
    return torch.from_numpy(np.require(x, _NP[dtype], ["C", "W"]))     # copies read-only views (np.broadcast_to)


def _broadcast_to_play(to_play, B):
    return np.broadcast_to(np.asarray(to_play, np.int32).reshape(-1), (B,)) if np.size(to_play) in (1, B) else to_play


def _legal_dirichlet(action_mask, alpha):
    """Root noise drawn with np.random as the reference policies do (policy/muzero.py:763-766, gumbel_muzero.py:555-558):
    per root, Dirichlet(alpha) over its legal actions, in legal order, zero padded to [B, A]."""
    B, A = action_mask.shape
    noises = np.zeros((B, A), np.float32)
    for j in range(B):
        n = int(action_mask[j].sum())
        noises[j, :n] = np.random.dirichlet([alpha] * n).astype(np.float32)
    return noises


class MuZeroCollectPolicy:
    def __init__(self, model: MuZeroModel, cfg: Optional[dict] = None):
        self.model = model
        self.mcts = MuZeroMCTSCtree(cfg or {})
        self.cfg = self.mcts._cfg
        self.device = model.device
        self._buf = {}
        self.h2d_chunks = 2      # host observation batches are copied in this many overlapped pieces
        self._tree_mode = ()     # the search_for / TreeHandle.set_mode mode: MuZero trees

    # ---- device-resident fast path ---------------------------------------------------------------
    def _bufs(self, B, A):
        key = (B, A)
        if key not in self._buf:
            d = self.device
            self._buf[key] = dict(
                pred_value=torch.empty(B, device=d), logits=torch.empty(B, A, device=d),
                obs=None, mask=torch.empty(B, A, dtype=torch.uint8, device=d), noise=torch.empty(B, A, device=d),
                to_play=torch.empty(B, dtype=torch.int32, device=d),
                h_visits=torch.empty(B, A, dtype=torch.int32).pin_memory(),
                h_values=torch.empty(B).pin_memory(), h_pred=torch.empty(B).pin_memory(),
                h_logits=torch.empty(B, A).pin_memory(), h_nlegal=torch.empty(B, dtype=torch.int32).pin_memory(),
                action=torch.empty(B, dtype=torch.int32, device=d), action_pos=torch.empty(B, dtype=torch.int32, device=d),
                entropy=torch.empty(B, device=d), h_action=torch.empty(B, dtype=torch.int32).pin_memory(),
                h_entropy=torch.empty(B).pin_memory())
        return self._buf[key]

    def search_batch(self, obs: torch.Tensor, action_mask, noises, to_play=None, deterministic=None,
                     read_back: bool = True, select=None):
        """obs [B,C,H,W] (host or device), action_mask [B,A] 0/1, noises [B,A] rows in legal order or None
        (eval).  Returns dict of tensors; with read_back=True they are pinned host tensors and the call
        ends with the single stream synchronisation of the step.  select=(temperature, deterministic_action, seed) also
        runs select_action (policy/utils.py:637-661) on the device and returns 'action' / 'entropy' (GumbelMuZeroCollectPolicy: the
        Gumbel read-out, which adds 'improved_policy' / 'completed_values' [B, A])."""
        B = obs.shape[0]
        A = self._width()
        S = int(self.cfg.num_simulations)
        bufs = self._bufs(B, A)
        dev = self.device
        det = self.mcts.deterministic if deterministic is None else bool(deterministic)
        with torch.cuda.device(dev):
            host_path = not obs.is_cuda
            # uint8 frames (what the Atari emulator delivers) stay uint8 on the wire: a quarter of the bytes; the [0, 1] scaling
            # of the reference's ScaledFloatFrameWrapper happens inside the first conv kernel (lz_search_collect*_u8)
            u8 = obs.dtype == torch.uint8
            obs = obs.contiguous() if u8 else obs.to(torch.float32).contiguous()
            args = ((action_mask, "mask"), (noises, "noise"), (to_play, "to_play"))
            if host_path:
                mask, noise, tp = (None if x is None else _as_tensor(x, bufs[k].dtype).contiguous() for x, k in args)
                assert not mask.is_cuda and (noise is None or not noise.is_cuda), "host observation batch needs host mask / noise"
                self._keep_host = (obs, mask, noise, tp)
            else:
                mask, noise, tp = (None if x is None else bufs[k].copy_(_as_tensor(x, bufs[k].dtype), non_blocking=True)
                                   for x, k in args)
            # the search and the clones below may still be queued when the tree is released: the next holder waits for them
            with self._held_tree(B, A, S, det) as tree:
                q = tree.search_for(self.model, S, self._tree_mode)
                s = cabi.stream_ptr()
                if host_path:
                    fn = tree.lib.lz_search_collect_host_u8 if u8 else tree.lib.lz_search_collect_host
                    cabi.check(fn(q, obs.data_ptr(), mask.data_ptr(), cabi.ptr(noise),
                                  float(self.cfg.root_noise_weight), cabi.ptr(tp), int(det),
                                  int(self.h2d_chunks), bufs["pred_value"].data_ptr(),
                                  bufs["logits"].data_ptr(), s), "lz_search_collect_host")
                else:
                    fn = tree.lib.lz_search_collect_u8 if u8 else tree.lib.lz_search_collect
                    cabi.check(fn(q, obs.data_ptr(), mask.data_ptr(), cabi.ptr(noise),
                                  float(self.cfg.root_noise_weight), cabi.ptr(tp), int(det),
                                  bufs["pred_value"].data_ptr(), bufs["logits"].data_ptr(), s),
                               "lz_search_collect")
                cabi.check(tree.lib.lz_tree_results(tree.h, tree.visits.data_ptr(), tree.values.data_ptr(),
                                                    tree.nlegal.data_ptr(), None, s), "lz_tree_results")
                self.last_num_kernels = tree.lib.lz_search_num_kernels(q)
                selected = self._select(tree, bufs, select, s) if select is not None else ()
                if not read_back:
                    dev_out = dict(visits=tree.visits.clone(), values=tree.values.clone(), nlegal=tree.nlegal.clone(),
                                   pred_value=bufs["pred_value"], policy_logits=bufs["logits"])
                    # the device-side select_action results stay on the device too
                    dev_out.update({k: bufs[k].clone() for k in selected})
                    return dev_out
                bufs["h_visits"].copy_(tree.visits, non_blocking=True)
                bufs["h_values"].copy_(tree.values, non_blocking=True)
                bufs["h_nlegal"].copy_(tree.nlegal, non_blocking=True)
                bufs["h_pred"].copy_(bufs["pred_value"], non_blocking=True)
                bufs["h_logits"].copy_(bufs["logits"], non_blocking=True)
                for k in selected:
                    bufs["h_" + k].copy_(bufs[k], non_blocking=True)
                torch.cuda.current_stream().synchronize()
        out = dict(visits=bufs["h_visits"], values=bufs["h_values"], nlegal=bufs["h_nlegal"],
                   pred_value=bufs["h_pred"], policy_logits=bufs["h_logits"])
        out.update({k: bufs["h_" + k] for k in selected})
        return out

    def _width(self):
        """The row width of the tree and of the mask, noise and logits buffers: the action count."""
        return self.model.action_space_size

    def _held_tree(self, B, A, S, det):
        """A pooled tree in this policy's mode for one search_batch: the collect's tie rule is its ``deterministic``, which
        lz_search_collect also applies to EfficientZero trees."""
        return mz_tree.held_tree(self.device, B, A, S, self.mcts._params(), self._tree_mode, det)

    def _select(self, tree, bufs, select, s):
        """select_action on the device into bufs; returns the names of the tensors it wrote."""
        cabi.check(tree.lib.lz_tree_select_action(tree.h, float(select[0]), int(bool(select[1])), int(select[2]) & (2 ** 64 - 1),
                                                  bufs["action"].data_ptr(), bufs["action_pos"].data_ptr(),
                                                  bufs["entropy"].data_ptr(), s), "lz_tree_select_action")
        return ("action", "entropy")

    # ---- reference-shaped API --------------------------------------------------------------------
    def forward_collect(self, data: torch.Tensor, action_mask, temperature: float = 1, to_play=(-1,),
                        epsilon: float = 0.25, ready_env_id=None, device_select_action: bool = False, seed: int = 0,
                        **kwargs) -> Dict[int, dict]:
        """policy/muzero.py:705-829 (collect_with_pure_policy=False, no eps-greedy).  device_select_action=True draws the
        actions on the GPU (lz_tree_select_action, keyed by `seed`) instead of np.random.choice on the host."""
        B = data.shape[0]
        if ready_env_id is None:
            ready_env_id = np.arange(B)
        action_mask = np.asarray(action_mask)
        noises = _legal_dirichlet(action_mask, float(self.cfg.root_dirichlet_alpha))
        r = self.search_batch(data, action_mask, noises, _broadcast_to_play(to_play, B), deterministic=self.mcts.deterministic,
                              select=(temperature, False, seed) if device_select_action else None)
        return self._format(r, action_mask, ready_env_id, temperature, deterministic_action=False)

    def forward_eval(self, data: torch.Tensor, action_mask, to_play=(-1,), ready_env_id=None, **kwargs):
        """policy/muzero.py:872-956: no noise, arg-max action."""
        B = data.shape[0]
        if ready_env_id is None:
            ready_env_id = np.arange(B)
        action_mask = np.asarray(action_mask)
        r = self.search_batch(data, action_mask, None, _broadcast_to_play(to_play, B), deterministic=self.mcts.deterministic)
        return self._format(r, action_mask, ready_env_id, 1, deterministic_action=True)

    def _format(self, r, action_mask, ready_env_id, temperature, deterministic_action) -> Dict[int, dict]:
        visits, nl = r["visits"].numpy(), r["nlegal"].numpy()
        values, pred, logits = r["values"].numpy(), r["pred_value"].numpy(), r["policy_logits"].numpy()
        output = {}
        for i, env_id in enumerate(ready_env_id):
            distributions = visits[i, :nl[i]].tolist()
            if "action" in r:                                              # chosen on the device
                action, ent = int(r["action"][i]), float(r["entropy"][i])
            else:
                pos, ent = select_action(distributions, temperature=temperature, deterministic=deterministic_action)
                action = np.where(action_mask[i] == 1.0)[0][pos]            # policy/muzero.py:800
            output[env_id] = {
                'action': action,
                'visit_count_distributions': distributions,
                'visit_count_distribution_entropy': ent,
                'searched_value': float(values[i]),
                'predicted_value': float(pred[i]),
                'predicted_policy_logits': logits[i].tolist(),
            }
        return output


class EfficientZeroCollectPolicy(MuZeroCollectPolicy):
    """The same for ``EfficientZeroPolicy._forward_collect`` / ``_forward_eval`` (lzero/policy/efficientzero.py:539-640,
    690-760): value-prefix trees, the reward hidden state starts as zeros after ``initial_inference`` (:580-590) and is reset
    every ``lstm_horizon_len`` steps of search depth.  Same output dict."""

    def __init__(self, model: Union[EfficientZeroModel, EfficientZeroModelMLP], cfg: Optional[dict] = None):
        super().__init__(model, cfg)
        self.mcts = EfficientZeroMCTSCtree(cfg or {})
        self.cfg = self.mcts._cfg
        self._tree_mode = (1, int(self.cfg.lstm_horizon_len))     # value-prefix trees


class GumbelMuZeroCollectPolicy(MuZeroCollectPolicy):
    """The same for ``GumbelMuZeroPolicy._forward_collect`` / ``_forward_eval`` (lzero/policy/gumbel_muzero.py:498-720) with a
    ``MuZeroModel`` (conv or board) or ``MuZeroModelMLP``: the pooled tree is a Gumbel tree (``max_num_considered_actions``,
    default 4 as the reference policy's config, and ``num_simulations``), the roots are prepared with the initial inference's
    value, and one device read-out gives per root the improved policy, the masked completed Q, the action (the first maximum
    of the improved policy over the legal actions, in collect and eval alike) and select_action's visit-count entropy.  Output
    dicts have the reference's keys."""

    def __init__(self, model: Union[MuZeroModel, MuZeroModelMLP], cfg: Optional[dict] = None):
        if isinstance(model, LzModel) and model.value_prefix:
            raise TypeError(f"GumbelMuZeroCollectPolicy: the Gumbel search runs MuZero models, not an {type(model).__name__}")
        super().__init__(model, cfg)
        self.mcts = GumbelMuZeroMCTSCtree(cfg or {})
        self.cfg = self.mcts._cfg
        self.cfg.setdefault("max_num_considered_actions", 4)
        self._tree_mode = ("gumbel",)

    def _bufs(self, B, A):
        bufs = super()._bufs(B, A)
        if "improved_policy" not in bufs:
            for k in ("improved_policy", "completed_values"):
                bufs[k] = torch.empty(B, A, device=self.device)
                bufs["h_" + k] = torch.empty(B, A).pin_memory()
        return bufs

    def _held_tree(self, B, A, S, det):
        """A Gumbel tree: its descents never read the tie rule."""
        return mz_tree.held_tree(self.device, B, A, S, self.mcts._params(),
                                 gumbel=(int(self.cfg.max_num_considered_actions), S))

    def _select(self, tree, bufs, select, s):
        """lz_tree_gumbel_select_action at temperature select[0]: the action never depends on a draw."""
        cabi.check(tree.lib.lz_tree_gumbel_select_action(tree.h, float(select[0]), bufs["action"].data_ptr(), bufs["entropy"].data_ptr(),
                                                         bufs["completed_values"].data_ptr(), bufs["improved_policy"].data_ptr(), s),
                   "lz_tree_gumbel_select_action")
        return ("action", "entropy", "improved_policy", "completed_values")

    def forward_collect(self, data: torch.Tensor, action_mask, temperature: float = 1, to_play=(-1,),
                        epsilon: float = 0.25, ready_env_id=None, **kwargs) -> Dict[int, dict]:
        """gumbel_muzero.py:498-607: Dirichlet noise in legal order drawn with np.random as the reference does."""
        B = data.shape[0]
        action_mask = np.asarray(action_mask)
        noises = _legal_dirichlet(action_mask, float(self.cfg.root_dirichlet_alpha))
        r = self.search_batch(data, action_mask, noises, _broadcast_to_play(to_play, B), select=(temperature, False, 0))
        return self._format_gumbel(r, B, ready_env_id, collect=True)

    def forward_eval(self, data: torch.Tensor, action_mask, to_play=(-1,), ready_env_id=None, **kwargs) -> Dict[int, dict]:
        """gumbel_muzero.py:619-720: no noise, entropy at temperature 1."""
        B = data.shape[0]
        r = self.search_batch(data, np.asarray(action_mask), None, _broadcast_to_play(to_play, B), select=(1.0, True, 0))
        return self._format_gumbel(r, B, ready_env_id, collect=False)

    def _format_gumbel(self, r, B, ready_env_id, collect) -> Dict[int, dict]:
        if ready_env_id is None:
            ready_env_id = np.arange(B)
        visits, nl = r["visits"].numpy(), r["nlegal"].numpy()
        values, pred, logits = r["values"].numpy(), r["pred_value"].numpy(), r["policy_logits"].numpy()
        action, ent = r["action"].numpy(), r["entropy"].numpy()
        improved, completed = r["improved_policy"].numpy(), r["completed_values"].numpy()
        output = {}
        for i, env_id in enumerate(ready_env_id):
            out = {
                'action': np.int64(action[i]),
                'visit_count_distributions': visits[i, :nl[i]].tolist(),
                'visit_count_distribution_entropy': float(ent[i]),
                'searched_value': float(values[i]),
            }
            if collect:
                out['roots_completed_value'] = completed[i].astype(np.float64)
                out['improved_policy_probs'] = improved[i].astype(np.float64)
            out['predicted_value'] = float(pred[i])
            out['predicted_policy_logits'] = logits[i].tolist()
            output[env_id] = out
        return output


def _pad_columns(x, W):
    """A [B, n] mask or noise argument (tensor, array or list of rows) zero padded to [B, W], where it already lives."""
    if isinstance(x, torch.Tensor):
        return torch.nn.functional.pad(x, (0, W - x.shape[1]))
    x = np.asarray(x)
    return np.pad(x, ((0, 0), (0, W - x.shape[1])))


class StochasticMuZeroCollectPolicy(MuZeroCollectPolicy):
    """The same for ``StochasticMuZeroPolicy._forward_collect`` / ``_forward_eval`` (lzero/policy/stochastic_muzero.py:578-760)
    with a Stochastic MuZero model (``StochasticMuZeroModelMLP`` or ``StochasticMuZeroModel``): the pooled tree is a
    stochastic tree W = max(action_space_size, chance_space_size) wide, and one ``lz_search_collect*`` call runs
    initial_inference, the root reset and prepare and the stochastic search graph.  The config key ``chance_seed`` is read as ``StochasticMuZeroMCTSCtree`` reads it: an integer pins every chance draw
    to std::mt19937(chance_seed)'s, None samples each step's draws afresh.  Masks and noises are [B, action_space_size] as the
    reference takes them; ``search_batch`` returns visits [B, W] (-1 padded, as ``stochastic_mz_tree.Roots``) and policy
    logits [B, action_space_size].  Output dicts have the reference's keys."""

    def __init__(self, model: StochasticLzModel, cfg: Optional[dict] = None):
        if not isinstance(model, StochasticLzModel):
            raise TypeError(f"StochasticMuZeroCollectPolicy: the stochastic search runs a StochasticMuZeroModelMLP or StochasticMuZeroModel, not a "
                            f"{type(model).__name__}")
        super().__init__(model, cfg)
        self.mcts = StochasticMuZeroMCTSCtree(cfg or {})
        self.cfg = self.mcts._cfg

    def _width(self):
        return max(self.model.action_space_size, self.model.chance_space_size)

    def _held_tree(self, B, W, S, det):
        """A stochastic tree; the decision nodes' tie rule is the collect's ``deterministic``."""
        seed = self.cfg.chance_seed
        u = -1.0 if seed is None else chance_uniform(seed)
        return mz_tree.held_tree(self.device, B, W, S, self.mcts._params(), (), det,
                                 stochastic=(self.model.action_space_size, self.model.chance_space_size, u))

    def search_batch(self, obs: torch.Tensor, action_mask, noises, to_play=None, deterministic=None,
                     read_back: bool = True, select=None):
        """MuZeroCollectPolicy.search_batch on the stochastic tree: action_mask and noises [B, action_space_size] are padded
        to the tree's width W with zero columns, and the returned policy logits are the first action_space_size columns of
        the [B, W] rows the collect writes."""
        W = self._width()
        out = super().search_batch(obs, _pad_columns(action_mask, W), None if noises is None else _pad_columns(noises, W),
                                   to_play, deterministic, read_back, select)
        out["policy_logits"] = out["policy_logits"][:, :self.model.action_space_size]
        return out
