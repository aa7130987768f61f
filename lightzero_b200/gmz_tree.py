"""Device-resident mirror of the reference's Cython module ``lzero.mcts.ctree.ctree_gumbel_muzero.gmz_tree``
(gmz_tree.pyx): ``Roots`` (6-argument ``prepare`` / 4-argument ``prepare_no_noise``, ``get_children_values``,
``get_policies`` and the read-outs), ``MinMaxStatsList``, ``ResultsWrapper``, ``batch_traverse`` and
``batch_back_propagate`` with the same names, argument order and meaning, so the reference search loop
(mcts_ctree.py:1104-1172) runs unchanged on it.  Every list argument may also be a numpy array or a CUDA tensor.  State
lives in the CUDA trees behind ``lz_tree_*_gumbel`` (include/lzb200.h); nothing here computes on the CPU.

Differences a caller can observe: ``batch_traverse`` returns the device tree's virtual to_play, which is the roots'
to_play given at prepare (the reference returns the ``virtual_to_play_batch`` argument unchanged, and its search loop
passes the prepare's to_play there, mcts_ctree.py:1123-1131); a root with an empty legal list has every action legal
and takes the first A Gumbel draws (the reference reads past its empty Gumbel vector there); ``MinMaxStatsList`` is
bookkeeping only (the Gumbel selection never reads min/max stats).
"""
from typing import List

import torch

from . import cabi, mz_tree
from .mz_tree import MinMaxStatsList, ResultsWrapper, _to_dev   # noqa: F401  (same classes as gmz_tree.pyx:5-26)


class Roots(mz_tree.Roots):
    """gmz_tree.pyx:28-65.  ``legal_actions_list``: list of lists, or a uint8/bool mask [root_num, A]."""

    def __init__(self, root_num: int, legal_actions_list, device=None):
        super().__init__(root_num, legal_actions_list, device)
        self._gumbel = None        # (max_num_considered_actions, num_simulations) the tree was set up with
        self._values = None

    # ---- reference API ---------------------------------------------------------------------------
    def prepare(self, root_noise_weight: float, noises, value_prefix_pool, value_pool, policy_logits_pool, to_play_batch):
        self._values = _to_dev(value_pool, torch.float32, self.device, (self.root_num,))
        self._stage(float(root_noise_weight), noises, value_prefix_pool, policy_logits_pool, to_play_batch)

    def prepare_no_noise(self, value_prefix_pool, value_pool, policy_logits_pool, to_play_batch):
        self._values = _to_dev(value_pool, torch.float32, self.device, (self.root_num,))
        self._stage(0.0, None, value_prefix_pool, policy_logits_pool, to_play_batch)

    def get_children_values(self, discount: float, action_space_size: int) -> List[List[float]]:
        return self.get_children_values_tensor(discount, action_space_size).cpu().tolist()

    def get_policies(self, discount: float, action_space_size: int) -> List[List[float]]:
        return self.get_policies_tensor(discount, action_space_size).cpu().tolist()

    def clear(self):
        if self._tree is not None:      # hand the pooled tree back as a MuZero tree
            with torch.cuda.device(self.device):
                cabi.check(self._tree.lib.lz_tree_set_gumbel(self._tree.h, 0, 0), "lz_tree_set_gumbel")
            self._gumbel = None
        super().clear()

    # ---- device-side extras ----------------------------------------------------------------------
    def get_children_values_tensor(self, discount: float, action_space_size: int):
        return self._policies(discount, action_space_size)[0]

    def get_policies_tensor(self, discount: float, action_space_size: int):
        return self._policies(discount, action_space_size)[1]

    # ---- internals -------------------------------------------------------------------------------
    def _policies(self, discount, A):
        t = self._need_tree()
        if int(A) != t.A:
            raise ValueError(f"action_space_size {A} != the {t.A} actions of the roots' logits")
        self._set_discount(float(discount))
        cv = torch.empty(self.root_num, t.A, dtype=torch.float32, device=self.device)
        pol = torch.empty_like(cv)
        with torch.cuda.device(self.device):
            cabi.check(t.lib.lz_tree_gumbel_policies(t.h, cv.data_ptr(), pol.data_ptr(), cabi.stream_ptr()),
                       "lz_tree_gumbel_policies")
        return cv, pol

    def _set_discount(self, discount):
        t = self._tree
        p = t.params or (19652, 1.25, 0.997, 0.01)
        t.set_params(p[0], p[1], discount, p[3])

    def _need_tree(self):
        if self._tree is None:
            raise RuntimeError("Roots: no search has run on these roots (call batch_traverse first)")
        return self._tree

    def _setup(self, max_num_considered_actions: int, num_simulations: int, discount: float = None):
        """Materialises the tree for this (m, S) on first use (reset + prepare on device), like the reference's lazily
        sized node maps; later calls only refresh the discount."""
        g = (int(max_num_considered_actions), int(num_simulations))
        if self._tree is None or self._gumbel != g or self._tree.max_sims < g[1]:
            self._materialize_gumbel(g)
        if discount is not None:
            self._set_discount(float(discount))
        return self._tree

    def _materialize_gumbel(self, g, params=None):
        m, S = g
        if self._pending is None:
            raise RuntimeError("Roots: prepare()/prepare_no_noise() has not been called")
        A = self._pending["A"]
        if self._tree is not None and (self._tree.max_sims < S or self._tree.A != A):
            self.clear()
        if self._tree is None:
            self._tree = mz_tree.acquire_tree(self.device, self.root_num, A, S)
        t = self._tree
        if params is not None:
            t.set_params(*params)
        with torch.cuda.device(self.device):
            cabi.check(t.lib.lz_tree_set_ez(t.h, 0, 5), "lz_tree_set_ez")
            cabi.check(t.lib.lz_tree_set_gumbel(t.h, m, S), "lz_tree_set_gumbel")
        self._gumbel = g
        self._reset_and_prepare()

    def _reset_and_prepare(self):
        """Reset to the legal lists and lz_tree_prepare_gumbel: a fresh search on these roots."""
        t, p = self._tree, self._pending
        with torch.cuda.device(self.device):
            s = cabi.stream_ptr()
            self._reset_tree(t, s)
            cabi.check(t.lib.lz_tree_prepare_gumbel(t.h, p["logits"].data_ptr(), cabi.ptr(p["noise"]), p["w"],
                                                    cabi.ptr(p["rewards"]), self._values.data_ptr(), cabi.ptr(p["to_play"]), s),
                       "lz_tree_prepare_gumbel")

    def _materialize(self, max_sims, params=None):
        # a re-prepare of a materialised tree (mz_tree.Roots._stage) starts a fresh Gumbel search
        if self._gumbel is None:
            self._gumbel = (max_sims, max_sims)
        self._materialize_gumbel(self._gumbel, params)


def batch_traverse(roots: Roots, num_simulations: int, max_num_considered_actions: int, discount: float,
                   results: ResultsWrapper, virtual_to_play_batch, return_tensors: bool = False):
    """gmz_tree.pyx:91-95 -> (latent_state_index_in_search_path, latent_state_index_in_batch, last_actions,
    virtual_to_play_batch)."""
    t = roots._setup(max_num_considered_actions, num_simulations, discount)
    with torch.cuda.device(roots.device):
        cabi.check(t.lib.lz_tree_traverse_gumbel(t.h, t.ix.data_ptr(), t.iy.data_ptr(), t.action.data_ptr(),
                                                 t.search_len.data_ptr(), t.vtp.data_ptr(), cabi.stream_ptr()),
                   "lz_tree_traverse_gumbel")
    results._roots = roots
    if return_tensors:
        return t.ix, t.iy, t.action, t.vtp
    packed = torch.stack((t.ix, t.iy, t.action, t.vtp)).cpu().numpy()
    return packed[0].tolist(), packed[1].tolist(), packed[2].tolist(), packed[3].tolist()


def batch_back_propagate(current_latent_state_index: int, discount: float, value_prefixs, values, policies,
                         min_max_stats_lst: MinMaxStatsList, results: ResultsWrapper, to_play_batch):
    """gmz_tree.pyx:81-88"""
    roots = results._roots
    t = roots._tree
    roots._set_discount(float(discount))
    B, A, dev = roots.root_num, t.A, roots.device
    rew = _to_dev(value_prefixs, torch.float32, dev, (B,))
    val = _to_dev(values, torch.float32, dev, (B,))
    pol = _to_dev(policies, torch.float32, dev, (B, A))
    tp = _to_dev(to_play_batch, torch.int32, dev, (B,)) if to_play_batch is not None else None
    with torch.cuda.device(dev):
        cabi.check(t.lib.lz_tree_backpropagate_gumbel(t.h, int(current_latent_state_index), rew.data_ptr(), val.data_ptr(),
                                                      pol.data_ptr(), cabi.ptr(tp), cabi.stream_ptr()),
                   "lz_tree_backpropagate_gumbel")
    t._keep = (rew, val, pol, tp)
