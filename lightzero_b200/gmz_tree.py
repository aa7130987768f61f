"""Device-resident mirror of the reference's Cython module ``lzero.mcts.ctree.ctree_gumbel_muzero.gmz_tree``
(gmz_tree.pyx): ``Roots`` (6-argument ``prepare`` / 4-argument ``prepare_no_noise``, ``get_children_values``,
``get_policies`` and the read-outs), ``MinMaxStatsList``, ``ResultsWrapper``, ``batch_traverse`` and
``batch_back_propagate`` with the same names, argument order and meaning, so the reference search loop
(mcts_ctree.py:1104-1172) runs unchanged on it.  Every list argument may also be a numpy array or a CUDA tensor.  State
lives in the CUDA Gumbel trees behind ``lz_tree_*`` (include/lzb200.h); nothing here computes on the CPU.

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
        t = self._acquire(g[1], params, True, gumbel=g)     # the Gumbel descents never read the tie rule
        self._gumbel = g
        self._reset_and_prepare(t)

    def _materialize(self, max_sims, params=None, deterministic=None):
        # a re-prepare of a materialised tree (mz_tree.Roots._stage) starts a fresh Gumbel search
        if self._gumbel is None:
            self._gumbel = (max_sims, max_sims)
        self._materialize_gumbel(self._gumbel, params)


def batch_traverse(roots: Roots, num_simulations: int, max_num_considered_actions: int, discount: float,
                   results: ResultsWrapper, virtual_to_play_batch, return_tensors: bool = False):
    """gmz_tree.pyx:91-95 -> (latent_state_index_in_search_path, latent_state_index_in_batch, last_actions,
    virtual_to_play_batch)."""
    roots._setup(max_num_considered_actions, num_simulations, discount)
    return mz_tree._traverse(roots, results, return_tensors)


def batch_back_propagate(current_latent_state_index: int, discount: float, value_prefixs, values, policies,
                         min_max_stats_lst: MinMaxStatsList, results: ResultsWrapper, to_play_batch):
    """gmz_tree.pyx:81-88"""
    results._roots._set_discount(float(discount))
    mz_tree._backpropagate(results, current_latent_state_index, value_prefixs, values, policies, to_play_batch)
