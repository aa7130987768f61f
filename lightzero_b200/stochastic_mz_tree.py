"""Device-resident mirror of the reference's Cython module ``lzero.mcts.ctree.ctree_stochastic_muzero.stochastic_mz_tree``
(stochastic_mz_tree.pyx): ``Roots(root_num, legal_actions_list, chance_space_size)``, ``MinMaxStatsList``, ``ResultsWrapper``,
``batch_traverse`` and ``batch_backpropagate`` with the same names, argument order and meaning, so the reference search loop
(mcts_ctree_stochastic.py:117-252) drives the CUDA trees around any model step by step.  Every list argument may also be a
numpy array or a CUDA tensor.  State lives in the stochastic trees behind ``lz_tree_*`` (``lz_tree_set_stochastic``).

Chance nodes draw their outcome as the reference's ``std::discrete_distribution(priors)(std::mt19937(rd()))``
(ctree_stochastic_muzero/lib/cnode.cpp:610-630).  ``Roots(..., chance_seed=s)`` pins that draw to the one a
``std::random_device`` returning s gives (``chance_uniform``); ``chance_seed=None`` (the default) samples every selection from
the tree's counter-based RNG.

Differences a caller can observe: the tree's logits rows are max(A, chance_space_size) wide, so ``get_distributions`` and the
tensors are padded to that width; ``batch_backpropagate`` only stages its rows, and the back-up of every tree runs once the
calls of one simulation have covered all of them (the reference backs up the chance subset, then the decision subset; the
trees are independent, so the result is the same); ``MinMaxStatsList`` is bookkeeping only, as in ``mz_tree``.
"""
from typing import Optional

import numpy as np
import torch

from . import cabi, mz_tree
from .mz_tree import MinMaxStatsList, _to_dev   # noqa: F401  (same classes as stochastic_mz_tree.pyx:5-15)


def _mt19937_first2(seed: int):
    """The first two outputs of std::mt19937(seed)."""
    mt = [0] * 624
    mt[0] = seed & 0xffffffff
    for i in range(1, 624):
        mt[i] = (1812433253 * (mt[i - 1] ^ (mt[i - 1] >> 30)) + i) & 0xffffffff
    out = []
    for i in range(2):      # the first twist only needs elements 0, 1, 2 and 397, 398
        y = (mt[i] & 0x80000000) | (mt[i + 1] & 0x7fffffff)
        x = mt[i + 397] ^ (y >> 1) ^ (0x9908b0df if y & 1 else 0)
        x ^= x >> 11
        x ^= (x << 7) & 0x9d2c5680
        x ^= (x << 15) & 0xefc60000
        x ^= x >> 18
        out.append(x)
    return out


def chance_uniform(seed: int) -> float:
    """The uniform std::discrete_distribution draws from std::mt19937(seed) in libstdc++: generate_canonical<double, 53> of
    two 32-bit outputs, (g1 + g2 * 2^32) / 2^64 in double, values >= 1 clamped to the largest double below 1."""
    g1, g2 = _mt19937_first2(int(seed))
    u = (float(g1) + float(g2) * 4294967296.0) / 18446744073709551616.0
    return u if u < 1.0 else float(np.nextafter(1.0, 0.0))


class ResultsWrapper(mz_tree.ResultsWrapper):
    """stochastic_mz_tree.pyx:17-24; also stages the rows of the batch_backpropagate calls of one simulation."""

    def __init__(self, num: int):
        super().__init__(num)
        self._staged = None


class Roots(mz_tree.Roots):
    """stochastic_mz_tree.pyx:26-59.  ``legal_actions_list``: list of lists, or a uint8/bool mask [root_num, A].
    ``chance_seed``: an integer pins every chance draw to std::mt19937(chance_seed)'s; None samples.  ``max_simulations``:
    the node capacity of a tree driven step by step by batch_traverse / batch_backpropagate (a search sizes its own)."""

    def __init__(self, root_num: int, legal_actions_list, chance_space_size: int = 2, device=None,
                 chance_seed: Optional[int] = None, max_simulations: int = mz_tree.DEFAULT_MAX_SIMS):
        super().__init__(root_num, legal_actions_list, device)
        if int(chance_space_size) < 1:
            raise ValueError(f"chance_space_size must be >= 1 (got {chance_space_size})")
        self.chance_space_size = int(chance_space_size)
        self._max_sims = int(max_simulations)
        self.set_chance_seed(chance_seed)

    def _need_tree(self):
        if self._tree is None:
            self._materialize(self._max_sims)
        return self._tree

    def set_chance_seed(self, chance_seed: Optional[int]):
        self._chance_u = -1.0 if chance_seed is None else chance_uniform(chance_seed)
        if self._stochastic[1]:
            self._stochastic = self._stochastic[:2] + (self._chance_u,)

    def _stage(self, w, noises, rewards, policies, to_play):
        pol = _to_dev(policies, torch.float32, self.device).reshape(self.root_num, -1)
        A = pol.shape[1]
        W = max(A, self.chance_space_size)
        pol = torch.nn.functional.pad(pol, (0, W - A))      # the tree's rows are max(A, chance_space_size) wide
        if isinstance(noises, (torch.Tensor, np.ndarray)):
            noises = torch.nn.functional.pad(_to_dev(noises, torch.float32, self.device, (self.root_num, A)), (0, W - A))
        if self._mask is not None and np.shape(self._mask)[1] < W:
            m = _to_dev(self._mask, torch.uint8, self.device)
            self._mask = torch.nn.functional.pad(m, (0, W - m.shape[1]))
            self._mask_dev = None
        self._stochastic = (A, self.chance_space_size, self._chance_u)
        super()._stage(w, noises, rewards, pol, to_play)


def batch_traverse(roots: Roots, pb_c_base: int, pb_c_init: float, discount_factor: float,
                   min_max_stats_lst: MinMaxStatsList, results: ResultsWrapper, virtual_to_play_batch,
                   deterministic: bool = False, return_tensors: bool = False):
    """stochastic_mz_tree.pyx:85-91 -> (leaf_node_is_chance, latent_state_index_in_search_path,
    latent_state_index_in_batch, last_actions, virtual_to_play_batch).  A leaf is a chance node when its depth is odd.
    ``deterministic``: PUCT ties at decision nodes go to the first maximum (the reference's rand() % len(ties) with
    rand() == 0), else a uniform draw from the tie list."""
    roots._need_tree().set_params(pb_c_base, pb_c_init, discount_factor, min_max_stats_lst.value_delta_max)
    ix, iy, act, vtp = mz_tree._traverse(roots, results, True, deterministic)
    is_chance = (roots._tree.search_len & 1).bool()
    results._staged = None
    if return_tensors:
        return is_chance, ix, iy, act, vtp
    host = torch.stack((is_chance.to(torch.int32), ix, iy, act, vtp)).cpu().numpy()
    return ([bool(x) for x in host[0]],) + tuple(x.tolist() for x in host[1:])


def batch_backpropagate(current_latent_state_index: int, discount_factor: float, value_prefixs, values, policies,
                        min_max_stats_lst: MinMaxStatsList, results: ResultsWrapper, to_play_batch, is_chance_list,
                        leaf_idx_list=None):
    """stochastic_mz_tree.pyx:73-83 (cbatch_backpropagate, cnode.cpp:559-592): ``value_prefixs`` / ``values`` / ``policies``
    are the rows of the trees in ``leaf_idx_list`` (all trees when it is empty), in that order; a chance leaf's policy row has
    chance_space_size logits, a decision leaf's action_space_size.  ``to_play_batch`` and ``is_chance_list`` are indexed by
    tree; a leaf's kind follows from its depth, so ``is_chance_list`` is not read."""
    roots = results._roots
    t = roots._tree
    B, W, dev = roots.root_num, t.A, roots.device
    idx = list(range(B)) if leaf_idx_list is None or len(leaf_idx_list) == 0 else [int(i) for i in leaf_idx_list]
    if results._staged is None:
        results._staged = dict(rew=torch.zeros(B, device=dev), val=torch.zeros(B, device=dev),
                               pol=torch.zeros(B, W, device=dev), seen=np.zeros(B, bool))
    st = results._staged
    n = len(idx)
    rows = torch.as_tensor(idx, device=dev, dtype=torch.long)
    st["rew"][rows] = _to_dev(value_prefixs, torch.float32, dev, (n,))
    st["val"][rows] = _to_dev(values, torch.float32, dev, (n,))
    pol = _to_dev(policies, torch.float32, dev).reshape(n, -1)
    st["pol"][rows, :pol.shape[1]] = pol
    st["seen"][idx] = True
    if not st["seen"].all():
        return
    results._staged = None
    tp = _to_dev(to_play_batch, torch.int32, dev, (B,))
    rew, val, pol = st["rew"], st["val"], st["pol"]
    with torch.cuda.device(dev):
        cabi.check(t.lib.lz_tree_backpropagate(t.h, int(current_latent_state_index), rew.data_ptr(), val.data_ptr(),
                                               pol.data_ptr(), None, None, None, cabi.ptr(tp), cabi.stream_ptr()),
                   "lz_tree_backpropagate")
    t._keep = (rew, val, pol, tp)

