"""ctypes front-end of oracle/ctree_port.c in Stochastic MuZero mode, with the SAME module-level API as the reference's
``lzero.mcts.ctree.ctree_stochastic_muzero.stochastic_mz_tree`` (stochastic_mz_tree.pyx): ``Roots(root_num, legal_actions_list,
chance_space_size)``, ``batch_traverse`` returning ``leaf_node_is_chance`` first, and ``batch_backpropagate`` taking
``is_chance_list`` and ``leaf_idx_list`` (rows in that order, a chance leaf's policy C logits, a decision leaf's A).

Draws:
- decision-node ties: the reference draws ``rand() % len(ties)``; its compiled build under oracle/_ref is linked with
  oracle/rand_shim.c (rand() == 0), the first maximum.  ``batch_traverse(..., deterministic=False)`` after
  ``Roots.set_tie_hash`` draws with the device trees' hash instead.
- chance nodes: ``Roots.set_chance_u(u)`` pins every draw to the uniform u (``stochastic_mz_tree.chance_uniform(seed)`` is
  the reference's draw when std::random_device returns seed); without it every draw takes its uniform from the tie hash
  key (seed, epoch, tree, step, depth) of ``set_tie_hash``, the device trees' draw when ``chance_seed`` is None.

The tree is max(A, C) wide; A is taken from the first prepare's policy logits (or ``action_space_size``).

TEST INFRASTRUCTURE ONLY -- never imported by the product package ``lightzero_b200``.
"""
import ctypes

import numpy as np

from . import ctree_port as _mz
from .ctree_port import MinMaxStatsList, ResultsWrapper, _p, lib  # noqa: F401  (same classes as the MuZero front-end)


def _lib():
    L = lib()
    if not getattr(L, "_stoch_ready", False):
        P, I = ctypes.c_void_p, ctypes.c_int
        L.lzo_tree_set_stochastic.argtypes = [P, I, I]
        L.lzo_tree_set_stochastic.restype = I
        L.lzo_tree_set_chance_u.argtypes = [P, ctypes.c_double]
        L.lzo_tree_set_chance_variant.argtypes = [P, I]
        L.lzo_tree_backpropagate_stoch.argtypes = [P, I, ctypes.c_float, P, P, P, P, P, I]
        L._stoch_ready = True
    return L


class Roots(_mz.Roots):
    """stochastic_mz_tree.pyx Roots on top of the array tree in stochastic mode.  ``max_sims`` bounds the node pool."""

    def __init__(self, root_num, legal_actions_list, chance_space_size, max_sims=None, action_space_size=None):
        self.root_num = root_num
        self.C = int(chance_space_size)
        self.max_sims = max_sims or 256
        self.tie_hash = False
        self._legal_in = legal_actions_list
        self._chance_u = -1.0
        self._h = None
        if action_space_size is not None:
            self._create(int(action_space_size))

    def _create(self, A):
        self.na = A
        W = max(A, self.C)
        _mz.Roots.__init__(self, self.root_num, self._legal_in, W, self.max_sims)
        if _lib().lzo_tree_set_stochastic(self._h, A, self.C) != 0:
            raise ValueError(f"stochastic tree: width {W} does not fit A={A}, C={self.C}")
        _lib().lzo_tree_set_chance_u(self._h, self._chance_u)

    def _rows(self, policy_logits_pool):
        pol = np.asarray(policy_logits_pool, np.float32).reshape(self.root_num, -1)
        if self._h is None:
            self._create(pol.shape[1])
        return np.ascontiguousarray(np.pad(pol, ((0, 0), (0, self.A - pol.shape[1]))))

    def prepare(self, root_noise_weight, noises, value_prefix_pool, policy_logits_pool, to_play_batch):
        super().prepare(root_noise_weight, noises, value_prefix_pool, self._rows(policy_logits_pool), to_play_batch)

    def prepare_no_noise(self, value_prefix_pool, policy_logits_pool, to_play_batch):
        super().prepare_no_noise(value_prefix_pool, self._rows(policy_logits_pool), to_play_batch)

    def set_chance_u(self, u):
        """u >= 0: every chance draw takes the uniform u; u < 0 (the default): the tie hash key's uniform per draw"""
        self._chance_u = float(u)
        if self._h is not None:
            _lib().lzo_tree_set_chance_u(self._h, self._chance_u)

    def set_chance_variant(self, variant):
        """sensitivity tests only: 1 keys the chance draw at epoch + 1, 2 at step + 1, 3 at depth - 1, 4 draws h % C"""
        _lib().lzo_tree_set_chance_variant(self._h, int(variant))

    def __del__(self):
        if self._h is not None:
            super().__del__()


def batch_traverse(roots, pb_c_base, pb_c_init, discount_factor, min_max_stats_lst, results, virtual_to_play_batch,
                   deterministic=None):
    """stochastic_mz_tree.pyx batch_traverse (cnode.cpp:711-786) -> (leaf_node_is_chance, latent_state_index_in_search_path,
    latent_state_index_in_batch, last_actions, virtual_to_play_batchs).  deterministic=None: the first maximum (rand() == 0)
    unless ``roots.set_tie_hash`` was called."""
    det = (not roots.tie_hash) if deterministic is None else deterministic
    ix, iy, la, vtp = _mz.batch_traverse(roots, pb_c_base, pb_c_init, discount_factor, min_max_stats_lst, results,
                                         virtual_to_play_batch, det)
    return [bool(n & 1) for n in results.search_lens.tolist()], ix, iy, la, vtp


def batch_backpropagate(current_latent_state_index, discount_factor, value_prefixs, values, policies, min_max_stats_lst,
                        results, to_play_batch, is_chance_list, leaf_idx_list):
    """stochastic_mz_tree.pyx batch_backpropagate (cnode.cpp:559-592).  A leaf's kind follows from its depth, so
    ``is_chance_list`` is not read."""
    roots = results._roots
    B, W = roots.root_num, roots.A
    rows = list(range(B)) if len(leaf_idx_list) == 0 else [int(i) for i in leaf_idx_list]
    n = len(rows)
    pol = np.zeros((max(n, 1), W), np.float32)
    for k, p in enumerate(policies):
        p = np.asarray(p, np.float32).reshape(-1)
        pol[k, :p.size] = p
    rew = np.ascontiguousarray(np.asarray(value_prefixs, np.float32).reshape(n))
    val = np.ascontiguousarray(np.asarray(values, np.float32).reshape(n))
    tp = np.ascontiguousarray(np.asarray(to_play_batch, np.int32))
    idx = np.ascontiguousarray(np.asarray(rows, np.int32))
    _lib().lzo_tree_backpropagate_stoch(roots._h, int(current_latent_state_index), ctypes.c_float(discount_factor),
                                        _p(rew), _p(val), _p(pol), _p(tp), _p(idx), n)
