"""ctypes front-end of oracle/ctree_port.c in EfficientZero mode, with the SAME module-level API as the reference's
``lzero.mcts.ctree.ctree_efficientzero.ez_tree`` (ez_tree.pyx): ``batch_traverse`` has no ``deterministic`` argument and
``batch_backpropagate`` takes ``is_reset_list``.

Tie-breaking: the reference draws ``rand() % len(ties)``; the compiled reference under oracle/_ref is linked with
oracle/rand_shim.c (rand() == 0), which is element 0 of the tie list = this port's deterministic rule.  After
``Roots.set_tie_hash`` the descents draw with the device trees' hash instead (``lz_tree_set_tiebreak(t, 0)``).

TEST INFRASTRUCTURE ONLY -- never imported by the product package ``lightzero_b200``.
"""
import ctypes

import numpy as np

from . import ctree_port as _mz
from .ctree_port import MinMaxStatsList, ResultsWrapper, _p, lib  # noqa: F401  (same classes as the MuZero front-end)


def _lib():
    L = lib()
    if not getattr(L, "_ez_ready", False):
        P, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
        L.lzo_tree_set_ez.argtypes = [P, I]
        L.lzo_tree_backpropagate_ez.argtypes = [P, I, F, P, P, P, P, P]
        L.lzo_tree_backpropagate_with_reuse_ez.argtypes = [P, I, F, P, P, P, P, P, P, P, P]
        L._ez_ready = True
    return L


class Roots(_mz.Roots):
    """ez_tree.pyx Roots on top of the array tree in value-prefix mode."""

    def __init__(self, root_num, legal_actions_list, action_space_size=None, max_sims=None):
        super().__init__(root_num, legal_actions_list, action_space_size, max_sims)
        _lib().lzo_tree_set_ez(self._h, 1)


def batch_traverse(roots, pb_c_base, pb_c_init, discount_factor, min_max_stats_lst, results, virtual_to_play_batch):
    """ez_tree.pyx batch_traverse (ctree_efficientzero/lib/cnode.cpp:876-958): first maximum (rand() == 0), or the hashed
    draw once ``roots.set_tie_hash`` was called"""
    return _mz.batch_traverse(roots, pb_c_base, pb_c_init, discount_factor, min_max_stats_lst, results,
                              virtual_to_play_batch, not roots.tie_hash)


def batch_backpropagate(current_latent_state_index, discount_factor, value_prefixs, values, policies,
                        min_max_stats_lst, results, is_reset_list, to_play_batch):
    """ez_tree.pyx batch_backpropagate (ctree_efficientzero/lib/cnode.cpp:577-601)"""
    roots = results._roots
    B, A = roots.root_num, roots.A
    vp = np.ascontiguousarray(np.asarray(value_prefixs, np.float32))
    val = np.ascontiguousarray(np.asarray(values, np.float32))
    pol = np.ascontiguousarray(np.asarray(policies, np.float32).reshape(B, A))
    rs = np.ascontiguousarray(np.asarray(is_reset_list, np.int32))
    tp = np.ascontiguousarray(np.asarray(to_play_batch, np.int32))
    _lib().lzo_tree_backpropagate_ez(roots._h, int(current_latent_state_index), ctypes.c_float(discount_factor),
                                     _p(vp), _p(val), _p(pol), _p(rs), _p(tp))


def batch_traverse_with_reuse(roots, pb_c_base, pb_c_init, discount_factor, min_max_stats_lst, results, virtual_to_play_batch,
                              true_action, reuse_value):
    """ez_tree.pyx batch_traverse_with_reuse (ctree_efficientzero/lib/cnode.cpp:960-1072)"""
    return _mz.batch_traverse_with_reuse(roots, pb_c_base, pb_c_init, discount_factor, min_max_stats_lst, results,
                                         virtual_to_play_batch, true_action, reuse_value)


def batch_backpropagate_with_reuse(current_latent_state_index, discount_factor, value_prefixs, values, policies, min_max_stats_lst,
                                   results, is_reset_list, to_play_batch, no_inference_lst, reuse_lst, reuse_value_lst):
    """ez_tree.pyx batch_backpropagate_with_reuse (ctree_efficientzero/lib/cnode.cpp:603-650)"""
    roots = results._roots
    B, A = roots.root_num, roots.A
    n = len(value_prefixs)
    vp = np.ascontiguousarray(np.asarray(value_prefixs, np.float32).reshape(n))
    val = np.ascontiguousarray(np.asarray(values, np.float32).reshape(n))
    pol = np.ascontiguousarray(np.asarray(policies, np.float32).reshape(n, A)) if n else np.zeros((1, A), np.float32)
    rs = np.ascontiguousarray(np.asarray(is_reset_list, np.int32))
    tp = np.ascontiguousarray(np.asarray(to_play_batch, np.int32))
    ni = np.ascontiguousarray(np.asarray(no_inference_lst, np.int32))
    ru = np.ascontiguousarray(np.asarray(reuse_lst, np.int32))
    rv = np.ascontiguousarray(np.asarray(reuse_value_lst, np.float32))
    _lib().lzo_tree_backpropagate_with_reuse_ez(roots._h, int(current_latent_state_index), ctypes.c_float(discount_factor),
                                                _p(vp), _p(val), _p(pol), _p(rs), _p(tp), _p(ni), _p(ru), _p(rv))
