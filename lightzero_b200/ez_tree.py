"""Device-resident mirror of the reference's Cython module ``lzero.mcts.ctree.ctree_efficientzero.ez_tree``
(ez_tree.pyx): ``Roots``, ``MinMaxStatsList``, ``ResultsWrapper``, ``batch_traverse`` (no ``deterministic`` argument),
``batch_backpropagate`` (with ``is_reset_list``) -- same names, argument order and meaning as the reference.

The trees are the same CUDA trees as ``lightzero_b200.mz_tree`` switched to value-prefix semantics with
``lz_tree_set_ez`` (include/lzb200.h): ``value_prefixs`` are stored where MuZero stores rewards, every expanded node
carries ``is_reset`` and a step's reward is the prefix difference unless the parent was reset
(ctree_efficientzero/lib/cnode.cpp:185-195, 496-573, 786-790).

Tie-breaking: the reference draws ``rand() % len(ties)`` reseeded from the wall clock (cnode.cpp:691) and offers no
deterministic switch; this module always takes the first maximum, which is that draw with ``rand() == 0`` (the
configuration in which the parity tests build the unmodified reference, see DESIGN.md).
"""
from . import mz_tree as _mz
from .mz_tree import MinMaxStatsList, ResultsWrapper, _to_dev  # noqa: F401  (identical classes)


class Roots(_mz.Roots):
    """ez_tree.pyx Roots.  ``lstm_horizon_len`` is only needed by the fused search (it derives is_reset on device)."""

    def __init__(self, root_num: int, legal_actions_list, device=None, lstm_horizon_len: int = 5):
        super().__init__(root_num, legal_actions_list, device)
        self._ez, self._lstm_horizon = True, int(lstm_horizon_len)


def batch_traverse(roots: Roots, pb_c_base: int, pb_c_init: float, discount_factor: float,
                   min_max_stats_lst: MinMaxStatsList, results: ResultsWrapper, virtual_to_play_batch,
                   return_tensors: bool = False):
    """ez_tree.pyx batch_traverse -> (latent_state_index_in_search_path, latent_state_index_in_batch, last_actions,
    virtual_to_play_batch)."""
    roots._need_tree().set_params(pb_c_base, pb_c_init, discount_factor, min_max_stats_lst.value_delta_max)
    return _mz._traverse(roots, results, return_tensors)


def batch_backpropagate(current_latent_state_index: int, discount_factor: float, value_prefixs, values, policies,
                        min_max_stats_lst: MinMaxStatsList, results: ResultsWrapper, is_reset_list, to_play_batch):
    """ez_tree.pyx batch_backpropagate"""
    _mz._backpropagate(results, current_latent_state_index, value_prefixs, values, policies, to_play_batch, is_reset_list)


def batch_traverse_with_reuse(roots: Roots, pb_c_base: int, pb_c_init: float, discount_factor: float,
                              min_max_stats_lst: MinMaxStatsList, results: ResultsWrapper, virtual_to_play_batch,
                              true_action, reuse_value, return_tensors: bool = False):
    """ez_tree.pyx batch_traverse_with_reuse (ctree_efficientzero/lib/cnode.cpp:960-1072)"""
    return _mz.batch_traverse_with_reuse(roots, pb_c_base, pb_c_init, discount_factor, min_max_stats_lst, results,
                                         virtual_to_play_batch, true_action, reuse_value, return_tensors)


def batch_backpropagate_with_reuse(current_latent_state_index: int, discount_factor: float, value_prefixs, values, policies,
                                   min_max_stats_lst: MinMaxStatsList, results: ResultsWrapper, is_reset_list, to_play_batch,
                                   no_inference_lst, reuse_lst, reuse_value_lst):
    """ez_tree.pyx batch_backpropagate_with_reuse (ctree_efficientzero/lib/cnode.cpp:603-650)"""
    return _mz.batch_backpropagate_with_reuse(current_latent_state_index, discount_factor, value_prefixs, values, policies,
                                              min_max_stats_lst, results, to_play_batch, no_inference_lst, reuse_lst,
                                              reuse_value_lst, _is_reset_list=is_reset_list)
