"""ctypes front-end of oracle/ctree_port.c with the SAME module-level API as the reference's
Cython module ``lzero.mcts.ctree.ctree_muzero.mz_tree`` (mz_tree.pyx:5-107), so the restated
search loop (oracle/search_ref.py) can run on either the compiled reference (oracle/_ref) or this
port, and the two can be compared call by call.

TEST INFRASTRUCTURE ONLY -- never imported by the product package ``lightzero_b200``.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liblzoracle.so")
_lib = None


def build(force: bool = False) -> str:
    if force or not os.path.exists(_LIB_PATH) or \
            os.path.getmtime(_LIB_PATH) < os.path.getmtime(os.path.join(_HERE, "ctree_port.c")):
        os.makedirs(os.path.dirname(_LIB_PATH), exist_ok=True)
        subprocess.check_call(
            ["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
             "-o", _LIB_PATH, os.path.join(_HERE, "ctree_port.c"), "-lm"])
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(_LIB_PATH)
        P, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
        L.lzo_tree_create.restype = P
        L.lzo_tree_create.argtypes = [I, I, I]
        L.lzo_tree_destroy.argtypes = [P]
        L.lzo_tree_reset.argtypes = [P, P, P]
        L.lzo_tree_minmax_reset.argtypes = [P, F]
        L.lzo_tree_prepare.argtypes = [P, F, P, P, P, P]
        L.lzo_tree_traverse.argtypes = [P, I, F, F, P, I, P, P, P, P]
        L.lzo_tree_backpropagate.argtypes = [P, I, F, P, P, P, P]
        L.lzo_tree_distributions.argtypes = [P, P, P]
        L.lzo_tree_values.argtypes = [P, P]
        L.lzo_tree_trajectories.argtypes = [P, P, P]
        L.lzo_tree_seed.argtypes = [P, ctypes.c_uint]
        L.lzo_tree_traverse_with_reuse.argtypes = [P, I, F, F, P, P, P, P, P, P, P]
        L.lzo_tree_backpropagate_with_reuse.argtypes = [P, I, F, P, P, P, P, P, P, P]
        L.lzo_tree_set_tie_hash.argtypes = [P, ctypes.c_uint64, ctypes.c_uint64]
        L.lzo_tree_set_tie_step.argtypes = [P, ctypes.c_uint]
        L.lzo_tree_set_tie_variant.argtypes = [P, I]
        L.lzo_tree_tie_stats_reset.argtypes = [P]
        L.lzo_tree_tie_stats.argtypes = [P, P]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


class MinMaxStatsList:
    """mz_tree.pyx:5-15.  The port keeps min/max inside the tree; this object only carries delta
    and (re)initialises the stats of the Roots it is first used with."""

    def __init__(self, num):
        self.num = num
        self.delta = 0.0
        self._bound = None

    def set_delta(self, value_delta_max):
        self.delta = float(value_delta_max)

    def _bind(self, roots):
        if self._bound is not roots:
            lib().lzo_tree_minmax_reset(roots._h, ctypes.c_float(self.delta))
            self._bound = roots


class ResultsWrapper:
    """mz_tree.pyx:17-24"""

    def __init__(self, num):
        self.num = num
        self.search_lens = None

    def get_search_len(self):
        return self.search_lens.tolist()


class Roots:
    """mz_tree.pyx:26-59 on top of the array tree.  max_sims bounds the node pool."""

    def __init__(self, root_num, legal_actions_list, action_space_size=None, max_sims=None):
        self.root_num = root_num
        A = action_space_size or (max(max(l) for l in legal_actions_list if len(l)) + 1)
        self.A = A
        self.max_sims = max_sims or 256
        self.tie_hash = False
        self._h = lib().lzo_tree_create(root_num, A, self.max_sims)
        legal = np.full((root_num, A), -1, np.int32)
        nlegal = np.zeros(root_num, np.int32)
        for i, l in enumerate(legal_actions_list):
            nlegal[i] = len(l)
            legal[i, :len(l)] = l
        self._legal, self._nlegal = legal, nlegal
        lib().lzo_tree_reset(self._h, _p(legal), _p(nlegal))

    def _grow_action_space(self, A):
        if A != self.A:
            raise ValueError("action space mismatch: construct Roots(action_space_size=...)")

    def prepare(self, root_noise_weight, noises, value_prefix_pool, policy_logits_pool, to_play_batch):
        A = self.A
        pol = np.ascontiguousarray(np.asarray(policy_logits_pool, np.float32).reshape(self.root_num, A))
        nz = np.zeros((self.root_num, A), np.float32)
        for i, n in enumerate(noises):
            nz[i, :len(n)] = n
        rew = np.ascontiguousarray(np.asarray(value_prefix_pool, np.float32))
        tp = np.ascontiguousarray(np.asarray(to_play_batch, np.int32))
        lib().lzo_tree_prepare(self._h, ctypes.c_float(root_noise_weight), _p(nz), _p(rew), _p(pol), _p(tp))

    def prepare_no_noise(self, value_prefix_pool, policy_logits_pool, to_play_batch):
        A = self.A
        pol = np.ascontiguousarray(np.asarray(policy_logits_pool, np.float32).reshape(self.root_num, A))
        rew = np.ascontiguousarray(np.asarray(value_prefix_pool, np.float32))
        tp = np.ascontiguousarray(np.asarray(to_play_batch, np.int32))
        lib().lzo_tree_prepare(self._h, ctypes.c_float(0.0), None, _p(rew), _p(pol), _p(tp))

    def get_distributions(self):
        out = np.empty((self.root_num, self.A), np.int32)
        nl = np.empty(self.root_num, np.int32)
        lib().lzo_tree_distributions(self._h, _p(out), _p(nl))
        return [out[i, :nl[i]].tolist() for i in range(self.root_num)]

    def get_values(self):
        out = np.empty(self.root_num, np.float32)
        lib().lzo_tree_values(self._h, _p(out))
        return out.tolist()

    def get_values_f32(self):
        out = np.empty(self.root_num, np.float32)
        lib().lzo_tree_values(self._h, _p(out))
        return out

    def get_trajectories(self):
        N = self.max_sims + 1
        out = np.empty((self.root_num, N), np.int32)
        ln = np.empty(self.root_num, np.int32)
        lib().lzo_tree_trajectories(self._h, _p(out), _p(ln))
        return [out[i, :ln[i]].tolist() for i in range(self.root_num)]

    def set_tie_hash(self, seed, epoch, step=0, variant=0):
        """Hash mode: non-deterministic descents draw from the tie list with the device trees' counter-based hash keyed by
        (seed, epoch, tree, step, depth) instead of rand().  ``step`` is the step of the next traverse (each traverse
        consumes one).  ``variant`` is for sensitivity tests: 1 always draws the first tie, 2 draws the tie after the hashed one.
        Also clears the tie statistics."""
        L = lib()
        L.lzo_tree_set_tie_hash(self._h, int(seed) & (2 ** 64 - 1), int(epoch) & (2 ** 64 - 1))
        L.lzo_tree_set_tie_step(self._h, int(step) & (2 ** 32 - 1))
        L.lzo_tree_set_tie_variant(self._h, int(variant))
        L.lzo_tree_tie_stats_reset(self._h)
        self.tie_hash = True

    def tie_stats(self):
        """descents with more than one tie, hash draws other than the first tie, tie lists with unequal scores (near ties),
        longest search path, chance draws over two or more outcomes (Stochastic MuZero trees)"""
        out = np.zeros(5, np.int64)
        lib().lzo_tree_tie_stats(self._h, _p(out))
        return dict(ties=int(out[0]), draws=int(out[1]), near=int(out[2]), max_len=int(out[3]), chance=int(out[4]))

    def clear(self):
        pass

    @property
    def num(self):
        return self.root_num

    def __del__(self):
        try:
            lib().lzo_tree_destroy(self._h)
        except Exception:
            pass


def batch_traverse(roots, pb_c_base, pb_c_init, discount_factor, min_max_stats_lst, results,
                   virtual_to_play_batch, deterministic=False):
    """mz_tree.pyx:94-99"""
    min_max_stats_lst._bind(roots)
    B = roots.root_num
    vtp = np.ascontiguousarray(np.asarray(virtual_to_play_batch, np.int32))
    ix = np.empty(B, np.int32); iy = np.empty(B, np.int32)
    la = np.empty(B, np.int32); sl = np.empty(B, np.int32)
    lib().lzo_tree_traverse(roots._h, int(pb_c_base), ctypes.c_float(pb_c_init), ctypes.c_float(discount_factor),
                            _p(vtp), int(bool(deterministic)), _p(ix), _p(iy), _p(la), _p(sl))
    results.search_lens = sl
    results._roots = roots
    return ix.tolist(), iy.tolist(), la.tolist(), vtp.tolist()


def batch_backpropagate(current_latent_state_index, discount_factor, value_prefixs, values, policies,
                        min_max_stats_lst, results, to_play_batch):
    """mz_tree.pyx:73-82"""
    roots = results._roots
    B, A = roots.root_num, roots.A
    rew = np.ascontiguousarray(np.asarray(value_prefixs, np.float32))
    val = np.ascontiguousarray(np.asarray(values, np.float32))
    pol = np.ascontiguousarray(np.asarray(policies, np.float32).reshape(B, A))
    tp = np.ascontiguousarray(np.asarray(to_play_batch, np.int32))
    lib().lzo_tree_backpropagate(roots._h, int(current_latent_state_index), ctypes.c_float(discount_factor),
                                 _p(rew), _p(val), _p(pol), _p(tp))


def batch_traverse_with_reuse(roots, pb_c_base, pb_c_init, discount_factor, min_max_stats_lst, results,
                              virtual_to_play_batch, true_action, reuse_value):
    """mz_tree.pyx batch_traverse_with_reuse (cnode.cpp:828-932); ties as with rand() == 0"""
    min_max_stats_lst._bind(roots)
    B = roots.root_num
    vtp = np.ascontiguousarray(np.asarray(virtual_to_play_batch, np.int32))
    ta = np.ascontiguousarray(np.asarray(true_action, np.int32))
    rv = np.ascontiguousarray(np.asarray(reuse_value, np.float32))
    ix = np.empty(B, np.int32); iy = np.empty(B, np.int32)
    la = np.empty(B, np.int32); sl = np.empty(B, np.int32)
    lib().lzo_tree_traverse_with_reuse(roots._h, int(pb_c_base), ctypes.c_float(pb_c_init), ctypes.c_float(discount_factor),
                                       _p(vtp), _p(ta), _p(rv), _p(ix), _p(iy), _p(la), _p(sl))
    results.search_lens = sl
    results._roots = roots
    return ix.tolist(), iy.tolist(), la.tolist(), vtp.tolist()


def batch_backpropagate_with_reuse(current_latent_state_index, discount_factor, value_prefixs, values, policies,
                                   min_max_stats_lst, results, to_play_batch, no_inference_lst, reuse_lst, reuse_value_lst):
    """mz_tree.pyx batch_backpropagate_with_reuse (cnode.cpp:502-549): compacted network outputs + the driver's index lists"""
    roots = results._roots
    B, A = roots.root_num, roots.A
    n = len(value_prefixs)
    rew = np.ascontiguousarray(np.asarray(value_prefixs, np.float32).reshape(n))
    val = np.ascontiguousarray(np.asarray(values, np.float32).reshape(n))
    pol = np.ascontiguousarray(np.asarray(policies, np.float32).reshape(n, A)) if n else np.zeros((1, A), np.float32)
    tp = np.ascontiguousarray(np.asarray(to_play_batch, np.int32))
    ni = np.ascontiguousarray(np.asarray(no_inference_lst, np.int32))
    ru = np.ascontiguousarray(np.asarray(reuse_lst, np.int32))
    rv = np.ascontiguousarray(np.asarray(reuse_value_lst, np.float32))
    lib().lzo_tree_backpropagate_with_reuse(roots._h, int(current_latent_state_index), ctypes.c_float(discount_factor),
                                            _p(rew), _p(val), _p(pol), _p(tp), _p(ni), _p(ru), _p(rv))
