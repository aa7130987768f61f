"""Device-resident mirror of the reference's Cython module ``lzero.mcts.ctree.ctree_muzero.mz_tree``
(mz_tree.pyx:5-107): ``Roots``, ``MinMaxStatsList``, ``ResultsWrapper``, ``batch_traverse``,
``batch_backpropagate`` with the same names, argument order and meaning.  Every list argument may
also be a numpy array or a CUDA tensor (which avoids the host round trip).  State lives in the CUDA
trees behind ``lz_tree_*`` (include/lzb200.h); nothing here computes on the CPU.

Differences a caller can observe:
  * list outputs are materialised with ONE device->host copy when asked for (``get_distributions``,
    ``get_values``, the tuple returned by ``batch_traverse``); ``*_tensor`` variants stay on device;
  * ``MinMaxStatsList`` is bookkeeping only -- min/max live inside the tree and are reset when the
    Roots are (re)prepared, i.e. once per search like mcts_ctree.py:291-292.
"""
import contextlib
import threading
from typing import List, Optional

import numpy as np
import torch

from . import cabi

DEFAULT_MAX_SIMS = 64     # node-pool capacity when a Roots is driven step-wise without a known budget
_tree_pool = {}           # (device index, B, A, max_sims) -> [TreeHandle]
_pool_lock = threading.Lock()


class TreeHandle:
    """Owns one lz_tree (+ lazily one lz_search per model) and its scratch tensors."""

    def __init__(self, device, B, A, max_sims):
        self.device, self.B, self.A, self.max_sims = device, B, A, max_sims
        self.lib = cabi.load()
        h = cabi.c_void_p()
        with torch.cuda.device(device):
            cabi.check(self.lib.lz_tree_create(B, A, max_sims, h), "lz_tree_create")
        self.h = h
        self.busy = False
        self.params = None
        self._released = None  # CUDA event recorded where the last holder let go: its searches / read-outs may still be queued
        i32 = dict(dtype=torch.int32, device=device)
        self.ix, self.iy, self.action = (torch.empty(B, **i32) for _ in range(3))
        self.search_len, self.vtp = torch.empty(B, **i32), torch.empty(B, **i32)
        self.visits = torch.empty(B, A, **i32)
        self.nlegal = torch.empty(B, **i32)
        self.values = torch.empty(B, dtype=torch.float32, device=device)
        self.traj = torch.empty(B, max_sims + 1, **i32)
        self.searches = {}    # (model serial, num_simulations, mode...) -> lz_search handle; dropped when the model dies

    def set_params(self, pb_c_base, pb_c_init, discount, delta):
        p = (int(pb_c_base), float(pb_c_init), float(discount), float(delta))
        if p != self.params:
            # lz_tree_set_params rewrites the pb_c table on the library's setup stream, which no caller stream is ordered
            # against: first wait, on the host, for every search that may still read it -- the earlier holders' (the release
            # event) and this holder's own queued work (the current stream)
            with torch.cuda.device(self.device):
                if self._released is not None:
                    self._released.synchronize()
                torch.cuda.current_stream(self.device).synchronize()
                cabi.check(self.lib.lz_tree_set_params(self.h, *p), "lz_tree_set_params")
            self.params = p

    def set_mode(self, mode=(), deterministic: bool = True, gumbel=(0, 0), stochastic=(0, 0, -1.0)):
        """Puts the tree in one holder's whole mode: ``mode`` () for MuZero or (1, lstm_horizon_len) for EfficientZero
        value-prefix trees (the ``search_for`` mode), ``gumbel`` (max_num_considered_actions, num_simulations) for a Gumbel
        tree, ``stochastic`` (action_space_size, chance_space_size, chance_u) for a Stochastic MuZero tree
        (lz_tree_set_stochastic), and the tie rule of the EfficientZero and *_with_reuse descents (``deterministic``: the first
        maximum, else the uniform draw).  The mode is C state that outlives its holder, so every acquirer sets all of it,
        once: a change bumps the tree's generation and re-captures its search graphs (csrc/search.cu)."""
        if not stochastic[1]:       # first: the EfficientZero and Gumbel modes refuse a stochastic tree
            cabi.check(self.lib.lz_tree_set_stochastic(self.h, 0, 0, -1.0), "lz_tree_set_stochastic")
        if gumbel[1]:       # a Gumbel tree is a MuZero tree
            cabi.check(self.lib.lz_tree_set_ez(self.h, 0, 5), "lz_tree_set_ez")
            cabi.check(self.lib.lz_tree_set_gumbel(self.h, int(gumbel[0]), int(gumbel[1])), "lz_tree_set_gumbel")
        else:
            cabi.check(self.lib.lz_tree_set_gumbel(self.h, 0, 0), "lz_tree_set_gumbel")
            cabi.check(self.lib.lz_tree_set_ez(self.h, *(mode or (0, 5))), "lz_tree_set_ez")
        if stochastic[1]:
            cabi.check(self.lib.lz_tree_set_stochastic(self.h, int(stochastic[0]), int(stochastic[1]), float(stochastic[2])),
                       "lz_tree_set_stochastic")
        cabi.check(self.lib.lz_tree_set_tiebreak(self.h, int(bool(deterministic))), "lz_tree_set_tiebreak")

    def release(self):
        """Hands the tree back to the pool.  The holder's work on it may still be queued on the current stream (a
        search_batch(read_back=False), Roots.clear() before the read-outs ran): the event recorded here orders the next
        holder after it (acquire_tree, set_params)."""
        with torch.cuda.device(self.device):
            if self._released is None:
                self._released = torch.cuda.Event()
            self._released.record(torch.cuda.current_stream(self.device))
        self.busy = False

    def search_for(self, model, num_simulations, mode=()):
        # keyed by the model's serial (unique for the life of the process; id() is recycled after garbage collection).  The
        # captured graph is re-captured inside the library when the model's weights / math mode or this tree's parameters
        # change (generation counters, csrc/search.cu), so one lz_search per (model, num_simulations, mode) is enough
        key = (model._serial, num_simulations) + tuple(mode)     # mode: (ez, lstm_horizon_len)
        if key not in self.searches:
            q = cabi.c_void_p()
            with torch.cuda.device(self.device):
                cabi.check(self.lib.lz_search_create(self.h, model._h, num_simulations, q), "lz_search_create")
            self.searches[key] = q
        return self.searches[key]

    def __del__(self):
        try:
            for q in self.searches.values():
                self.lib.lz_search_destroy(q)
            self.lib.lz_tree_destroy(self.h)
        except Exception:
            pass


def acquire_tree(device, B, A, max_sims) -> TreeHandle:
    """A free pooled tree of this shape, or a new one.  The current stream waits for the work the last holder queued on it
    (TreeHandle.release), so two holders on two streams never use one tree, its searches or its scratch at the same time."""
    key = (device.index, B, A, max_sims)
    with _pool_lock:
        for h in _tree_pool.setdefault(key, []):
            if not h.busy:
                h.busy = True
                if h._released is not None:
                    torch.cuda.current_stream(device).wait_event(h._released)
                return h
        h = TreeHandle(device, B, A, max_sims)
        h.busy = True
        _tree_pool[key].append(h)
        return h


@contextlib.contextmanager
def held_tree(device, B, A, max_sims, params, mode=(), deterministic: bool = True, gumbel=(0, 0), stochastic=(0, 0, -1.0)):
    """A pooled tree with these parameters and this whole mode (TreeHandle.set_mode) for the length of one call, released
    at its end even when the call raises.  ``A`` is the tree's width: max(action_space_size, chance_space_size) for a
    ``stochastic`` (action_space_size, chance_space_size, chance_u) tree."""
    t = acquire_tree(device, B, A, max_sims)
    try:
        t.set_params(*params)
        t.set_mode(mode, deterministic, gumbel, stochastic)
        yield t
    finally:
        t.release()


def drop_model_searches(serial: int):
    """Called when a model wrapper is destroyed: destroys every lz_search bound to that lz_model (they hold its pointer and
    graphs captured against its device tables)."""
    with _pool_lock:
        handles = [h for hs in _tree_pool.values() for h in hs]
    for h in handles:
        for key in [k for k in h.searches if k[0] == serial]:
            q = h.searches.pop(key)
            try:
                h.lib.lz_search_destroy(q)
            except Exception:
                pass


def _to_dev(x, dtype, device, shape=None):
    if x is None:
        return None
    if isinstance(x, torch.Tensor):
        t = x.to(device=device, dtype=dtype, non_blocking=True)
    else:
        t = torch.from_numpy(np.ascontiguousarray(np.asarray(x, dtype={torch.float32: np.float32, torch.int32: np.int32,
                                                                       torch.uint8: np.uint8}[dtype]))).to(device, non_blocking=True)
    if shape is not None:
        t = t.reshape(shape)
    return t.contiguous()


class MinMaxStatsList:
    """mz_tree.pyx:5-15"""

    def __init__(self, num: int):
        self.num = num
        self.value_delta_max = 0.0

    def set_delta(self, value_delta_max: float):
        self.value_delta_max = float(value_delta_max)


class ResultsWrapper:
    """mz_tree.pyx:17-24"""

    def __init__(self, num: int):
        self.num = num
        self._roots = None

    def get_search_len(self) -> List[int]:
        return self._roots._tree.search_len.cpu().tolist()


class Roots:
    """mz_tree.pyx:26-59.  ``legal_actions_list``: list of lists (any order), or a uint8/bool mask
    tensor/array [root_num, A]."""

    def __init__(self, root_num: int, legal_actions_list, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("lightzero_b200.mz_tree.Roots needs a CUDA device; there is no CPU fallback")
        self.root_num = root_num
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._legal_lists = None
        self._mask = None
        self._mask_dev = None
        if isinstance(legal_actions_list, (torch.Tensor, np.ndarray)) and np.ndim(legal_actions_list) == 2 and \
                str(legal_actions_list.dtype).split(".")[-1] in ("uint8", "bool"):
            self._mask = legal_actions_list
        else:
            self._legal_lists = [list(l) for l in legal_actions_list]
            assert len(self._legal_lists) == root_num
        self._pending = None      # prepare() arguments until the tree is materialised
        self._values = None       # root value estimates of a Gumbel tree's prepare (set by gmz_tree.Roots)
        self._ez, self._lstm_horizon = False, 5     # EfficientZero value-prefix semantics (set by ez_tree.Roots)
        self._deterministic = True     # tie rule of the EfficientZero / *_with_reuse descents (the mirrors: first maximum)
        self._stochastic = (0, 0, -1.0)     # Stochastic MuZero tree mode (set by stochastic_mz_tree.Roots)
        self._tree: Optional[TreeHandle] = None
        self._delta_reset = None

    # ---- reference API ---------------------------------------------------------------------------
    def prepare(self, root_noise_weight: float, noises, value_prefix_pool, policy_logits_pool, to_play_batch):
        self._stage(float(root_noise_weight), noises, value_prefix_pool, policy_logits_pool, to_play_batch)

    def prepare_no_noise(self, value_prefix_pool, policy_logits_pool, to_play_batch):
        self._stage(0.0, None, value_prefix_pool, policy_logits_pool, to_play_batch)

    def get_distributions(self) -> List[List[int]]:
        v, n = self.get_distributions_tensor()
        v, n = v.cpu().numpy(), n.cpu().numpy()
        return [v[i, :n[i]].tolist() for i in range(self.root_num)]

    def get_values(self) -> List[float]:
        return self.get_values_tensor().cpu().tolist()

    def get_trajectories(self) -> List[List[int]]:
        t = self._need_tree()
        with torch.cuda.device(self.device):
            cabi.check(t.lib.lz_tree_results(t.h, None, None, None, t.traj.data_ptr(), cabi.stream_ptr()), "lz_tree_results")
        tr = t.traj.cpu().numpy()
        return [row[row >= 0].tolist() for row in tr]

    def clear(self):
        if self._tree is not None:
            self._tree.release()
            self._tree = None

    @property
    def num(self) -> int:
        return self.root_num

    def __del__(self):
        try:
            self.clear()
        except Exception:
            pass

    # ---- device-side extras ----------------------------------------------------------------------
    def get_distributions_tensor(self):
        """(visits int32 [B,A] in legal order, -1 padded; nlegal int32 [B]) on device."""
        t = self._need_tree()
        with torch.cuda.device(self.device):
            cabi.check(t.lib.lz_tree_results(t.h, t.visits.data_ptr(), t.values.data_ptr(), t.nlegal.data_ptr(), None,
                                             cabi.stream_ptr()), "lz_tree_results")
        return t.visits, t.nlegal

    def select_action_tensor(self, temperature: float = 1.0, deterministic: bool = False, seed: int = 0):
        """lzero/policy/utils.py:637-661 for every root on the device -> (action id, position in the legal list, entropy)."""
        t = self._need_tree()
        act = torch.empty(self.root_num, dtype=torch.int32, device=self.device)
        pos = torch.empty(self.root_num, dtype=torch.int32, device=self.device)
        ent = torch.empty(self.root_num, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            cabi.check(t.lib.lz_tree_select_action(t.h, float(temperature), int(bool(deterministic)), int(seed) & (2 ** 64 - 1),
                                                   act.data_ptr(), pos.data_ptr(), ent.data_ptr(), cabi.stream_ptr()),
                       "lz_tree_select_action")
        return act, pos, ent

    def get_values_tensor(self):
        t = self._need_tree()
        with torch.cuda.device(self.device):
            cabi.check(t.lib.lz_tree_results(t.h, None, t.values.data_ptr(), None, None, cabi.stream_ptr()), "lz_tree_results")
        return t.values

    # ---- internals -------------------------------------------------------------------------------
    def _stage(self, w, noises, rewards, policies, to_play):
        B = self.root_num
        pol = _to_dev(policies, torch.float32, self.device)
        pol = pol.reshape(B, -1).contiguous()
        A = pol.shape[1]
        nz = None
        if noises is not None:
            if isinstance(noises, (torch.Tensor, np.ndarray)):
                nz = _to_dev(noises, torch.float32, self.device, (B, A))
            else:   # list of per-root lists in legal order (policy/muzero.py:763-766)
                arr = np.zeros((B, A), np.float32)
                for i, n in enumerate(noises):
                    arr[i, :len(n)] = n
                nz = torch.from_numpy(arr).to(self.device, non_blocking=True)
        rew = None
        if rewards is not None and not (isinstance(rewards, list) and all(r == 0 for r in rewards)):
            rew = _to_dev(rewards, torch.float32, self.device, (B,))
        tp = _to_dev(to_play, torch.int32, self.device, (B,)) if to_play is not None else None
        self._pending = dict(w=w, noise=nz, rewards=rew, logits=pol, to_play=tp, A=A)
        if self._tree is not None:      # re-prepare of an already materialised tree
            self._materialize(self._tree.max_sims)

    def _need_tree(self) -> TreeHandle:
        if self._tree is None:
            self._materialize(DEFAULT_MAX_SIMS)
        return self._tree

    def _materialize(self, max_sims: int, params=None, deterministic=None):
        """Reset + prepare on device in a pooled tree of at least max_sims simulations.  ``deterministic``: the tie rule the
        holder searches with (MCTS searches pass their own); None keeps these roots' rule."""
        self._reset_and_prepare(self._acquire(max_sims, params, deterministic))

    def _reset_and_prepare(self, t):
        """Reset tree t to the legal lists and lz_tree_prepare it: a fresh search on these roots."""
        p = self._pending
        with torch.cuda.device(self.device):
            s = cabi.stream_ptr()
            self._reset_tree(t, s)
            cabi.check(t.lib.lz_tree_prepare(t.h, p["logits"].data_ptr(), cabi.ptr(p["noise"]), p["w"], cabi.ptr(p["rewards"]),
                                             cabi.ptr(self._values), cabi.ptr(p["to_play"]), s), "lz_tree_prepare")

    def _acquire(self, max_sims, params, deterministic, gumbel=(0, 0)) -> TreeHandle:
        """This Roots' pooled tree, at least max_sims deep and in its whole mode (TreeHandle.set_mode)."""
        if self._pending is None:
            raise RuntimeError("Roots: prepare()/prepare_no_noise() has not been called")
        A = self._pending["A"]
        if self._tree is not None and (self._tree.max_sims < max_sims or self._tree.A != A):
            self.clear()
        if self._tree is None:
            self._tree = acquire_tree(self.device, self.root_num, A, max_sims)
        if deterministic is not None:
            self._deterministic = bool(deterministic)
        t = self._tree
        if params is not None:
            t.set_params(*params)
        with torch.cuda.device(self.device):
            t.set_mode((1, int(self._lstm_horizon)) if self._ez else (), self._deterministic, gumbel, self._stochastic)
        return t

    def _reset_tree(self, t, s):
        """lz_tree_reset / lz_tree_reset_mask of tree t to these roots' legal actions, on stream s."""
        A = self._pending["A"]
        with torch.cuda.device(self.device):
            if self._mask is not None:
                if self._mask_dev is None:      # uploaded once per Roots, not once per search
                    self._mask_dev = _to_dev(self._mask, torch.uint8, self.device, (self.root_num, A))
                cabi.check(t.lib.lz_tree_reset_mask(t.h, self._mask_dev.data_ptr(), s), "lz_tree_reset_mask")
            else:
                identity = list(range(A))
                if all(l == identity for l in self._legal_lists):
                    cabi.check(t.lib.lz_tree_reset(t.h, None, None, s), "lz_tree_reset")
                else:
                    legal = np.full((self.root_num, A), -1, np.int32)
                    nl = np.zeros(self.root_num, np.int32)
                    for i, l in enumerate(self._legal_lists):
                        nl[i] = len(l)
                        legal[i, :len(l)] = l
                    dl = torch.from_numpy(legal).to(self.device)
                    dn = torch.from_numpy(nl).to(self.device)
                    cabi.check(t.lib.lz_tree_reset(t.h, dl.data_ptr(), dn.data_ptr(), s), "lz_tree_reset")
                    self._keep = (dl, dn)


def _traverse(roots: Roots, results: ResultsWrapper, return_tensors: bool, deterministic=False, true_action=None,
              reuse_value=None):
    """lz_tree_traverse of the roots' tree, the descent of its mode (reuse with true_action / reuse_value), and what every
    batch_traverse returns: (latent_state_index_in_search_path, latent_state_index_in_batch, last_actions,
    virtual_to_play_batch) as lists, or the device tensors."""
    t = roots._tree
    dev = roots.device
    ta = _to_dev(true_action, torch.int32, dev, (roots.root_num,))
    rv = _to_dev(reuse_value, torch.float32, dev, (roots.root_num,))
    with torch.cuda.device(dev):
        cabi.check(t.lib.lz_tree_traverse(t.h, int(bool(deterministic)), cabi.ptr(ta), cabi.ptr(rv), t.ix.data_ptr(),
                                          t.iy.data_ptr(), t.action.data_ptr(), t.search_len.data_ptr(), t.vtp.data_ptr(),
                                          None, cabi.stream_ptr()), "lz_tree_traverse")
    if rv is not None:
        t._keep = (ta, rv)
    results._roots = roots
    if return_tensors:
        return t.ix, t.iy, t.action, t.vtp
    return tuple(x.tolist() for x in torch.stack((t.ix, t.iy, t.action, t.vtp)).cpu().numpy())


def _backpropagate(results: ResultsWrapper, current_latent_state_index: int, value_prefixs, values, policies, to_play_batch,
                   is_reset_list=None):
    """lz_tree_backpropagate of the tree the last batch_traverse descended, the back-up of its mode, on the inputs every
    batch_backpropagate stages on the device: rewards (value prefixes on an EfficientZero tree, with is_reset_list), values,
    policy logits, to_play or None."""
    roots = results._roots
    t = roots._tree
    B, A, dev = roots.root_num, t.A, roots.device
    rew, val = _to_dev(value_prefixs, torch.float32, dev, (B,)), _to_dev(values, torch.float32, dev, (B,))
    pol, tp = _to_dev(policies, torch.float32, dev, (B, A)), _to_dev(to_play_batch, torch.int32, dev, (B,))
    rs = _to_dev(is_reset_list, torch.int32, dev, (B,))
    with torch.cuda.device(dev):
        cabi.check(t.lib.lz_tree_backpropagate(t.h, int(current_latent_state_index), rew.data_ptr(), val.data_ptr(),
                                               pol.data_ptr(), None, None, cabi.ptr(rs), cabi.ptr(tp), cabi.stream_ptr()),
                   "lz_tree_backpropagate")
    t._keep = (rew, val, pol, rs, tp)


def batch_traverse(roots: Roots, pb_c_base: int, pb_c_init: float, discount_factor: float,
                   min_max_stats_lst: MinMaxStatsList, results: ResultsWrapper, virtual_to_play_batch,
                   deterministic: bool = False, return_tensors: bool = False):
    """mz_tree.pyx:94-99 -> (latent_state_index_in_search_path, latent_state_index_in_batch, last_actions,
    virtual_to_play_batch)."""
    roots._need_tree().set_params(pb_c_base, pb_c_init, discount_factor, min_max_stats_lst.value_delta_max)
    return _traverse(roots, results, return_tensors, deterministic)


def batch_backpropagate(current_latent_state_index: int, discount_factor: float, value_prefixs, values, policies,
                        min_max_stats_lst: MinMaxStatsList, results: ResultsWrapper, to_play_batch):
    """mz_tree.pyx:73-82"""
    _backpropagate(results, current_latent_state_index, value_prefixs, values, policies, to_play_batch)


def batch_traverse_with_reuse(roots: Roots, pb_c_base: int, pb_c_init: float, discount_factor: float,
                              min_max_stats_lst: MinMaxStatsList, results: ResultsWrapper, virtual_to_play_batch,
                              true_action, reuse_value, return_tensors: bool = False):
    """mz_tree.pyx batch_traverse_with_reuse (cnode.cpp:828-932): ``latent_state_index_in_search_path`` is -1 for trees
    that stopped on an already expanded child of the root (no inference needed)."""
    roots._need_tree().set_params(pb_c_base, pb_c_init, discount_factor, min_max_stats_lst.value_delta_max)
    return _traverse(roots, results, return_tensors, true_action=true_action, reuse_value=reuse_value)


def batch_backpropagate_with_reuse(current_latent_state_index: int, discount_factor: float, value_prefixs, values, policies,
                                   min_max_stats_lst: MinMaxStatsList, results: ResultsWrapper, to_play_batch,
                                   no_inference_lst, reuse_lst, reuse_value_lst, _is_reset_list=None):
    """mz_tree.pyx batch_backpropagate_with_reuse (cnode.cpp:502-549).  ``value_prefixs`` / ``values`` / ``policies`` are the
    COMPACTED network outputs of the trees that were inferred (the driver skips the others, mcts_ctree.py:424-432);
    they are scattered back to per-tree rows here, using ``no_inference_lst`` exactly as the C++ loop consumes it."""
    roots = results._roots
    t = roots._tree
    B, A = roots.root_num, t.A
    dev = roots.device
    skip = np.zeros(B, bool)
    skip[[i for i in no_inference_lst if i >= 0]] = True
    rank = np.cumsum(~skip) - 1                     # compact row of every inferred tree
    rank[skip] = -1
    n = int((~skip).sum())
    idx = torch.from_numpy(np.nonzero(~skip)[0]).to(dev)

    def scatter(x, shape):
        full = torch.zeros((B,) + shape, device=dev, dtype=torch.float32)
        if n:
            full[idx] = _to_dev(x, torch.float32, dev, (n,) + shape)
        return full
    rew, val, pol = scatter(value_prefixs, ()), scatter(values, ()), scatter(policies, (A,))
    rv = _to_dev(reuse_value_lst, torch.float32, dev, (B,))
    rk = torch.from_numpy(rank.astype(np.int32)).to(dev)
    tp = _to_dev(to_play_batch, torch.int32, dev, (B,))
    rs = _to_dev(_is_reset_list, torch.int32, dev, (B,))
    with torch.cuda.device(dev):
        cabi.check(t.lib.lz_tree_backpropagate(t.h, int(current_latent_state_index), rew.data_ptr(), val.data_ptr(),
                                               pol.data_ptr(), rv.data_ptr(), rk.data_ptr(), cabi.ptr(rs), cabi.ptr(tp),
                                               cabi.stream_ptr()), "lz_tree_backpropagate")
    t._keep = (rew, val, pol, rv, rk, rs, tp)
