"""Device-resident collector state (SURVEY 8(f) row f-3): the parts of ``MuZeroCollector.collect`` (lzero/worker/muzero_collector.py:
508-760) that sit between the environments and the search, kept on the GPU so that a collect step moves ONE new uint8 frame per
environment over PCIe and nothing comes back except the chosen actions.

* ``FrameStack``     -- ``GameSegment.get_obs()`` / ``append()`` / the ``frame_stack_num`` seeding (game_segment.py:140-181,
                        muzero_collector.py:451-457): [B, stack, H, W] uint8 on the device, oldest frame first;
* ``SegmentStats``   -- ``GameSegment.store_search_stats`` / ``reset`` (game_segment.py:241-263, 340-362): child-visit distributions
                        and root values (and Gumbel MuZero's improved policies) appended per step for B segments of capacity T,
                        from any search family's collect, Stochastic MuZero's wider tree rows included;
* ``gather_segments``-- the all-gather of finished segments across ranks (one NCCL ``all_gather_into_tensor`` of a packed buffer).

All compute is in ``csrc/collector.cu`` behind the C ABI (include/lzb200.h); there is no CPU fallback.
"""
import ctypes

import numpy as np
import torch

from . import cabi


class _DevArray:
    """A library-owned device buffer exposed through ``__cuda_array_interface__`` so that torch can view it without a copy."""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"data": (int(ptr), False), "shape": tuple(shape), "typestr": typestr, "version": 2, "strides": None}


def _view(ptr, shape, typestr, device):
    return torch.as_tensor(_DevArray(ptr, shape, typestr), device=device)


class FrameStack:
    def __init__(self, env_num: int, frame_stack_num: int, height: int, width: int, device=None):
        self._lib = cabi.load()
        self.B, self.stack, self.H, self.W = int(env_num), int(frame_stack_num), int(height), int(width)
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            cabi.check(self._lib.lz_frames_create(self.B, self.stack, self.H, self.W, ctypes.byref(h)), "lz_frames_create")
        self._h = h
        self._keep = None

    def push(self, new_frames, reset=None) -> None:
        """One new frame per environment: uint8 [B, H, W] (numpy / CPU tensor: copied from pinned memory; CUDA tensor: used in
        place).  ``reset``: bool / uint8 [B] or None -- environments whose episode just (re)started: their whole stack becomes the
        new frame, as ``GameSegment.reset([init_obs] * frame_stack_num)`` does (muzero_collector.py:451-457)."""
        with torch.cuda.device(self.device):
            if isinstance(new_frames, torch.Tensor) and new_frames.is_cuda:
                nf = new_frames.to(torch.uint8).contiguous()
                assert tuple(nf.shape) == (self.B, self.H, self.W), nf.shape
                rs = None if reset is None else torch.as_tensor(reset).to(self.device, torch.uint8).contiguous()
                cabi.check(self._lib.lz_frames_push(self._h, nf.data_ptr(), cabi.ptr(rs), cabi.stream_ptr()), "lz_frames_push")
            else:
                def pinned(x):        # pinned host tensors are used in place; anything else is staged through pinned memory
                    if isinstance(x, torch.Tensor) and x.dtype == torch.uint8 and x.is_contiguous() and x.is_pinned():
                        return x
                    return torch.as_tensor(np.ascontiguousarray(np.asarray(x), dtype=np.uint8)).pin_memory()
                nf = pinned(new_frames)
                assert tuple(nf.shape) == (self.B, self.H, self.W), nf.shape
                rs = None if reset is None else pinned(reset)
                assert rs is None or rs.numel() == self.B
                cabi.check(self._lib.lz_frames_push_host(self._h, nf.data_ptr(), cabi.ptr(rs), cabi.stream_ptr()), "lz_frames_push_host")
            self._keep = (nf, rs)

    def stacked_ptr(self) -> int:
        """Device pointer of the [B, stack, H, W] uint8 batch for ``lz_search_collect_u8``; valid until the next push."""
        return int(self._lib.lz_frames_stacked(self._h))

    def view(self) -> torch.Tensor:
        """Zero-copy uint8 [B, stack, H, W] tensor over the current stacks (valid until the next push): the observation batch for
        ``MuZeroCollectPolicy.search_batch`` / ``lz_search_collect_u8``."""
        return _view(self.stacked_ptr(), (self.B, self.stack, self.H, self.W), "|u1", self.device)

    def get_obs(self) -> torch.Tensor:
        """A copy of the stacked observations (uint8 [B, stack, H, W], oldest first) -- for tests and for callers that want a tensor."""
        with torch.cuda.device(self.device):
            return _view(self.stacked_ptr(), (self.B, self.stack, self.H, self.W), "|u1", self.device).clone()

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self._lib.lz_frames_destroy(self._h)
        except Exception:
            pass


class SegmentStats:
    def __init__(self, env_num: int, game_segment_length: int, action_space_size: int, device=None):
        self._lib = cabi.load()
        self.B, self.T, self.A = int(env_num), int(game_segment_length), int(action_space_size)
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            cabi.check(self._lib.lz_segments_create(self.B, self.T, self.A, ctypes.byref(h)), "lz_segments_create")
        self._h = h

    def store_search_stats(self, visit_counts: torch.Tensor, root_values: torch.Tensor, active=None, improved_policy=None) -> None:
        """game_segment.py:241-263 for every (active) environment: ``visit_counts`` int32 [B, A] (-1 beyond the legal list, as
        ``lz_tree_results`` / ``Roots`` deliver them on the device), ``root_values`` f32 [B], and for Gumbel MuZero
        ``improved_policy`` f32 [B, A] by action id (``GumbelMuZeroCollectPolicy.search_batch``'s ``improved_policy``).  The
        visits of a Stochastic MuZero tree are [B, max(A, chance_space_size)] wide: the first A columns, which hold every legal
        root child, are stored."""
        v = visit_counts.to(self.device, torch.int32)
        if v.shape[1] > self.A:
            v = v[:, :self.A]
        v = v.contiguous()
        r = root_values.to(self.device, torch.float32).contiguous()
        a = None if active is None else torch.as_tensor(active).to(self.device, torch.uint8).contiguous()
        with torch.cuda.device(self.device):
            if improved_policy is not None:      # stored at the position store_search_stats is about to fill
                ip = improved_policy.to(self.device, torch.float32).contiguous()
                cabi.check(self._lib.lz_segments_store_improved_policy(self._h, ip.data_ptr(), cabi.ptr(a), cabi.stream_ptr()),
                           "lz_segments_store_improved_policy")
            cabi.check(self._lib.lz_segments_store_search_stats(self._h, v.data_ptr(), r.data_ptr(), cabi.ptr(a), cabi.stream_ptr()),
                       "lz_segments_store_search_stats")

    def reset(self, done=None) -> None:
        d = None if done is None else torch.as_tensor(done).to(self.device, torch.uint8).contiguous()
        with torch.cuda.device(self.device):
            cabi.check(self._lib.lz_segments_reset(self._h, cabi.ptr(d), cabi.stream_ptr()), "lz_segments_reset")

    def tensors(self):
        """Copies of (child_visits f32 [B, T, A], root_values f32 [B, T], len int32 [B])."""
        p = [ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()]
        cabi.check(self._lib.lz_segments_data(self._h, ctypes.byref(p[0]), ctypes.byref(p[1]), ctypes.byref(p[2])), "lz_segments_data")
        shapes = [((self.B, self.T, self.A), "<f4"), ((self.B, self.T), "<f4"), ((self.B,), "<i4")]
        with torch.cuda.device(self.device):
            outs = [_view(ptr.value, shape, ts, self.device).clone() for ptr, (shape, ts) in zip(p, shapes)]
        return tuple(outs)

    def improved_policy(self):
        """A copy of the improved policies f32 [B, T, A] stored so far (0 where none was), or None before the first one."""
        p = ctypes.c_void_p()
        cabi.check(self._lib.lz_segments_improved_policy(self._h, ctypes.byref(p)), "lz_segments_improved_policy")
        if not p.value:
            return None
        with torch.cuda.device(self.device):
            return _view(p.value, (self.B, self.T, self.A), "<f4", self.device).clone()

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self._lib.lz_segments_destroy(self._h)
        except Exception:
            pass


def pack_segments(child_visits: torch.Tensor, root_values: torch.Tensor, lengths: torch.Tensor) -> torch.Tensor:
    """One contiguous f32 buffer per rank for the collective: [B, T * A + T + 1] = child visits | root values | length."""
    B = child_visits.shape[0]
    return torch.cat([child_visits.reshape(B, -1), root_values.reshape(B, -1), lengths.reshape(B, 1).to(torch.float32)], dim=1).contiguous()


def unpack_segments(packed: torch.Tensor, T: int, A: int):
    n = packed.shape[0]
    return (packed[:, :T * A].reshape(n, T, A), packed[:, T * A:T * A + T].reshape(n, T), packed[:, T * A + T].to(torch.int32))


def gather_segments(child_visits: torch.Tensor, root_values: torch.Tensor, lengths: torch.Tensor):
    """All-gathers the finished segments of every rank's environments (rank-major order) with ONE collective on one packed
    buffer (NCCL over NVLink on GPUs, gloo in the CPU tests).  Every rank holds the same number of environments."""
    import torch.distributed as dist
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return child_visits, root_values, lengths
    B, T, A = child_visits.shape
    mine = pack_segments(child_visits, root_values, lengths)
    out = torch.empty(dist.get_world_size() * B, mine.shape[1], dtype=torch.float32, device=mine.device)
    dist.all_gather_into_tensor(out, mine)
    return unpack_segments(out, T, A)
