"""Mirror of lzero/policy/scaling_transform.py:6-13,64-92 (DiscreteSupport, InverseScalarTransform)
for callers that keep their own PyTorch model but want the fused CUDA transform, and the check every model and transform
runs on its support range at construction."""
import math
from fractions import Fraction

import numpy as np
import torch

from . import cabi


def _round_f32(x: Fraction) -> np.float32:
    """x rounded to the nearest float32, ties to even (no double rounding through float64)"""
    f = np.float32(float(x))
    cands = (np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf)))
    return min(cands, key=lambda c: (abs(Fraction(float(c)) - x), int(c.view(np.uint32)) & 1))


def library_support(start: float, stop: float, step: float):
    """The support the kernels use for the range (start, stop, step): the bounds and step are rounded to float32, the size is
    K = ceil(fl32(fl32(stop - start) / step)) (check_create, model.cu) and value k is fmaf(step, k, start) in float32
    (support_at, net6.cuh).  Returns (K, float32 values)."""
    lo, hi, st = np.float32(start), np.float32(stop), np.float32(step)
    K = math.ceil(float(np.float32(hi - lo) / st))
    vals = [_round_f32(Fraction(float(st)) * k + Fraction(float(lo))) for k in range(max(K, 0))]
    return K, np.array(vals, np.float32)


def check_support(support_range) -> None:
    """Refuses a support range whose size or values on the device differ from the reference's
    ``torch.arange(start, stop, step, dtype=torch.float32)`` (scaling_transform.py:6-13).  Integer and dyadic steps such as
    1 and 0.25 pass; steps such as 0.1 or 0.3 round differently in float32 and are refused (ValueError)."""
    start, stop, step = (float(v) for v in support_range)
    ref = torch.arange(start, stop, step, dtype=torch.float32).numpy()
    K, vals = library_support(start, stop, step)
    if K != ref.size:
        raise ValueError(f"support range ({start}, {stop}, {step}): the kernels would use {K} support values, "
                         f"torch.arange gives {ref.size}")
    bad = np.flatnonzero(vals.view(np.uint32) != ref.view(np.uint32))
    if bad.size:
        k = int(bad[0])
        raise ValueError(f"support range ({start}, {stop}, {step}): {bad.size} of {K} support values differ from torch.arange "
                         f"in float32 (value {k}: {float(vals[k])!r} vs {float(ref[k])!r}); use an integer or dyadic step")


class DiscreteSupport(object):
    """scaling_transform.py:6-13"""

    def __init__(self, start: float, stop: float, step: float = 1., device="cuda") -> None:
        assert start < stop
        self.start, self.stop, self.step = float(start), float(stop), float(step)
        self.arange = torch.arange(start, stop, step, dtype=torch.float32).unsqueeze(0).to(device)
        self.size = self.arange.shape[1]
        assert self.size > 0, "DiscreteSupport size must be greater than 0"


class InverseScalarTransform:
    """scaling_transform.py:64-92: softmax(logits) . support -> h^-1, one fused CUDA kernel."""

    def __init__(self, scalar_support: DiscreteSupport, categorical_distribution: bool = True) -> None:
        if not categorical_distribution:
            raise NotImplementedError("only the categorical (support) representation is implemented")
        check_support((scalar_support.start, scalar_support.stop, scalar_support.step))
        self.value_support = scalar_support.arange
        self.support = scalar_support
        self._lib = cabi.load()
        cfg = cabi.ModelConfig(4, 84, 84, 1, 1, 64, 16, 16, 16, 32, 32, 32, scalar_support.start,
                               scalar_support.stop, scalar_support.step, downsample=1)
        h = cabi.c_void_p()
        cabi.check(self._lib.lz_model_create(cfg, h), "lz_model_create")
        self._h = h

    def __call__(self, logits: torch.Tensor, epsilon: float = 0.001) -> torch.Tensor:
        assert abs(epsilon - 0.001) < 1e-12, "the kernel fixes epsilon = 0.001 (the reference default)"
        logits = logits.to(torch.float32).contiguous()
        assert logits.is_cuda and logits.shape[1] == self.support.size
        out = torch.empty(logits.shape[0], 1, device=logits.device)
        with torch.cuda.device(logits.device):
            cabi.check(self._lib.lz_inverse_scalar_transform(self._h, logits.shape[0], logits.data_ptr(),
                                                             out.data_ptr(), cabi.stream_ptr()),
                       "lz_inverse_scalar_transform")
        return out

    def __del__(self):
        try:
            self._lib.lz_model_destroy(self._h)
        except Exception:
            pass
