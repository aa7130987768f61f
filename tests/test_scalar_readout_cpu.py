"""CPU checks of the scalar read-out's support and of the fp32 inverse transform the GPU band test relies on.

- The support the kernels use for a range (size K = ceil(fl32(fl32(stop - start) / step)) in check_create, value k =
  fmaf(step, k, start) in support_at) against the reference's ``torch.arange(start, stop, step, dtype=float32)``, over a grid
  of ranges that includes the non-dyadic steps where the two disagree.  Every range where they disagree must be refused when
  a model or a stand-alone transform is constructed; every range where they agree, every shipped support among them, must be
  accepted.  tests/test_gpu_scalar_readout.py checks the same emulation against the device's support_at and lz_model_create.
- F32, the reference's fp32 formula for h^-1 (scaling_transform.py:88-90) with every operation rounded once, is monotone on
  each sign over the floats with 0 < |x| <= 301, and odd: that is what makes the extremes of F32 over [x - B, x + B] a
  valid band for a scalar whose expectation is known to within B.  It is not monotone across 0: F32(+-0) = 0, while the
  cancellation in sqrt(1 + 4 eps (|x| + 1 + eps)) - 1 gives F32(x) = -2.587e-5 for every 0 < x < 1e-4 or so (and
  +2.587e-5 for the negatives), so the GPU band takes 0 and F32 of the smallest float of each sign in the interval into
  account.  Strided sweep (stride 61); LZ_EXHAUSTIVE=1 sweeps every float.
"""
import itertools
import os
from fractions import Fraction

import numpy as np
import pytest
import torch

from lightzero_b200.scaling_transform import check_support, library_support

STARTS = (-300., -50., -30., -20., -10., -5., -1.1, -1., -0.7, 0., 0.1)
STOPS = (0.3, 0.5, 1., 1.1, 5., 10.5, 11., 20.5, 30., 51., 301.)
STEPS = (0.02, 0.05, 0.1, 0.2, 0.25, 0.3, 0.5, 0.7, 1., 1.5, 2., 3.)
# the ranges the library accepts (2 <= K <= 608), where the size or the values can disagree with torch.arange
GRID = [r for r in itertools.product(STARTS, STOPS, STEPS)
        if r[0] < r[1] and 2 <= len(torch.arange(*r, dtype=torch.float32)) <= 608]
SHIPPED = [(-300., 301., 1.), (-50., 51., 1.), (-10., 11., 1.), (-1., 1., 1.), (-20., 20.5, 0.5), (-303., 305., 1.),
           (-5., 5., 0.25), (-400., 401., 1.)]


def kernel_support(start, stop, step):
    """The kernels' support, derived here without the package: float32 arithmetic for K, and fmaf(step, k, start) as the
    float32 rounding of the float64 sum step * k + start, which this function checks is exact (so it is rounded once)."""
    lo, hi, st = np.float32(start), np.float32(stop), np.float32(step)
    K = int(np.ceil(np.float32(hi - lo) / st))
    vals = []
    for k in range(K):
        s = np.float64(st) * k + np.float64(lo)
        assert Fraction(float(s)) == Fraction(float(st)) * k + Fraction(float(lo)), (start, stop, step, k)
        vals.append(np.float32(s))
    return K, np.array(vals, np.float32)


def agrees(r):
    K, vals = kernel_support(*r)
    ref = torch.arange(*r, dtype=torch.float32).numpy()
    return K == ref.size and np.array_equal(vals.view(np.uint32), ref.view(np.uint32))


def test_package_emulation_matches_the_kernel_arithmetic():
    for r in GRID + SHIPPED:
        K, vals = library_support(*r)
        K2, vals2 = kernel_support(*r)
        assert K == K2 and np.array_equal(vals.view(np.uint32), vals2.view(np.uint32)), r


def test_the_grid_holds_the_ranges_that_disagree():
    bad = [r for r in GRID if not agrees(r)]
    size = [r for r in bad if kernel_support(*r)[0] != len(torch.arange(*r, dtype=torch.float32))]
    print(f"\n[support] {len(GRID)} accepted ranges, {len(bad)} disagree with torch.arange ({len(size)} in size)")
    assert (0.1, 0.3, 0.1) in size and (-1., 1.1, 0.3) in size
    assert kernel_support(0.1, 0.3, 0.1)[0] == 3 and len(torch.arange(0.1, 0.3, 0.1)) == 2
    assert kernel_support(-1., 1.1, 0.3)[0] == 7 and len(torch.arange(-1., 1.1, 0.3)) == 8
    assert len(size) >= 20 and len(bad) > len(size)
    for r in SHIPPED:
        assert agrees(r), r


def test_support_is_refused_unless_it_equals_arange():
    wrong = []
    for r in GRID + SHIPPED:
        try:
            check_support(r)
            refused = False
        except ValueError as e:
            assert "torch.arange" in str(e), e
            refused = True
        if refused == agrees(r):
            wrong.append((r, "refused" if refused else "accepted"))
    assert not wrong, wrong[:20]


def test_refused_at_construction_before_any_device_work():
    """The models and the stand-alone transform refuse the range in their constructors, before they look for a device."""
    import lightzero_b200 as lzb
    for r in ((0.1, 0.3, 0.1), (-1., 1.1, 0.3), (-1., 1., 0.1), (-30., 30., 0.3)):
        with pytest.raises(ValueError, match="support range"):
            lzb.InverseScalarTransform(lzb.DiscreteSupport(*r, device="cpu"))
        for cls in (lzb.MuZeroModel, lzb.MuZeroModelMLP, lzb.EfficientZeroModelMLP, lzb.EfficientZeroModel):
            with pytest.raises(ValueError, match="support range"):
                cls(reward_support_range=r, value_support_range=r)


def f32_formula(x):
    """F32: scaling_transform.py:88-90 applied to the expectation x, each operation rounded once in IEEE fp32 (numpy), in the
    reference's order: sign(x) * (t * t - 1), t = (sqrt(1 + (4 eps) (|x| + 1 + eps)) - 1) / (2 eps).  torch on the CPU
    evaluates the same expression but its vectorised sqrt is not always correctly rounded, so it differs by one quantum on
    about 0.07 % of the floats (printed by tests/test_gpu_scalar_readout.py)."""
    x = np.asarray(x, np.float32)
    eps = np.float32(0.001)
    t = (np.abs(x) + np.float32(1)) + eps
    t = np.float32(1) + (np.float32(4) * eps) * t
    t = (np.sqrt(t) - np.float32(1)) / (np.float32(2) * eps)
    sign = np.where(x > 0, np.float32(1), np.where(x < 0, np.float32(-1), np.float32(0))).astype(np.float32)
    return sign * (t * t - np.float32(1))


def test_f32_inverse_transform_is_monotone():
    stride = 1 if os.environ.get("LZ_EXHAUSTIVE") else 61
    top = int(np.float32(301.0).view(np.uint32))
    prev = None
    for lo in range(1, top + 1, stride << 24):
        bits = torch.arange(lo, min(lo + (stride << 24), top + 1), stride, dtype=torch.int64).to(torch.int32)
        x = bits.numpy().view(np.float32)
        y = f32_formula(x)
        assert np.isfinite(y).all()
        assert (y[1:] >= y[:-1]).all(), "F32 decreases between two positive floats"
        assert prev is None or prev <= y[0]
        prev = y[-1]
        assert np.array_equal(f32_formula(-x), -y), "F32 is not odd"
    tiny = np.array([1e-45, -1e-45, 0.0, -0.0], np.float32)
    assert f32_formula(tiny).tolist() == [F32_TINY, -F32_TINY, 0.0, 0.0]


F32_TINY = -2.586841583251953e-05       # F32 of the smallest positive floats
