"""The value and reward read-out (softmax of the categorical logits, dotted with the support, then h^-1) over the whole value
range, against float64.

1. The primitives on the device.  tests/csrc/scalar_math_dev.cu applies net6.cuh's inverse_scalar_transform and
   lz_exact_math.h's lz_expf_exact / lz_logf_exact to device arrays; it is built twice, with -fmad=false and with
   contraction on, as the library compiles these headers both ways, and both builds must give the same bits.  h^-1 is
   compared bit for bit with F32, the reference's fp32 formula (scaling_transform.py:88-90) with every operation rounded once
   (test_scalar_readout_cpu.f32_formula), for the floats with |x| <= 301; expf (every float in [-104, 0], -inf and inputs below -104) and logf (every positive
   normal float) with libm run by the harness's host side.  Strided by 61 by default; LZ_EXHAUSTIVE=1 sweeps every input
   (measured on an H100 80GB HBM3 at 700 W: h^-1 100 s, expf 13 s, logf 25 s, the host side dominating; 0 mismatches).  The counts of floats where torch differs from F32 are printed,
   not asserted: on the CPU its vectorised sqrt is not always correctly rounded (about 0.07 % of the floats, one quantum
   each), and on CUDA it divides by a scalar as a multiplication by its reciprocal.
   The device's support_at and the size lz_model_create computes are checked against the package's emulation
   (scaling_transform.library_support), which decides what the constructors refuse.
2. The read-out against float64.  From the kernel's own fp32 logits, x64 = sum softmax64(l)_k s_k with s_k the float32
   torch.arange values, and B_x = sum_k p_k rho_k (|s_k| + |x64|) + u |x64| bounds the fp32 evaluation: rho_k =
   d_k 2^-22 (the exponent arguments of term k, which telescope to d_k = max l - l_k, rounded in the subtraction and in the
   scaling by log2 e) + R (2^-22 + 2u) (R exponentials and products on its path, ex2.approx within 2^-22) + D u (its fp32
   additions), u = 2^-24, R = ceil(K/128) + 1, D = ceil(K/128) + 10.  Since h^-1 on the device is F32 (part 1) and F32 is
   monotone on each sign (test_scalar_readout_cpu.py), the scalar must lie within the extremes of F32 over
   [x64 - B_x, x64 + B_x].  The band is relative, so it means something at |v| ~ 1e4 where an absolute 2e-4 does not.
   Logit profiles: one-hot (the scalar is F32(s_k) bit for bit), a peak anywhere, bimodal at the support edges, near-uniform,
   a spread of 200, and the maximum in the last partial 128-block.  The models get them through the bias of the last Linear
   of the value and reward heads (weights scaled by a small alpha so that roots differ).  Canonical-order families (the
   conv heads, board, mlp.cu, k_ez_head) must also return the same bits as lz_inverse_scalar_transform of their own logits.
   mlp_tc.cu's quad combine gets its own R and D, with ceil(K/4) (the logits one quad lane folds) for ceil(K/128).  Every
   family runs at every support above, the conv MuZero model on 6x6 and 8x8 latents.
   Each sensitivity variant (fp16 logits, a dropped 32-piece, no exp(m - M) rescale, the support shifted by one step) must
   leave the band on some root.
3. The searches with node values in the thousands and more, bit for bit against the oracle driving the same network: the
   MuZero conv search (persistent and multi-kernel), the EfficientZero search at horizon 5, both MuZeroModelMLP kernels,
   EfficientZeroModelMLP, and the Gumbel search against the compiled reference tree.
"""
import ctypes
import itertools
import math
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu

EXHAUSTIVE = bool(os.environ.get("LZ_EXHAUSTIVE"))
STRIDE = 1 if EXHAUSTIVE else 61
CHUNK = 1 << 25
SUPPORTS = [(-300., 301., 1.), (-50., 51., 1.), (-10., 11., 1.), (-1., 1., 1.), (-5., 5., 0.25)]
U = 2.0 ** -24
F32_TINY = -2.586841583251953e-05       # F32 of the smallest positive floats (test_scalar_readout_cpu.py)


# ------------------------------------------------------------------------------------------------ the harness
@pytest.fixture(scope="module")
def harness():
    """{"fma": lib, "nofma": lib}: scalar_math_dev.cu built with and without -fmad=false"""
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not on PATH")
    from lightzero_b200 import _build
    tmp = tempfile.mkdtemp(prefix="lz_scalar_math_")
    libs = {}
    for tag, extra in (("fma", []), ("nofma", ["-fmad=false"])):
        so = os.path.join(tmp, f"scalar_math_{tag}.so")
        cmd = (["nvcc"] + _build.ARCH + _build.COMMON + extra + ["-I", _build.CSRC, "-shared", "-o", so,
               os.path.join(ROOT, "tests", "csrc", "scalar_math_dev.cu"), "-lm"])
        p = subprocess.run(cmd, capture_output=True, text=True)
        assert p.returncode == 0, p.stderr[-4000:]
        lib = ctypes.CDLL(so)
        lib.sm_apply.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]
        lib.sm_support.argtypes = [ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        lib.sm_host_libm.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong]
        libs[tag] = lib
    yield libs
    shutil.rmtree(tmp, ignore_errors=True)


def device_apply(lib, fn, x):
    out = torch.empty_like(x)
    assert lib.sm_apply(fn, x.data_ptr(), out.data_ptr(), x.numel(), torch.cuda.current_stream().cuda_stream) == 0
    return out


def host_libm(lib, fn, x):
    x = x.cpu().contiguous()
    out = torch.empty_like(x)
    assert lib.sm_host_libm(fn, x.data_ptr(), out.data_ptr(), x.numel()) == 0
    return out


def float_bits(lo, hi, stride=STRIDE):
    """the floats whose bit patterns are lo, lo + stride, ... < hi (unsigned), on the device, in chunks"""
    for a in range(lo, hi, CHUNK * stride):
        b = torch.arange(a, min(a + CHUNK * stride, hi), stride, dtype=torch.int64, device="cuda")
        yield b.to(torch.int32).view(torch.float32)


def f32_cpu(x):
    """F32, the reference's fp32 formula with every operation rounded once (test_scalar_readout_cpu.f32_formula)"""
    from test_scalar_readout_cpu import f32_formula
    return torch.from_numpy(f32_formula(x.detach().cpu().numpy()))


def f32_torch(x):
    """the same formula in torch, oracle/model_ref.py's class applied to x, on x's device"""
    from oracle.model_ref import DiscreteSupport, InverseScalarTransform
    return InverseScalarTransform(DiscreteSupport(-1., 1., 1., device=x.device), categorical_distribution=False)(x)


def bits(t):
    return t.contiguous().view(torch.int32)


def _sweep(harness, fn, ranges, ref_fn, specials=()):
    import time
    t0, n, bad, gpu_diff = time.time(), 0, 0, 0
    chunks = itertools.chain((c for lo, hi in ranges for c in float_bits(lo, hi)),
                             [torch.tensor(specials, dtype=torch.float32, device="cuda")] if specials else [])
    for x in chunks:
        a = device_apply(harness["fma"], fn, x)
        b = device_apply(harness["nofma"], fn, x)
        assert torch.equal(bits(a), bits(b)), "the -fmad=false and contracting builds differ"
        ref, extra = ref_fn(x)
        bad += int((bits(a.cpu()) != bits(ref)).sum())
        gpu_diff += extra
        n += x.numel()
    return n, bad, gpu_diff, time.time() - t0


def test_inverse_transform_is_the_reference_fp32_formula(harness):
    top = int(np.float32(301.0).view(np.uint32)) + 1

    torch_diff = [0, 0]

    def ref(x):
        r = f32_cpu(x)
        torch_diff[0] += int((bits(f32_torch(x.cpu())) != bits(r)).sum())
        torch_diff[1] += int((bits(f32_torch(x).cpu()) != bits(r)).sum())
        return r, 0
    n, bad, _, sec = _sweep(harness, 0, [(0, top), (1 << 31, (1 << 31) + top)], ref, (0.0, -0.0, 301.0, -301.0, 1e-45))
    print(f"\n[scalar-math] h^-1: {n} floats (stride {STRIDE}), {bad} mismatches with F32; torch on the CPU differs from F32 on "
          f"{torch_diff[0]}, torch on CUDA on {torch_diff[1]}; {sec:.1f} s")
    assert bad == 0


def test_expf_exact_matches_libm_on_the_device(harness):
    lo = 1 << 31
    hi = int(np.float32(-104.0).view(np.uint32)) + 1
    n, bad, _, sec = _sweep(harness, 1, [(lo, hi)], lambda x: (host_libm(harness["fma"], 1, x), 0),
                            (0.0, float("-inf"), -104.5, -200.0, -1e30, -3.4028235e38, float.fromhex("-0x1.f8cbb2p+5")))
    print(f"\n[scalar-math] lz_expf_exact: {n} floats in [-104, 0] (stride {STRIDE}), {bad} mismatches with libm; {sec:.1f} s")
    assert bad == 0


def test_logf_exact_matches_libm_on_the_device(harness):
    n, bad, _, sec = _sweep(harness, 2, [(0x00800000, 0x7f800000)], lambda x: (host_libm(harness["fma"], 2, x), 0),
                            (1.0, 1.1754944e-38, 3.4028235e38, 2.0, 601.0))
    print(f"\n[scalar-math] lz_logf_exact: {n} positive normal floats (stride {STRIDE}), {bad} mismatches with libm; {sec:.1f} s")
    assert bad == 0


def test_support_values_and_sizes_are_the_emulated_ones(harness):
    """The device's support_at and lz_model_create's K against scaling_transform.library_support, over the CPU file's grid;
    the models are created through the C ABI directly (the Python constructors refuse most of these ranges) and nothing
    is launched on them."""
    import test_scalar_readout_cpu as C
    from lightzero_b200 import cabi
    from lightzero_b200.scaling_transform import library_support
    lib = cabi.load()
    refused = 0
    for r in C.GRID + C.SHIPPED:
        K, vals = library_support(*r)
        out = torch.empty(K, device="cuda")
        assert harness["fma"].sm_support(np.float32(r[0]), np.float32(r[2]), K, out.data_ptr(),
                                         torch.cuda.current_stream().cuda_stream) == 0
        assert np.array_equal(out.cpu().numpy().view(np.uint32), vals.view(np.uint32)), r
        if K > 608:
            continue                              # beyond every head's support limit: lz_model_create refuses it
        cfg = cabi.ModelConfig(4, 84, 84, 1, 1, 64, 16, 16, 16, 32, 32, 32, r[0], r[1], r[2], downsample=1)
        h = cabi.c_void_p()
        cabi.check(lib.lz_model_create(cfg, h), "lz_model_create")
        assert lib.lz_model_support_size(h) == K, r
        lib.lz_model_destroy(h)
        refused += not C.agrees(r)
    print(f"\n[support] {len(C.GRID) + len(C.SHIPPED)} ranges: device support and size as emulated; {refused} refused by the constructors")


# ------------------------------------------------------------------------------------------------ float64 reference and band
def sup32(support):
    return torch.arange(*support, dtype=torch.float32)


def x64_and_bound(logits, support, order="canonical"):
    """(x64, B_x) per row from the fp32 logits (module docstring).  n, the logits one lane folds in sequence, sets R and D:
    ceil(K/128) in the canonical order (128 virtual threads); ceil(K/4) in mlp_tc.cu's quad combine, where each of a row's 4
    quad lanes folds every 4th pair of columns before one rescale and two shuffle additions."""
    L = logits.double().cpu()
    s = sup32(support).double()
    K = s.numel()
    p = torch.softmax(L, 1)
    x = (p * s).sum(1)
    d = L.max(1, keepdim=True).values - L
    d = torch.where(torch.isfinite(d), d, torch.zeros_like(d))
    nb = -(-K // (4 if order == "quad" else 128))
    rho = d * 2.0 ** -22 + (nb + 1) * (2.0 ** -22 + 2 * U) + (nb + 10) * U
    B = (p * rho * (s.abs() + x.abs().unsqueeze(1))).sum(1) + U * x.abs()
    return x, B


def _round_f32(x, up):
    f = x.float()
    fix = (f.double() < x) if up else (f.double() > x)
    return torch.where(fix, torch.nextafter(f, torch.full_like(f, math.inf if up else -math.inf)), f)


def band(x, B):
    """extremes of F32 over the floats in [x - B, x + B]: F32 is monotone on each sign, 0 at +-0"""
    lo, hi = _round_f32(x - B, False), _round_f32(x + B, True)
    cands = [f32_cpu(lo), f32_cpu(hi)]
    z = torch.zeros_like(lo)
    cands.append(torch.where((lo <= 0) & (hi >= 0), z, cands[0]))
    cands.append(torch.where((lo <= 0) & (hi > 0), z + F32_TINY, cands[0]))
    cands.append(torch.where((lo < 0) & (hi >= 0), z - F32_TINY, cands[0]))
    c = torch.stack(cands)
    return c.min(0).values, c.max(0).values


def check_band(v, logits, support, what, order="canonical"):
    """v inside the band; returns the worst |v - F32(x64)| / band half-width on the violating side"""
    x, B = x64_and_bound(logits, support, order)
    lo, hi = band(x, B)
    v = v.float().cpu().reshape(-1)
    out = (v < lo) | (v > hi)
    assert not out.any(), (what, int(out.sum()), v[out][:4].tolist(), lo[out][:4].tolist(), hi[out][:4].tolist())
    c = f32_cpu(x.float())
    half = torch.where(v >= c, hi - c, c - lo).double()
    r = torch.where(half > 0, (v - c).abs().double() / half, torch.zeros_like(half))
    return r.max().item()


def outside_band(v_var, logits, support, order="canonical"):
    x, B = x64_and_bound(logits, support, order)
    lo, hi = band(x, B)
    return (v_var < lo) | (v_var > hi)


# ------------------------------------------------------------------------------------------------ logit profiles
PROFILES = ("onehot", "peak", "bimodal", "uniform", "spread", "lastblock")


def profile_logits(name, K, B, g):
    """(B, K) float32 logits of a profile; rows differ"""
    k = torch.arange(K, dtype=torch.float64)
    L = torch.full((B, K), -1000.0, dtype=torch.float64)
    for b in range(B):
        if name == "onehot":
            L[b, [0, 1, K // 2, K - 2, K - 1, int(torch.randint(0, K, (1,), generator=g))][b % 6]] = 0.0
        elif name == "peak":
            c = [0, K - 1][b % 2] if b < 2 else float(torch.rand(1, generator=g)) * (K - 1)
            w = 0.5 + float(torch.rand(1, generator=g)) * K / 8
            L[b] = -((k - c) / w) ** 2 + 0.1 * torch.randn(K, generator=g, dtype=torch.float64)
        elif name == "bimodal":
            L[b, 0], L[b, K - 1] = 0.0, (float(torch.rand(1, generator=g)) - 0.5) * 2e-3
        elif name == "uniform":
            L[b] = 0.02 * torch.randn(K, generator=g, dtype=torch.float64)
        elif name == "spread":
            L[b] = -200.0 * torch.rand(K, generator=g, dtype=torch.float64)
            L[b, int(torch.randint(0, K, (1,), generator=g))] = 0.0
        elif name == "lastblock":
            L[b] = 2.0 * torch.randn(K, generator=g, dtype=torch.float64)
            first = 128 * ((K - 1) // 128) if K > 128 else 32 * ((K - 1) // 32)
            L[b, int(torch.randint(first, K, (1,), generator=g))] += 9.0
    return L.float()


def variants(logits, support):
    """scalars of the sensitivity variants, computed from the same logits: {name: (B,) float32}"""
    L = logits.double().cpu()
    s = sup32(support).double()
    K = s.numel()

    def h(x):
        return f32_cpu(x.float())
    out = {"fp16 logits": h((torch.softmax(L.float().half().double(), 1) * s).sum(1)),
           "support + step": h((torch.softmax(L, 1) * (s + support[2])).sum(1))}
    keep = torch.ones(K, dtype=torch.bool)
    keep[32 * ((K - 1) // 32):] = False                    # the last 32-piece
    if not keep.any():
        keep[:] = True
        keep[0] = False
    out["dropped piece"] = h((torch.softmax(L[:, keep], 1) * s[keep]).sum(1))
    # no exp(m - M): each virtual thread (k mod 128) keeps its sums relative to its own maximum
    vt = torch.arange(K) % 128
    Sx, Wx = torch.zeros(L.shape[0], dtype=torch.float64), torch.zeros(L.shape[0], dtype=torch.float64)
    for t in range(min(K, 128)):
        Lt = L[:, vt == t]
        e = torch.exp(Lt - Lt.max(1, keepdim=True).values)
        Sx, Wx = Sx + e.sum(1), Wx + (e * s[vt == t]).sum(1)
    out["no rescale"] = h(Wx / Sx)
    return out


def sensitivity(acc, v_list, order="canonical"):
    """acc: {variant: any root outside}; v_list: [(variants dict, logits, support)]"""
    for var, logits, support in v_list:
        for name, vv in var.items():
            acc[name] = acc.get(name, False) or bool(outside_band(vv, logits, support, order).any())


# ------------------------------------------------------------------------------------------------ the stand-alone transform
@pytest.mark.parametrize("support", SUPPORTS, ids=str)
def test_standalone_transform_against_float64(support):
    import lightzero_b200 as lzb
    tr = lzb.InverseScalarTransform(lzb.DiscreteSupport(*support))
    K = tr.support.size
    s = sup32(support)
    # one-hot at every k: F32(s_k) bit for bit
    L = torch.full((K, K), -1000.0)
    L[torch.arange(K), torch.arange(K)] = 0.0
    v = tr(L.cuda()).cpu().reshape(-1)
    assert torch.equal(bits(v), bits(f32_cpu(s))), "one-hot"
    g = torch.Generator().manual_seed(K)
    acc, report = {}, []
    for name in PROFILES:
        for B in (1, 3, 4, 5, 1201):
            logits = profile_logits(name, K, B, g)
            v = tr(logits.cuda()).cpu().reshape(-1)
            report.append((name, B, check_band(v, logits, support, (support, name, B))))
            if B == 1201:
                sensitivity(acc, [(variants(logits, support), logits, support)])
    worst = {}
    for name, B, r in report:
        worst[name] = max(worst.get(name, 0.0), r)
    print(f"\n[readout] standalone {support}: worst |v - F32(x64)| / band: " +
          ", ".join(f"{k} {w:.3f}" for k, w in worst.items()) + "; variants outside the band: " + str(acc))
    assert all(acc.values()) and len(acc) == 4, acc


@pytest.mark.parametrize("support", SUPPORTS, ids=str)
def test_standalone_transform_edges(support):
    """-inf logits (at the first position of a virtual thread, and rows with one finite logit), all-equal logits"""
    import lightzero_b200 as lzb
    tr = lzb.InverseScalarTransform(lzb.DiscreteSupport(*support))
    K = tr.support.size
    g = torch.Generator().manual_seed(7)
    rows = []
    for first in sorted({0, 1, 31, 32, 127, K - 1} & set(range(K))):
        r = torch.randn(K, generator=g)
        r[first] = -math.inf                      # -inf at the first logit a virtual thread sees
        rows.append(r)
        one = torch.full((K,), -math.inf)
        one[first] = float(torch.randn(1, generator=g))
        rows.append(one)                         # one finite logit
    r = torch.randn(K, generator=g)
    r[: min(K, 128)] = -math.inf                 # every virtual thread starts at -inf
    if K > 128:
        rows.append(r)
    rows += [torch.zeros(K), torch.full((K,), 3.5), torch.full((K,), -1000.0)]
    L = torch.stack(rows)
    v = tr(L.cuda()).cpu().reshape(-1)
    assert torch.isfinite(v).all(), v
    fin = torch.isfinite(L).sum(1) == 1
    exp = f32_cpu(sup32(support)[torch.isfinite(L[fin]).int().argmax(1)])
    assert torch.equal(bits(v[fin]), bits(exp)), "rows with one finite logit: F32(s_k)"
    lo, hi = band(*x64_and_bound(L, support))
    assert ((v >= lo) & (v <= hi)).all()
    assert torch.equal(v[-3:], v[-3:].flip(0)), "all-equal rows give one value"


# ------------------------------------------------------------------------------------------------ the model families
def shape_heads(bias, alpha):
    """mutate: the last Linear of every value / reward / value-prefix head gets weight * alpha and bias `bias`"""
    @torch.no_grad()
    def mutate(ref):
        for name, mod in ref.named_modules():
            if name.split(".")[-1] in ("fc_value", "fc_value_head", "fc_reward_head"):
                fc = [m for m in mod.modules() if isinstance(m, torch.nn.Linear)][-1]
                fc.weight.mul_(alpha)
                fc.bias.copy_(bias.to(fc.bias.dtype))
    return mutate


def mlp_pair(family, support, seed):
    """(restatement, CUDA model) of the family's MLP config with the given support"""
    import lightzero_b200 as lzb
    import mlp_ez_model_ref as EZ
    import mlp_fp32_model_ref as MF
    import mlp_mz_model_ref as MZ
    from oracle.model_ref import MuZeroModelMLPRef, emulate_trained_mlp_
    mod, name, cls, rcls = {"mlp_fp32": (MF, "cartpole", lzb.MuZeroModelMLP, MuZeroModelMLPRef),
                            "mlp_tc": (MZ, "lunarlander", lzb.MuZeroModelMLP, MuZeroModelMLPRef),
                            "mlp_ez": (EZ, "cartpole", lzb.EfficientZeroModelMLP, EZ.EfficientZeroModelMLPRef)}[family]
    kw = dict(mod.model_kwargs(name), reward_support_range=support, value_support_range=support)
    torch.manual_seed(seed)
    return emulate_trained_mlp_(rcls(**kw), seed).eval(), cls, kw


def family_outputs(family, support, mutate, B, seed):
    """[(what, logits fp32, scalar, read-out order)] of one model family on B roots: "canonical" (bits of
    lz_inverse_scalar_transform) or "quad" (mlp_tc.cu)"""
    import lightzero_b200 as lzb
    from oracle.model_ref import EfficientZeroModelRef, MuZeroModelRef, emulate_trained_
    g = torch.Generator().manual_seed(seed)
    act = torch.randint(0, 6, (B,), generator=g).cuda()
    if family in ("conv", "conv8", "conv_ez"):
        # conv: 84 px (6x6 latent); conv8: 64 px (8x8 latent, the Atari configs); conv_ez: 96 px EfficientZero
        px = {"conv": 84, "conv8": 64, "conv_ez": 96}[family]
        kw = dict(reward_support_range=support, value_support_range=support)
        torch.manual_seed(seed)
        if family == "conv_ez":
            kw["lstm_hidden_size"] = 64
        ref = emulate_trained_((EfficientZeroModelRef if family == "conv_ez" else MuZeroModelRef)((4, px, px), 6, **kw), seed)
        mutate(ref)
        cls = lzb.EfficientZeroModel if family == "conv_ez" else lzb.MuZeroModel
        cu = cls(observation_shape=(4, px, px), action_space_size=6, downsample=True, **kw).load_state_dict(ref.state_dict())
        o0 = cu.initial_inference(torch.rand(B, 4, px, px, generator=g).cuda(), return_scalar_value=True)
        latent = o0.latent_state * 4.0
        if family == "conv_ez":
            H = cu.lstm_hidden_size
            hc = (torch.randn(1, B, H, generator=g).cuda() * 0.5, torch.randn(1, B, H, generator=g).cuda())
            o1 = cu.recurrent_inference(latent, hc, act, return_scalars=True)
            return [("init value", o0.value, o0.value_scalar, "canonical"), ("value", o1.value, o1.value_scalar, "canonical"),
                    ("value prefix", o1.value_prefix, o1.value_prefix_scalar, "canonical")]
        o1 = cu.recurrent_inference(latent, act, return_scalars=True)
    elif family == "board":
        import board_model_ref as BR
        kw = dict(BR.model_kwargs("gomoku"), reward_support_range=support, value_support_range=support)
        torch.manual_seed(seed)
        ref = emulate_trained_(BR.BoardMuZeroModelRef(**kw), seed)
        mutate(ref)
        cu = lzb.MuZeroModel(**kw).load_state_dict(ref.state_dict())
        o0 = cu.initial_inference(torch.rand((B,) + BR.BOARD_CONFIGS["gomoku"][0], generator=g).cuda(), return_scalar_value=True)
        o1 = cu.recurrent_inference(o0.latent_state, act % cu.action_space_size, return_scalars=True)
    else:
        ref, cls, kw = mlp_pair(family, support, seed)
        mutate(ref)
        cu = cls(**kw).load_state_dict(ref.state_dict())
        obs = torch.rand(B, cu.observation_shape, generator=g).cuda() * 2 - 1
        act = act % cu.action_space_size
        o0 = cu.initial_inference(obs, return_scalar_value=True)
        order = "canonical" if family == "mlp_fp32" else "quad"
        if family == "mlp_ez":
            H = cu.lstm_hidden_size
            hc = (torch.rand(1, B, H, generator=g).cuda() - 0.5, torch.randn(1, B, H, generator=g).cuda())
            o1 = cu.recurrent_inference(o0.latent_state, hc, act, return_scalars=True)
            return [("init value", o0.value, o0.value_scalar, order), ("value", o1.value, o1.value_scalar, order),
                    ("value prefix", o1.value_prefix, o1.value_prefix_scalar, "canonical")]
        o1 = cu.recurrent_inference(o0.latent_state, act, return_scalars=True)
        return [("init value", o0.value, o0.value_scalar, order), ("value", o1.value, o1.value_scalar, order),
                ("reward", o1.reward, o1.reward_scalar, order)]
    return [("init value", o0.value, o0.value_scalar, "canonical"), ("value", o1.value, o1.value_scalar, "canonical"),
            ("reward", o1.reward, o1.reward_scalar, "canonical")]


def profile_biases(name, K, g):
    """the bias rows a profile is shaped with: the peak at the lower edge, the upper edge and inside; one row otherwise"""
    rows = profile_logits(name, K, 3, g)
    return list(rows) if name == "peak" else [rows[2]]


# every family accepts every support of SUPPORTS (2 <= K <= 608 for all of them)
FAMILIES = [(f, s) for f in ("conv", "conv8", "conv_ez", "board", "mlp_fp32", "mlp_tc", "mlp_ez") for s in SUPPORTS]


@pytest.mark.parametrize("family,support", FAMILIES, ids=lambda v: str(v))
def test_model_readout_against_float64(family, support):
    """Every profile through the model's heads: the band, one-hot bits, and the canonical families' bit identity with
    lz_inverse_scalar_transform of their own logits"""
    import lightzero_b200 as lzb
    K = len(sup32(support))
    s = sup32(support)
    g = torch.Generator().manual_seed(K + len(family))
    B = 133
    worst, acc, big = {}, {}, 0.0
    transform = lzb.InverseScalarTransform(lzb.DiscreteSupport(*support))
    for pi, name in enumerate(PROFILES):
        if name == "onehot":
            shapes = []
            for k in sorted({0, 1, K // 2, K - 2, K - 1}):
                bias = torch.full((K,), -1000.0)
                bias[k] = 0.0
                shapes.append((k, bias, 0.0))
        else:
            shapes = [(None, bias, 1e-3) for bias in profile_biases(name, K, g)]
        for k, bias, alpha in shapes:
            for what, logits, v, order in family_outputs(family, support, shape_heads(bias, alpha), B, seed=pi + 3):
                v = v.reshape(-1)
                if k is not None:
                    assert torch.equal(bits(v.cpu()), bits(f32_cpu(s[k:k + 1]).expand(B))), (what, k)
                if order == "canonical":
                    again = transform(logits).reshape(-1)
                    assert torch.equal(bits(again), bits(v)), (what, name, "not the canonical read-out")
                r = check_band(v, logits, support, (family, support, name, what), order)
                worst[f"{name}/{what}"] = max(worst.get(f"{name}/{what}", 0.0), r)
                sensitivity(acc, [(variants(logits, support), logits, support)], order)
                big = max(big, v.abs().max().item())
    print(f"\n[readout] {family} {support}: max |scalar| {big:.4g}; worst |v - F32(x64)| / band: " +
          ", ".join(f"{k} {w:.3f}" for k, w in worst.items()) + "; variants outside the band: " + str(acc))
    assert all(acc.values()) and len(acc) == 4, acc


# ------------------------------------------------------------------------------------------------ searches at large values
@torch.no_grad()
def large_values(ref):
    """value and reward (value prefix) logits peaked at about support index K/2 + 0.32 K (support +190 of +-300), the
    weights scaled so that the peak moves from node to node: scalars in the 10^4"""
    for name, mod in ref.named_modules():
        if name.split(".")[-1] in ("fc_value", "fc_value_head", "fc_reward_head"):
            fc = [m for m in mod.modules() if isinstance(m, torch.nn.Linear)][-1]
            K = fc.bias.numel()
            k = torch.arange(K, dtype=fc.bias.dtype)
            fc.weight.mul_(40.0)
            fc.bias.copy_(-((k - (K // 2 + int(0.32 * K))) / (0.05 * K)) ** 2)


def assert_large(what, *scalars):
    m = [float(np.abs(np.asarray(x, np.float64)).max()) for x in scalars]
    print(f"\n[readout] search {what}: max |scalar| " + ", ".join(f"{v:.4g}" for v in m))
    assert min(m) > 1e3, (what, m)


SEARCH_CASES = {
    "a18_b131_det_1p": (18, 131, 50, True, "1p", 0.997, 0.01),
    "a18_b131_sto_1p": (18, 131, 50, False, "1p", 0.997, 0.01),
    "a18_b131_sto_2p": (18, 131, 50, False, "2p", 0.997, 0.01),
    "a18_b131_det_2p_delta": (18, 131, 50, True, "2p", 0.997, 0.5),
    "a33_b40_sto_2p": (33, 40, 20, False, "2p", 0.997, 0.01),
}


@pytest.mark.parametrize("name", list(SEARCH_CASES))
def test_search_at_large_values_equals_oracle(name):
    import lightzero_b200 as lzb
    from oracle.tree_drive import assert_same
    from test_gpu_net_layers import make_latents, make_models
    from test_gpu_search_oracle import _inputs, fused_search, oracle_search, visits_sum_to
    A, B, S, det, players, discount, delta = SEARCH_CASES[name]
    seed = sum(map(ord, name)) % 97
    _, cu = make_models(A=A, seed=seed, mutate=large_values)
    latent = make_latents(B, seed)
    o = cu.recurrent_inference(latent, torch.arange(B, device="cuda") % A, return_scalars=True)
    vmax, rmax = o.value_scalar.abs().max().item(), o.reward_scalar.abs().max().item()
    legal, logits, noises, tp = _inputs(B, A, seed, players)
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=det, discount_factor=discount, value_delta_max=delta))
    got, key, plan, roots = fused_search(cu, mcts, S, latent, legal, logits, noises, tp)
    exp, st = oracle_search(cu, S, latent, legal, logits, noises, tp, det, key=key, discount=discount, delta=delta)
    kernels = mcts.last_num_kernels
    roots.clear()
    rv = np.abs(got["root_values_bits"].view(np.float32)).max()
    print(f"\n[readout] search {name}: max |value| {vmax:.4g}, max |reward| {rmax:.4g}, max |root value| {rv:.4g}, "
          f"kernels {kernels}, ties {st['ties']}")
    assert vmax > 1e3 and rmax > 1e3 and rv > 1e3
    assert_same(got, exp)
    assert visits_sum_to(got, S)
    assert plan["persistent"] == (A <= 32)


@pytest.mark.parametrize("det,players", [(True, "1p"), (False, "2p")])
def test_efficientzero_search_at_large_values_equals_oracle(det, players):
    """EfficientZeroMCTSCtree at horizon 5 (96 px, K = 601): value prefixes and values above 10^3.  A = 2 so that paths
    grow past the horizon and the value prefix is reset inside the search."""
    from oracle.tree_drive import assert_same
    from test_gpu_ez_oracle import D96, _mcts, _setup, fused_search_ez, oracle_search_ez
    from test_gpu_search_oracle import visits_sum_to
    A, B, S, horizon = 2, 131, 50, 5
    cu, latent, h0, c0, legal, logits, noises, tp = _setup(D96, A, B, 17 + det, players, {}, mutate=large_values)
    o = cu.recurrent_inference(latent, (h0[None], c0[None]), torch.arange(B, device="cuda") % A, return_scalars=True)
    mcts = _mcts(S, det, horizon)
    got, key, roots = fused_search_ez(cu, mcts, latent, h0, c0, legal, logits, noises, tp)
    exp, st, resets = oracle_search_ez(cu, S, horizon, latent, h0, c0, legal, logits, noises, tp, det, key=key)
    roots.clear()
    assert_large(f"ez det={det} {players} resets={resets} max_len={st['max_len']}", o.value_prefix_scalar.cpu(), o.value_scalar.cpu(),
                 got["root_values_bits"].view(np.float32))
    assert_same(got, exp)
    assert visits_sum_to(got, S) and resets > 0


@pytest.mark.parametrize("family", ["mlp_fp32", "mlp_tc", "mlp_ez"])
def test_mlp_search_at_large_values_equals_oracle(family):
    """both MuZeroModelMLP kernels (multi-kernel graph) and EfficientZeroModelMLP (horizon 5), stochastic, two players"""
    from oracle.tree_drive import assert_same
    from test_gpu_search_oracle import _inputs, fused_search, oracle_search, visits_sum_to
    ref, cls, kw = mlp_pair(family, (-300., 301., 1.), 23)
    large_values(ref)
    cu = cls(**kw).load_state_dict(ref.state_dict())
    A, B, S = cu.action_space_size, 96, 25
    g = torch.Generator().manual_seed(4)
    latent = cu.initial_inference((torch.rand(B, cu.observation_shape, generator=g) * 2 - 1).cuda()).latent_state
    legal, logits, noises, tp = _inputs(B, A, 5, "2p")
    act = torch.arange(B, device="cuda") % A
    if family == "mlp_ez":
        import lightzero_b200 as lzb
        from test_gpu_ez_oracle import fused_search_ez, hidden, oracle_search_ez
        h0, c0 = hidden(B, cu.lstm_hidden_size, 5)
        o = cu.recurrent_inference(latent, (h0[None], c0[None]), act, return_scalars=True)
        scalars = (o.value_prefix_scalar.cpu(), o.value_scalar.cpu())
        mcts = lzb.EfficientZeroMCTSCtree(dict(num_simulations=S, deterministic=False, discount_factor=0.997, lstm_horizon_len=5))
        got, key, roots = fused_search_ez(cu, mcts, latent, h0, c0, legal, logits, noises, tp)
        exp, _, _ = oracle_search_ez(cu, S, 5, latent, h0, c0, legal, logits, noises, tp, False, key=key)
    else:
        import lightzero_b200 as lzb
        o = cu.recurrent_inference(latent, act, return_scalars=True)
        scalars = (o.reward_scalar.cpu(), o.value_scalar.cpu())
        mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=False, discount_factor=0.997))
        got, key, _, roots = fused_search(cu, mcts, S, latent, legal, logits, noises, tp)
        exp, _ = oracle_search(cu, S, latent, legal, logits, noises, tp, False, key=key)
    roots.clear()
    assert_large(family, *scalars, got["root_values_bits"].view(np.float32))
    assert_same(got, exp)
    assert visits_sum_to(got, S)


@pytest.mark.parametrize("obs,A,m", [((4, 64, 64), 18, 8), (4, 2, 2)], ids=["conv64_a18_m8", "mlp_a2"])
def test_gumbel_search_at_large_values_equals_reference_tree(obs, A, m):
    """GumbelMuZeroMCTSCtree against the compiled reference tree driving the same network: the completed Q and the
    sigma transform of the improved policy see values above 10^3"""
    import lightzero_b200 as lzb
    from oracle.model_ref import MuZeroModelMLPRef, MuZeroModelRef, emulate_trained_, emulate_trained_mlp_
    from oracle.tree_drive import assert_same
    from test_gpu_gumbel import _fused_search, _oracle, _oracle_search, _roots_inputs
    B, S = 131, 50
    if isinstance(obs, tuple):
        ref = emulate_trained_(MuZeroModelRef(obs, A), 3)
        large_values(ref)
        model = lzb.MuZeroModel(observation_shape=obs, action_space_size=A, downsample=True).load_state_dict(ref.state_dict())
    else:
        ref = emulate_trained_mlp_(MuZeroModelMLPRef(obs, A, res_connection_in_dynamics=True), 5)
        large_values(ref)
        model = lzb.MuZeroModelMLP(observation_shape=obs, action_space_size=A, res_connection_in_dynamics=True).load_state_dict(ref.state_dict())
    out, legal, noises = _roots_inputs(model, B, A, obs, 11, True)
    o = model.recurrent_inference(out.latent_state, torch.arange(B, device="cuda") % A, return_scalars=True)
    got, mcts, roots = _fused_search(model, out, legal, noises, B, A, S, m)
    roots.clear()
    assert_large(f"gumbel {obs} A={A}", out.value_scalar.cpu(), o.reward_scalar.cpu(), o.value_scalar.cpu(),
                 got["root_values_bits"].view(np.float32))
    assert_same(got, _oracle_search(_oracle(), model, out, legal, noises, B, A, S, m))
