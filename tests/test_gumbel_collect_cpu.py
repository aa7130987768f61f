"""CPU checks of the Gumbel MuZero collect: the read-out kernel of csrc/gumbel.cu is built without fp32 contraction and
without spills, the collector kernels without spills, the new C entry points are declared and exported, and the collect
policy refuses EfficientZero models before touching a device."""
import os
import re
import subprocess

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "lightzero_b200", "csrc")


def _ptx_entry(ptx, name):
    """The body of the .entry whose mangled name contains `name`"""
    m = re.search(r"\.entry\s+(\S*" + name + r"\S*)\(.*?^}", ptx, flags=re.S | re.M)
    assert m, name
    return m.group(0)


def test_readout_kernel_has_no_fp32_contraction(tmp_path):
    """k_gumbel_readout (compiled -fmad=false with the rest of gumbel.cu): no fp32 fma in its PTX; the fma.rn.f64 are the
    explicit ones of the expf / logf restatements and libdevice's fp64 pow / log of the entropy"""
    ptx = str(tmp_path / "gumbel.ptx")
    subprocess.check_call(["nvcc", "-arch=sm_90a", "-std=c++17", "-fmad=false", "-ptx", os.path.join(CSRC, "gumbel.cu"), "-o", ptx])
    body = _ptx_entry(open(ptx).read(), "k_gumbel_readout")
    assert "fma.rn.f32" not in body and "mad.f32" not in body and "fma.rn.ftz.f32" not in body
    assert "div.rn.f32" in body and "fma.rn.f64" in body
    assert "k_gumbel_policies" not in open(os.path.join(CSRC, "gumbel.cu")).read()     # one read-out kernel, not two


@pytest.mark.parametrize("unit,flags,kernels", [
    ("gumbel.cu", ["-fmad=false"], ["k_gumbel_readout"]),
    ("collector.cu", [], ["k_segments_store_policy", "k_segments_clear_rows"]),
])
def test_kernels_do_not_spill(tmp_path, unit, flags, kernels):
    out = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17"] + flags +
                         ["-Xptxas", "-v", "-c", os.path.join(CSRC, unit), "-o", str(tmp_path / "u.o")],
                         capture_output=True, text=True, check=True).stderr
    for k in kernels:
        m = re.search(r"Compiling entry function '(\S*" + k + r"\S*)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", out, re.S)
        assert m, k
        assert m.group(2) == "0" and m.group(3) == "0", (k, m.group(0))


def test_entry_points_declared_and_exported():
    import ctypes
    from lightzero_b200 import _build, cabi
    header = open(os.path.join(ROOT, "include", "lzb200.h")).read()
    lib = ctypes.CDLL(_build.build())
    for name in ("lz_tree_gumbel_select_action", "lz_segments_store_improved_policy", "lz_segments_improved_policy"):
        assert re.search(r"\b" + name + r"\s*\(", header) and name in cabi.SIGNATURES and hasattr(lib, name), name
    lib = cabi.load()
    assert lib.lz_tree_gumbel_select_action(None, 1.0, None, None, None, None, None) < 0
    assert lib.lz_segments_store_improved_policy(None, None, None, None) < 0
    assert lib.lz_segments_improved_policy(None, None) < 0


def test_collect_policy_refuses_efficientzero_models():
    import lightzero_b200 as lzb
    for cls in (lzb.EfficientZeroModel, lzb.EfficientZeroModelMLP):
        with pytest.raises(TypeError, match="MuZero models"):
            lzb.GumbelMuZeroCollectPolicy(cls.__new__(cls))
