"""CPU-side checks of the drop-in boundary: the C-ABI library builds for sm_90a, loads without a GPU
and exports every symbol include/lzb200.h declares; the product package never imports the oracle."""
import ctypes
import os
import re
import subprocess
import sys

from conftest import ROOT


def _header_functions():
    src = open(os.path.join(ROOT, "include", "lzb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(lz_[a-z_0-9]+)\s*\(", src)))


def test_library_builds_and_exports_every_declared_symbol():
    from lightzero_b200 import _build, cabi
    lib_path = _build.build()
    assert os.path.exists(lib_path)
    lib = ctypes.CDLL(lib_path)
    declared = _header_functions()
    assert len(declared) >= 25
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/lzb200.h but not exported"
    assert sorted(cabi.SIGNATURES) == declared, "ctypes table and header disagree"
    assert cabi.load().lz_version() >= 100


def test_library_contains_sm90a_code():
    from lightzero_b200 import _build
    out = subprocess.run(["cuobjdump", "-lelf", _build.build()], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out


def test_no_device_is_a_loud_error():
    """Without a GPU the create calls must fail with LZ_ECUDA and a message, never fall back."""
    import torch
    if torch.cuda.is_available():
        return
    from lightzero_b200 import cabi
    lib = cabi.load()
    h = ctypes.c_void_p()
    rc = lib.lz_tree_create(4, 6, 10, h)
    assert rc < 0 and lib.lz_last_error()
    import pytest
    import lightzero_b200 as lzb
    with pytest.raises(RuntimeError):
        lzb.MuZeroModel()
    with pytest.raises(RuntimeError):
        lzb.mz_tree.Roots(2, [[0, 1], [0, 1]])


def test_product_package_never_touches_the_oracle():
    pkg = os.path.join(ROOT, "lightzero_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt and "oracle/" not in txt, f


def test_tree_unit_is_compiled_without_fma_contraction():
    """Bit-exactness of the tree depends on -fmad=false for tree.cu: no FFMA may appear in the tree
    kernels except inside the IEEE division / sqrt helper sequences (which are exactly rounded)."""
    from lightzero_b200 import _build
    _build.build()
    obj = os.path.join(ROOT, "lightzero_b200", "_lib", "tree.o")
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    # the tree step kernel in all four (EfficientZero x reuse) instantiations
    assert sum("Function :" in l and "k_tree_step" in l for l in sass.splitlines()) == 4
    # every explicit op is __f*_rn; what the compiler may not do is fuse them: count plain FMUL/FADD present
    assert sass.count("FMUL") > 10 and sass.count("FADD") > 10
