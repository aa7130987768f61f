"""CPU checks of the Gumbel MuZero tree (csrc/gumbel.cu): the host tables against the compiled reference tree
(oracle/build_gmz_ref.py), the glibc-exact logf, the no-contraction build of gumbel.cu, and the C ABI without a device."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT


def _ref():
    from oracle import build_gmz_ref
    mod = build_gmz_ref.load()
    if mod is None:
        pytest.skip("compiled reference Gumbel tree not built (oracle/build_gmz_ref.py)")
    return mod


def _tables(m, S, A):
    from lightzero_b200 import cabi
    lib = cabi.load()
    seq = np.zeros(S, np.int32)
    gum = np.zeros(max(A, 1), np.float32)
    assert lib.lz_gumbel_tables(m, S, A, seq.ctypes.data, gum.ctypes.data) == 0
    return seq, gum[:A]


def test_gumbel_vector_matches_reference():
    ref = _ref()
    _, gum = _tables(1, 1, 82)
    for n in range(0, 83):
        exp = np.asarray(ref.pgenerate_gumbel(10.0, 0.0, n), np.float32)
        assert np.array_equal(exp.view(np.uint32), gum[:n].view(np.uint32)), n


def test_considered_visit_rows_match_reference():
    """row min(m, S) of get_table_of_considered_visits(m, S): every S in 1..800 for a spread of m, every m in 1..40 for
    S in 1..60 and a few larger budgets"""
    ref = _ref()
    cases = [(m, S) for m in (1, 2, 3, 4, 5, 7, 8, 16, 18, 33, 40) for S in range(1, 801)]
    cases += [(m, S) for m in range(1, 41) for S in list(range(1, 61)) + [64, 100, 128, 199, 200, 256, 333, 400, 512, 640, 799]]
    for m, S in cases:
        table = ref.pget_table_of_considered_visits(m, S)
        seq, _ = _tables(m, S, 0)
        assert table[min(m, S)] == seq.tolist(), (m, S)


def _golden():
    import glob
    import sys
    from conftest import GOLDEN_DIR
    sys.path.insert(0, GOLDEN_DIR)
    import make_gumbel_golden
    return make_gumbel_golden, sorted(glob.glob(os.path.join(GOLDEN_DIR, "gumbel_*.npz")))


def test_golden_fixtures_present():
    """one fixture per case of tests/golden/make_gumbel_golden.py, covering masked, single-action and m <= 1 roots"""
    gen, files = _golden()
    assert sorted(os.path.basename(f)[:-4] for f in files) == sorted(gen.CASES)
    kinds = set()
    for f in files:
        d = np.load(f)
        S, B = int(d["S"]), int(d["B"])
        assert d["exp_rec"].shape == (5, S, B)
        kinds |= {"masked" if (d["nlegal"] < int(d["A"])).any() else "full", "single" if (d["nlegal"] == 1).all() else "",
                  "m<=1" if int(d["m"]) <= 1 else ""}
    assert {"masked", "single", "m<=1"} <= kinds


def test_golden_fixtures_reproduce_from_reference():
    from oracle.tree_drive import check_fixture
    ref = _ref()
    _, files = _golden()
    for f in files:
        check_fixture(ref, np.load(f))


def test_logf_matches_libm(tmp_path):
    """every positive normal float with LZ_EXHAUSTIVE=1 (2.1e9 inputs, 0 mismatches), a strided sweep otherwise; plus
    expf on -inf and every float below -104 (the illegal entries of get_policies)"""
    exe = str(tmp_path / "check_logf")
    subprocess.check_call(["gcc", "-O2", "-o", exe, os.path.join(ROOT, "tests", "csrc", "check_logf.c"), "-lm"])
    stride = "1" if os.environ.get("LZ_EXHAUSTIVE") else "61"
    out = subprocess.run([exe, stride], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout
    assert "mismatches 0" in out.stdout


def test_gumbel_unit_has_no_fp32_contraction(tmp_path):
    """gumbel.cu is compiled with -fmad=false: its PTX has no fp32 fma (the only fma are the explicit double ones of the
    expf / logf restatements); FFMA in the SASS come only from the IEEE division sequences of div.rn.f32."""
    ptx = str(tmp_path / "gumbel.ptx")
    subprocess.check_call(["nvcc", "-arch=sm_90a", "-std=c++17", "-fmad=false", "-ptx",
                           os.path.join(ROOT, "lightzero_b200", "csrc", "gumbel.cu"), "-o", ptx])
    txt = open(ptx).read()
    assert "fma.rn.f32" not in txt and "mad.f32" not in txt and "fma.rn.ftz.f32" not in txt
    assert "div.rn.f32" in txt and "fma.rn.f64" in txt
    from lightzero_b200 import _build
    assert ("gumbel.cu", ["-fmad=false"]) in _build.UNITS


def test_gumbel_entry_points_exported_and_no_device_is_loud():
    from lightzero_b200 import _build, cabi
    lib = ctypes.CDLL(_build.build())
    for name in ("lz_tree_set_gumbel", "lz_tree_prepare", "lz_tree_traverse", "lz_tree_backpropagate",
                 "lz_tree_gumbel_policies", "lz_search_run", "lz_gumbel_tables"):
        assert hasattr(lib, name) and name in cabi.SIGNATURES, name
    lib = cabi.load()
    assert lib.lz_gumbel_tables(4, 0, 6, None, None) < 0 and b"bad arguments" in lib.lz_last_error()
    assert lib.lz_tree_set_gumbel(None, 4, 50) < 0
    assert lib.lz_search_run(None, None, 1, None) < 0
    import torch
    if torch.cuda.is_available():
        return
    import lightzero_b200 as lzb
    with pytest.raises(RuntimeError):
        lzb.gmz_tree.Roots(2, [[0, 1], [0, 1]])
