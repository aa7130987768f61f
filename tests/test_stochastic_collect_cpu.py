"""CPU checks of the Stochastic MuZero collect: the collect policy refuses every model but StochasticMuZeroModelMLP before
touching a device, the kernels a stochastic collect step runs and this change touches (the MlpTc network, the tree's mask reset,
step, read-out and select_action) neither spill nor use local memory, and the collect entry points keep their declarations."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "lightzero_b200", "csrc")


def test_collect_policy_refuses_other_models():
    import lightzero_b200 as lzb
    for cls in (lzb.MuZeroModel, lzb.MuZeroModelMLP, lzb.EfficientZeroModel, lzb.EfficientZeroModelMLP):
        with pytest.raises(TypeError, match="StochasticMuZeroModelMLP"):
            lzb.StochasticMuZeroCollectPolicy(cls.__new__(cls))


def test_pad_columns():
    import numpy as np
    import torch
    from lightzero_b200.collect import _pad_columns
    m = np.array([[1, 0], [0, 1]], np.uint8)
    assert _pad_columns(m, 3).tolist() == [[1, 0, 0], [0, 1, 0]] and _pad_columns(m, 3).dtype == np.uint8
    t = torch.tensor([[0.5, 0.25]])
    assert _pad_columns(t, 4).tolist() == [[0.5, 0.25, 0.0, 0.0]]
    assert _pad_columns(torch.from_numpy(m), 2).tolist() == m.tolist()


KERNELS = {"mlp_tc.cu": ["k_mez_tc"],
           "tree.cu": ["k_tree_reset", "k_tree_stepILb0ELb0E", "k_tree_results", "k_tree_select_action"]}


def _local_memory(obj):
    """kernel -> number of local-memory instructions (STL / LDL) in its SASS"""
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out.setdefault(cur, 0)
        elif cur and re.search(r"\b(STL|LDL)\b", line):
            out[cur] += 1
    return out


def test_collect_kernels_do_not_spill():
    if shutil.which("nvcc") is None or shutil.which("cuobjdump") is None:
        pytest.skip("nvcc / cuobjdump not on PATH")
    from lightzero_b200 import _build
    flags = dict(_build.UNITS)
    with tempfile.TemporaryDirectory() as tmp:
        log, local = "", {}
        for unit, kernels in KERNELS.items():
            obj = os.path.join(tmp, unit.replace(".cu", ".o"))
            p = subprocess.run(["nvcc"] + _build.ARCH + _build.COMMON + flags[unit] + ["-Xptxas", "-v", "-c",
                               os.path.join(CSRC, unit), "-o", obj], capture_output=True, text=True)
            assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
            log += p.stdout + p.stderr
            local.update({k: v for k, v in _local_memory(obj).items() if any(n in k for n in kernels)})
    names = [n for ks in KERNELS.values() for n in ks]
    seen = set()
    for m in re.finditer(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log):
        hit = [n for n in names if n in m.group(1)]
        if hit:
            assert m.group(3) == "0" and m.group(4) == "0", m.group(0)
            seen.update(hit)
    assert seen == set(names), set(names) - seen
    assert local and not any(local.values()), local


def test_collect_entry_points_declared():
    from lightzero_b200 import cabi
    header = open(os.path.join(ROOT, "include", "lzb200.h")).read()
    for name in ("lz_search_collect", "lz_search_collect_host", "lz_tree_select_action", "lz_tree_set_stochastic"):
        assert re.search(r"\b" + name + r"\s*\(", header) and name in cabi.SIGNATURES, name
