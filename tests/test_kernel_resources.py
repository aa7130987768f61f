"""CPU-side guard of the register budget of the wgmma kernels: net_tc.cu and conv_tc.cu compiled for sm_90a with `-Xptxas -v`.

What is checked, for every k_net_tc / k_resblock_tc / k_conv_tc instantiation:
  - ptxas reports no spill stores or loads, and the SASS has no local-memory instructions (STL / LDL);
  - the kernels of the wide layout (a producer warpgroup, 384 threads) contain the register reallocation (setmaxnreg), and those
    of the narrow layout (a producer warp, 288 threads) do not.
The register counts themselves are not asserted: __launch_bounds__ caps them (168 at launch; 112 for k_conv_tc<64, false>, two
CTAs per SM) and setmaxnreg caps the MMA warpgroups at 232, so a kernel that needs more spills instead, which the checks above
catch.  Needs nvcc, no GPU; skipped where nvcc is not on PATH."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "lightzero_b200", "csrc")

KERNELS = {"k_net_tc<6>", "k_net_tc<8>",
           "k_resblock_tc<32, false>", "k_resblock_tc<64, false>", "k_resblock_tc<64, true>",
           "k_conv_tc<64, false>", "k_conv_tc<128, false>", "k_conv_tc<128, true>"}
REALLOC = {"k_net_tc<6>", "k_net_tc<8>", "k_resblock_tc<64, true>", "k_conv_tc<128, true>"}
MANGLED = re.compile(r"_ZN2lz\d+(k_net_tc|k_resblock_tc|k_conv_tc)ILi(\d+)E(?:Lb([01])E)?E")


def _kernel(mangled):
    m = MANGLED.search(mangled)
    if not m:
        return None
    return f"{m.group(1)}<{m.group(2)}>" if m.group(3) is None else f"{m.group(1)}<{m.group(2)}, {'true' if m.group(3) == '1' else 'false'}>"


@pytest.fixture(scope="module")
def compiled():
    if shutil.which("nvcc") is None or shutil.which("cuobjdump") is None:
        pytest.skip("nvcc / cuobjdump not on PATH")
    from lightzero_b200 import _build
    with tempfile.TemporaryDirectory() as tmp:
        procs = []
        for unit in ("net_tc.cu", "conv_tc.cu"):
            obj = os.path.join(tmp, unit.replace(".cu", ".o"))
            cmd = ["nvcc"] + _build.ARCH + _build.COMMON + ["-Xptxas", "-v", "-c", os.path.join(CSRC, unit), "-o", obj]
            procs.append((obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        logs, sass = [], []
        for obj, p in procs:
            out, _ = p.communicate()
            assert p.returncode == 0, out[-4000:]
            logs.append(out)
            sass.append(subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout)
    return "\n".join(logs), "\n".join(sass)


def _ptxas_spills(log):
    """kernel -> (spill store bytes, spill load bytes) from the -Xptxas -v report"""
    table, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = _kernel(m.group(1))
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            table[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    return table


def _sass_functions(sass):
    """kernel -> its SASS text"""
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = _kernel(m.group(1))
            continue
        if cur is not None:
            out[cur] = out.get(cur, "") + line + "\n"
    return out


def test_wgmma_kernels_do_not_spill(compiled):
    table = _ptxas_spills(compiled[0])
    assert set(table) == KERNELS, sorted(table)
    for k in sorted(KERNELS):
        assert table[k] == (0, 0), f"{k}: {table[k][0]} B spill stores, {table[k][1]} B spill loads"
    funcs = _sass_functions(compiled[1])
    assert set(funcs) == KERNELS, sorted(funcs)
    for k in sorted(KERNELS):
        assert not re.search(r"\b(STL|LDL)\b", funcs[k]), f"{k}: local-memory traffic in the SASS"


def test_wide_layout_kernels_reallocate_registers_to_the_mma_warpgroups(compiled):
    funcs = _sass_functions(compiled[1])
    for k in sorted(KERNELS):
        has_realloc = "USETMAXREG" in funcs[k]
        assert has_realloc == (k in REALLOC), f"{k}: setmaxnreg {'missing' if k in REALLOC else 'unexpected'}"
