"""CPU checks of the board-game network (downsample=False): the PyTorch restatement (tests/board_model_ref.py) against the
fixtures of the reference class, the fixtures regenerated from the reference class when its sources are present, and the
register budget of the board kernel (no spills, no local memory)."""
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import board_model_ref as BR
from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden")
if GOLDEN not in sys.path:
    sys.path.insert(0, GOLDEN)      # the fixture generators
REF = os.environ.get("LZ_REFERENCE", "/root/reference")
NAMES = list(BR.BOARD_CONFIGS)


@pytest.mark.parametrize("name", NAMES)
def test_restatement_reproduces_the_fixture(name):
    from make_model_golden import weights_digest
    d = np.load(os.path.join(GOLDEN, f"board_{name}.npz"))
    mine = BR.build(name, int(d["seed"]))
    assert weights_digest(mine) == str(d["weights_sha256"])
    obs, action = torch.from_numpy(d["obs"]), torch.from_numpy(d["action"])
    with torch.no_grad():
        o0 = mine.initial_inference(obs)
        o1 = mine.recurrent_inference(o0.latent_state, action)
    for f in ("value", "policy_logits", "latent_state"):
        assert torch.equal(getattr(o0, f), torch.from_numpy(d["init_" + f])), f
    for f in ("value", "reward", "policy_logits", "latent_state"):
        assert torch.equal(getattr(o1, f), torch.from_numpy(d["rec_" + f])), f
    for f in ("init_value", "init_policy_logits", "rec_reward", "rec_value", "rec_policy_logits"):
        x = d[f]
        assert (x != x[:1]).any(), f        # every head depends on its root: none is a dead ReLU that outputs its bias


@pytest.mark.parametrize("name", NAMES)
def test_fixture_regenerates_from_the_reference_class(name):
    if not os.path.isdir(os.path.join(REF, "lzero", "model")):
        pytest.skip("reference sources not present")
    import make_board_golden as G
    d = np.load(os.path.join(GOLDEN, f"board_{name}.npz"))
    out = G.case_outputs(G.import_reference_models()[0], name, int(d["seed"]))
    assert sorted(out) == sorted(d.files)
    for k in d.files:
        assert np.array_equal(np.asarray(out[k]), d[k]) and np.asarray(out[k]).dtype == d[k].dtype, k


def test_board_kernel_does_not_spill():
    if shutil.which("nvcc") is None or shutil.which("cuobjdump") is None:
        pytest.skip("nvcc / cuobjdump not on PATH")
    from lightzero_b200 import _build
    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, "board_tc.o")
        cmd = ["nvcc"] + _build.ARCH + _build.COMMON + ["-Xptxas", "-v", "-c", os.path.join(ROOT, "lightzero_b200", "csrc", "board_tc.cu"), "-o", obj]
        p = subprocess.run(cmd, capture_output=True, text=True)
        assert p.returncode == 0, p.stderr[-4000:]
        sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    # the rule of test_kernel_resources.py (whose helpers name only the k_net_tc / k_resblock_tc / k_conv_tc instantiations)
    spills, cur = {}, None
    for line in p.stdout.splitlines() + p.stderr.splitlines():
        m = re.search(r"Compiling entry function '(_ZN2lz10k_board_tcILi(\d+)ELi(\d+)E\S*)'", line)
        if m:
            cur = f"k_board_tc<{m.group(2)}, {m.group(3)}>"
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            spills[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    assert len(spills) == 20, sorted(spills)      # C = 16, 32: NT = 1 .. 8; C = 64: NT = 1 .. 4
    assert all(v == (0, 0) for v in spills.values()), spills
    funcs = re.split(r"Function : ", sass)[1:]
    board = [f for f in funcs if f.startswith("_ZN2lz10k_board_tc")]
    assert len(board) == 20
    for f in board:
        assert not re.search(r"\b(STL|LDL)\b", f), f.split("\n", 1)[0]
        assert "USETMAXREG" not in f          # one warpgroup: nothing to reallocate, the launch gives it 255 registers
