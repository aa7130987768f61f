"""CPU checks of EfficientZeroModelMLP: the PyTorch restatement (tests/mlp_ez_model_ref.py) against the fixtures of the reference
class, the fixtures regenerated from the reference class when its sources are present, and the register budget of the
tensor-core kernel (no spills, no local memory, no serialised wgmma)."""
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import mlp_ez_model_ref as MR
from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden")
if GOLDEN not in sys.path:
    sys.path.insert(0, GOLDEN)      # the fixture generators
REF = os.environ.get("LZ_REFERENCE", "/root/reference")
NAMES = list(MR.CONFIGS)


@pytest.mark.parametrize("name", NAMES)
def test_restatement_reproduces_the_fixture(name):
    from make_model_golden import weights_digest
    d = np.load(os.path.join(GOLDEN, f"mlp_ez_{name}.npz"))
    mine = MR.build(name, int(d["seed"]))
    assert weights_digest(mine) == str(d["weights_sha256"])
    obs, action = torch.from_numpy(d["obs"]), torch.from_numpy(d["action"])
    h0, c0 = torch.from_numpy(d["h0"]), torch.from_numpy(d["c0"])
    assert float(h0.abs().sum()) > 0 and float(c0.abs().sum()) > 0
    with torch.no_grad():
        o0 = mine.initial_inference(obs)
        o1 = mine.recurrent_inference(o0.latent_state, (h0, c0), action)
    for f in ("value", "policy_logits", "latent_state"):
        assert torch.equal(getattr(o0, f), torch.from_numpy(d["init_" + f])), f
    for f in ("value", "value_prefix", "policy_logits", "latent_state"):
        assert torch.equal(getattr(o1, f), torch.from_numpy(d["rec_" + f])), f
    for i, f in enumerate(("h", "c")):
        assert torch.equal(o1.reward_hidden_state[i], torch.from_numpy(d["rec_" + f])), f


@pytest.mark.parametrize("name", NAMES)
def test_fixture_regenerates_from_the_reference_class(name):
    if not os.path.isdir(os.path.join(REF, "lzero", "model")):
        pytest.skip("reference sources not present")
    import make_mlp_ez_golden as G
    d = np.load(os.path.join(GOLDEN, f"mlp_ez_{name}.npz"))
    out = G.case_outputs(G.reference_module(), name, int(d["seed"]))
    assert sorted(out) == sorted(d.files)
    for k in d.files:
        assert np.array_equal(np.asarray(out[k]), d[k]) and np.asarray(out[k]).dtype == d[k].dtype, k


def test_table_configs_fit_the_accepted_space():
    for name, (obs, A, L, H, _) in MR.CONFIGS.items():
        assert L % 32 == 0 and 32 <= L <= 256 and H % 16 == 0 and 16 <= H <= 512 and 1 <= obs <= 4096 and 1 <= A <= 608, name


def test_mlp_tc_kernel_does_not_spill():
    if shutil.which("nvcc") is None or shutil.which("cuobjdump") is None:
        pytest.skip("nvcc / cuobjdump not on PATH")
    from lightzero_b200 import _build
    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, "mlp_tc.o")
        cmd = ["nvcc"] + _build.ARCH + _build.COMMON + ["-Xptxas", "-v", "-c", os.path.join(ROOT, "lightzero_b200", "csrc", "mlp_tc.cu"), "-o", obj]
        p = subprocess.run(cmd, capture_output=True, text=True)
        assert p.returncode == 0, p.stderr[-4000:]
        sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    log = p.stdout + p.stderr
    spills, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(_ZN2lz8k_mez_tcILi(\d+)E\S*)'", line)
        if m:
            cur = f"k_mez_tc<{m.group(2)}>"
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            spills[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    assert len(spills) == 8, sorted(spills)      # L = 32 .. 256
    assert all(v == (0, 0) for v in spills.values()), spills
    assert "C7514" not in log, "wgmma serialised"
    funcs = [f for f in re.split(r"Function : ", sass)[1:] if f.startswith("_ZN2lz8k_mez_tc")]
    assert len(funcs) == 8
    for f in funcs:
        assert not re.search(r"\b(STL|LDL)\b", f), f.split("\n", 1)[0]
