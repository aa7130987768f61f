"""CPU checks of the MuZeroModelMLP configs that run on the tensor-core MLP kernel: the PyTorch restatement
(oracle.model_ref.MuZeroModelMLPRef) against the fixtures of the reference class, and the fixtures regenerated from the
reference class when its sources are present."""
import os
import sys

import numpy as np
import pytest
import torch

import mlp_mz_model_ref as MR
from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden")
if GOLDEN not in sys.path:
    sys.path.insert(0, GOLDEN)      # the fixture generators
REF = os.environ.get("LZ_REFERENCE", "/root/reference")
NAMES = list(MR.CONFIGS)


@pytest.mark.parametrize("name", NAMES)
def test_restatement_reproduces_the_fixture(name):
    from make_model_golden import weights_digest
    d = np.load(os.path.join(GOLDEN, f"mlp_mz_{name}.npz"))
    mine = MR.build(name, int(d["seed"]))
    assert weights_digest(mine) == str(d["weights_sha256"])
    obs, action = torch.from_numpy(d["obs"]), torch.from_numpy(d["action"])
    with torch.no_grad():
        o0 = mine.initial_inference(obs)
        o1 = mine.recurrent_inference(o0.latent_state, action)
    for f in ("value", "policy_logits", "latent_state"):
        assert torch.equal(getattr(o0, f), torch.from_numpy(d["init_" + f])), f
    for f in ("value", "reward", "policy_logits", "latent_state"):
        assert torch.equal(getattr(o1, f), torch.from_numpy(d["rec_" + f])), f
    assert float(torch.from_numpy(d["rec_reward"]).std()) > 0      # an emulated-trained reward head, not the zero init


@pytest.mark.parametrize("name", NAMES)
def test_fixture_regenerates_from_the_reference_class(name):
    if not os.path.isdir(os.path.join(REF, "lzero", "model")):
        pytest.skip("reference sources not present")
    import make_mlp_mz_golden as G
    d = np.load(os.path.join(GOLDEN, f"mlp_mz_{name}.npz"))
    out = G.case_outputs(G.reference_module(), name, int(d["seed"]))
    assert sorted(out) == sorted(d.files)
    for k in d.files:
        assert np.array_equal(np.asarray(out[k]), d[k]) and np.asarray(out[k]).dtype == d[k].dtype, k


def test_table_configs_are_outside_the_fp32_kernels_and_inside_the_tensor_core_one():
    """every fixture config is one lz_model_create_mlp sends to the tensor-core kernel (model kind 4)"""
    for name, (obs, A, L, res, hid, sup) in MR.CONFIGS.items():
        fp32 = 8 <= L <= 128 and obs <= 160 and L + A <= 160
        tc = L % 32 == 0 and 32 <= L <= 256 and 1 <= obs <= 4096 and 1 <= A <= 608 and 1 <= hid <= 32
        assert tc and not fp32, name
        assert len(torch.arange(*sup)) <= 608, name
