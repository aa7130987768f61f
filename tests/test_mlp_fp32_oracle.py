"""CPU checks of the MuZeroModelMLP configs that run on the fp32 MLP kernels (csrc/mlp.cu): the PyTorch restatement
(oracle.model_ref.MuZeroModelMLPRef) against the fixtures of the reference class, the fixtures regenerated from the
reference class when its sources are present, and the config table against the fp32 kernels' envelope."""
import math
import os
import sys

import numpy as np
import pytest
import torch

import mlp_fp32_model_ref as MR
from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden")
if GOLDEN not in sys.path:
    sys.path.insert(0, GOLDEN)      # the fixture generators
REF = os.environ.get("LZ_REFERENCE", "/root/reference")
NAMES = list(MR.CONFIGS)


@pytest.mark.parametrize("name", NAMES)
def test_restatement_reproduces_the_fixture(name):
    from make_model_golden import weights_digest
    d = np.load(os.path.join(GOLDEN, f"mlp_fp32_{name}.npz"))
    mine = MR.build(name, int(d["seed"]))
    assert weights_digest(mine) == str(d["weights_sha256"])
    obs, action = torch.from_numpy(d["obs"]), torch.from_numpy(d["action"])
    assert int(action.max()) == MR.CONFIGS[name][1] - 1
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
    import make_mlp_fp32_golden as G
    d = np.load(os.path.join(GOLDEN, f"mlp_fp32_{name}.npz"))
    out = G.case_outputs(G.reference_module(), name, int(d["seed"]))
    assert sorted(out) == sorted(d.files)
    for k in d.files:
        assert np.array_equal(np.asarray(out[k]), d[k]) and np.asarray(out[k]).dtype == d[k].dtype, k


def fp32_fits(obs, A, L, hid):
    """mlp_fits of csrc/mlp.cu"""
    return 8 <= L <= 128 and 1 <= obs <= 160 and A >= 1 and L + A <= 160 and hid <= 160


def support_size(sup):
    """lz_model_create_mlp's support size"""
    lo, hi, step = (np.float32(v) for v in sup)
    return int(math.ceil((hi - lo) / step))


@pytest.mark.parametrize("name", NAMES)
def test_table_config_is_inside_the_fp32_envelope(name):
    obs, A, L, res, hid, sup = MR.CONFIGS[name]
    assert fp32_fits(obs, A, L, hid), name
    K = len(torch.arange(*sup))
    assert support_size(sup) == K and 2 <= K <= 608, name


def test_table_reaches_every_edge_of_the_envelope():
    rows = MR.CONFIGS.values()
    assert min(L for _, _, L, *_ in rows) == 8 and max(L for _, _, L, *_ in rows) == 128
    assert max(obs for obs, *_ in rows) == 160 and max(L + A for _, A, L, *_ in rows) == 160
    assert min(r[4] for r in rows) == 1 and max(r[4] for r in rows) == 160
    assert max(len(torch.arange(*r[5])) for r in rows) == 608
    assert any(r[5][2] != 1.0 for r in rows) and {r[3] for r in rows} == {True, False}
    assert any(L % 32 for _, _, L, *_ in rows) and any(L < 32 for _, _, L, *_ in rows)
    # the dense layers read obs, latent or head-hidden inputs: between them every length of the 8-wide loop's tail
    assert {n % 8 for r in rows for n in (r[0], r[2], r[4])} == set(range(8))


def test_first_configs_outside_the_envelope_are_outside():
    """the configs test_gpu_mlp_fp32.py's refusal test sends elsewhere: one step past each edge"""
    assert not fp32_fits(4, 2, 129, 32) and not fp32_fits(161, 2, 128, 32)
    assert not fp32_fits(4, 33, 128, 32) and not fp32_fits(4, 2, 128, 161) and not fp32_fits(4, 2, 7, 32)
    assert support_size((-304., 305., 1.)) == 609
