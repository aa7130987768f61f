"""CPU checks of the board Stochastic MuZero network (StochasticMuZeroModel, downsample=False): the PyTorch restatement
(tests/stoch_board_model_ref.py) against the fixtures of the reference class, and the fixtures regenerated from the reference
class when its sources are present."""
import os
import sys

import numpy as np
import pytest
import torch

import stoch_board_model_ref as SB
from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden")
if GOLDEN not in sys.path:
    sys.path.insert(0, GOLDEN)      # the fixture generators
REF = os.environ.get("LZ_REFERENCE", "/root/reference")
NAMES = list(SB.CONFIGS)


@pytest.mark.parametrize("name", NAMES)
def test_restatement_reproduces_the_fixture(name):
    from make_model_golden import weights_digest
    d = np.load(os.path.join(GOLDEN, f"stoch_board_{name}.npz"))
    mine = SB.build(name, int(d["seed"]))
    assert weights_digest(mine) == str(d["weights_sha256"])
    obs, action, chance = (torch.from_numpy(d[k]) for k in ("obs", "action", "chance"))
    with torch.no_grad():
        o0 = mine.initial_inference(obs)
        o1 = mine.recurrent_inference(o0.latent_state, action, False)
        o2 = mine.recurrent_inference(o1.latent_state, chance, True)
    for f in ("value", "policy_logits", "latent_state"):
        assert torch.equal(getattr(o0, f), torch.from_numpy(d["init_" + f])), f
    for prefix, o in (("after_", o1), ("rec_", o2)):
        for f in ("value", "reward", "policy_logits", "latent_state"):
            assert torch.equal(getattr(o, f), torch.from_numpy(d[prefix + f])), prefix + f
    for f in ("init_value", "init_policy_logits", "after_reward", "after_value", "after_policy_logits", "rec_reward",
              "rec_value", "rec_policy_logits"):
        x = d[f]
        assert (x != x[:1]).any(), f        # every head depends on its root: none is a dead ReLU that outputs its bias


@pytest.mark.parametrize("name", NAMES)
def test_fixture_regenerates_from_the_reference_class(name):
    if not os.path.isdir(os.path.join(REF, "lzero", "model")):
        pytest.skip("reference sources not present")
    import make_stochastic_board_golden as G
    d = np.load(os.path.join(GOLDEN, f"stoch_board_{name}.npz"))
    out = G.case_outputs(G.reference_module(), name, int(d["seed"]))
    assert sorted(out) == sorted(d.files)
    for k in d.files:
        assert np.array_equal(np.asarray(out[k]), d[k]) and np.asarray(out[k]).dtype == d[k].dtype, k
