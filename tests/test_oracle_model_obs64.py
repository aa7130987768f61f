"""Pins the 64x64 restatement (oracle/model_ref.py, 8x8 latent, no pooling2) to the vectors the reference's own model
classes produced (tests/golden/obs64_*.npz, written by tests/golden/make_obs64_golden.py after asserting bit-equality with the
restatement).  CPU only: rebuild the restatement under the fixture's seed, check the weights are the same bytes, re-run
the stored inputs."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, ROOT

sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_model_golden import build_restated, weights_digest  # noqa: E402
from make_obs64_golden import CASES as GEN_CASES  # noqa: E402

CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "obs64_*.npz")))
TOL = 2e-6


@pytest.mark.parametrize("name", CASES)
def test_restatement_reproduces_reference_vectors_64px(name):
    d = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    kind, obs_shape = str(d["kind"]), tuple(int(x) for x in d["obs_shape"])
    assert obs_shape[1:] == (64, 64)
    model = build_restated(kind, obs_shape, int(d["A"]), int(d["nres"]), int(d["seed"]))
    if weights_digest(model) != str(d["weights_sha256"]):
        pytest.skip("this torch build initialises parameters differently from the one that wrote the fixture")
    obs, action = torch.from_numpy(d["obs"]), torch.from_numpy(d["action"])
    with torch.no_grad():
        o0 = model.initial_inference(obs)
        assert o0.latent_state.shape[1:] == (64, 8, 8)
        for f in ("value", "policy_logits", "latent_state"):
            assert np.allclose(getattr(o0, f).numpy(), d["init_" + f], rtol=0, atol=TOL), f
        latent = torch.from_numpy(d["init_latent_state"])
        if kind == "efficientzero":
            hc = (torch.from_numpy(d["in_hidden0"]), torch.from_numpy(d["in_hidden1"]))
            o1 = model.recurrent_inference(latent, hc, action)
            fields = ("value", "value_prefix", "policy_logits", "latent_state")
            for i in range(2):
                assert np.allclose(o1.reward_hidden_state[i].numpy(), d[f"rec_hidden{i}"], rtol=0, atol=TOL)
        else:
            o1 = model.recurrent_inference(latent, action)
            fields = ("value", "reward", "policy_logits", "latent_state")
        for f in fields:
            assert np.allclose(getattr(o1, f).numpy(), d["rec_" + f], rtol=0, atol=TOL), f


def test_fixture_set_is_complete_64px():
    assert CASES == sorted(c[0] for c in GEN_CASES)
    kinds = {str(np.load(os.path.join(GOLDEN_DIR, n + ".npz"))["kind"]) for n in CASES}
    assert kinds == {"muzero", "efficientzero"}
