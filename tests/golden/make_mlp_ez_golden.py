"""Pin the EfficientZeroModelMLP restatement (tests/mlp_ez_model_ref.py) to the REFERENCE'S OWN EfficientZeroModelMLP and generate
tests/golden/mlp_ez_<name>.npz for every config of tests/mlp_ez_model_ref.CONFIGS.

Run where the reference sources are (LZ_REFERENCE, default /root/reference):   python tests/golden/make_mlp_ez_golden.py

Same procedure as make_model_golden.py: the restated model is built under a fixed seed, its state_dict is loaded into the
reference class (strict; the reference's SSL heads are switched off so that both have the same keys), both run the same seeded
inputs -- with a non-zero LSTM state -- and must agree bit for bit; the reference's outputs are stored with the inputs."""
import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import mlp_ez_model_ref as MR  # noqa: E402
from make_model_golden import import_reference_models, weights_digest  # noqa: E402

B = 5
CASES = [(name, seed) for seed, name in enumerate(MR.CONFIGS)]


def reference_module():
    import_reference_models()
    return importlib.import_module("lzero.model.efficientzero_model_mlp")


def case_outputs(mod, name, seed):
    """the fixture arrays of one case: inputs and the reference class's outputs (asserting the restatement equals them)"""
    mine = MR.build(name, seed)
    theirs = mod.EfficientZeroModelMLP(**MR.model_kwargs(name), self_supervised_learning_loss=False)
    theirs.load_state_dict(mine.state_dict(), strict=True)
    theirs.eval()
    obs_dim, A, L, H, _ = MR.CONFIGS[name]
    g = torch.Generator().manual_seed(3000 + seed)
    obs = torch.rand((B, obs_dim), generator=g) * 2.0 - 1.0
    action = torch.randint(0, A, (B,), generator=g)
    h0 = (torch.rand((1, B, H), generator=g) * 2.0 - 1.0) * 0.5
    c0 = torch.randn((1, B, H), generator=g)
    out = {}
    with torch.no_grad():
        a0, b0 = theirs.initial_inference(obs), mine.initial_inference(obs)
        for f in ("value", "policy_logits", "latent_state"):
            assert torch.equal(getattr(a0, f), getattr(b0, f)), (name, "initial", f)
            out["init_" + f] = getattr(a0, f).numpy()
        latent = a0.latent_state * 1.0
        a1, b1 = theirs.recurrent_inference(latent, (h0, c0), action), mine.recurrent_inference(latent, (h0, c0), action)
        for f in ("value", "value_prefix", "policy_logits", "latent_state"):
            assert torch.equal(getattr(a1, f), getattr(b1, f)), (name, "recurrent", f)
            out["rec_" + f] = getattr(a1, f).numpy()
        for i, f in enumerate(("h", "c")):
            assert torch.equal(a1.reward_hidden_state[i], b1.reward_hidden_state[i]), (name, "recurrent", f)
            out["rec_" + f] = a1.reward_hidden_state[i].numpy()
    out.update(obs=obs.numpy(), action=action.numpy().astype(np.int64), h0=h0.numpy(), c0=c0.numpy(), seed=seed,
               weights_sha256=weights_digest(mine))
    return out


def main():
    mod = reference_module()
    for name, seed in CASES:
        np.savez_compressed(os.path.join(HERE, f"mlp_ez_{name}.npz"), **case_outputs(mod, name, seed))
        print(name, "restatement == reference class bit for bit; fixture written")


if __name__ == "__main__":
    main()
