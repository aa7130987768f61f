"""Pin the MuZeroModelMLP restatement (oracle.model_ref.MuZeroModelMLPRef, configs of tests/mlp_mz_model_ref.py) to the
REFERENCE'S OWN MuZeroModelMLP and generate tests/golden/mlp_mz_<name>.npz for every config of tests/mlp_mz_model_ref.CONFIGS:
the configs that run on the tensor-core MLP kernel.

Run where the reference sources are (LZ_REFERENCE, default /root/reference):   python tests/golden/make_mlp_mz_golden.py

Same procedure as make_mlp_ez_golden.py: the restated model is built under a fixed seed, its state_dict is loaded into the
reference class (strict), both run the same seeded inputs and must agree bit for bit; the reference's outputs are stored with
the inputs."""
import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import mlp_mz_model_ref as MR  # noqa: E402
from make_model_golden import import_reference_models, weights_digest  # noqa: E402

B = 5
CASES = [(name, seed) for seed, name in enumerate(MR.CONFIGS)]


def reference_module():
    import_reference_models()
    return importlib.import_module("lzero.model.muzero_model_mlp")


def case_outputs(mod, name, seed):
    """the fixture arrays of one case: inputs and the reference class's outputs (asserting the restatement equals them)"""
    mine = MR.build(name, seed)
    theirs = mod.MuZeroModelMLP(**MR.model_kwargs(name), self_supervised_learning_loss=False)
    theirs.load_state_dict(mine.state_dict(), strict=True)
    theirs.eval()
    obs_dim, A = MR.CONFIGS[name][:2]
    g = torch.Generator().manual_seed(4000 + seed)
    obs = torch.rand((B, obs_dim), generator=g) * 2.0 - 1.0
    action = torch.randint(0, A, (B,), generator=g)
    out = {}
    with torch.no_grad():
        a0, b0 = theirs.initial_inference(obs), mine.initial_inference(obs)
        for f in ("value", "policy_logits", "latent_state"):
            assert torch.equal(getattr(a0, f), getattr(b0, f)), (name, "initial", f)
            out["init_" + f] = getattr(a0, f).numpy()
        latent = a0.latent_state * 1.0
        a1, b1 = theirs.recurrent_inference(latent, action), mine.recurrent_inference(latent, action)
        for f in ("value", "reward", "policy_logits", "latent_state"):
            assert torch.equal(getattr(a1, f), getattr(b1, f)), (name, "recurrent", f)
            out["rec_" + f] = getattr(a1, f).numpy()
    out.update(obs=obs.numpy(), action=action.numpy().astype(np.int64), seed=seed, weights_sha256=weights_digest(mine))
    return out


def main():
    mod = reference_module()
    for name, seed in CASES:
        np.savez_compressed(os.path.join(HERE, f"mlp_mz_{name}.npz"), **case_outputs(mod, name, seed))
        print(name, "restatement == reference class bit for bit; fixture written")


if __name__ == "__main__":
    main()
