"""Pin the board Stochastic MuZero restatement (tests/stoch_board_model_ref.py) to the REFERENCE'S OWN StochasticMuZeroModel
(downsample=False) and generate tests/golden/stoch_board_<name>.npz for every config of stoch_board_model_ref.CONFIGS: the
shipped 2048 network and the corners (C 16 / 32 / 64, 3x3, 6x7 and 8x8 boards, 1 to 64 chance outcomes, 4 blocks, head
channels 1 and 16).

Run where the reference sources are (LZ_REFERENCE, default /root/reference):   python tests/golden/make_stochastic_board_golden.py

Same procedure as make_stochastic_mlp_golden.py: the restated model is built under a fixed seed, its state_dict is loaded
strictly into the reference class (its chance_encoder, used in training only, keeps its own initial weights), both run the same
seeded inputs through initial_inference and both recurrent_inference programs and must agree bit for bit; the reference's
outputs are stored with the inputs."""
import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import stoch_board_model_ref as SB  # noqa: E402
from make_model_golden import import_reference_models, weights_digest  # noqa: E402

B = 5


def reference_module():
    import_reference_models()
    return importlib.import_module("lzero.model.stochastic_muzero_model")


def case_outputs(mod, name, seed):
    mine = SB.build(name, seed)
    theirs = mod.StochasticMuZeroModel(**SB.model_kwargs(name), downsample=False, self_supervised_learning_loss=False)
    sd = dict(theirs.state_dict())
    assert set(mine.state_dict()) == {k for k in sd if not k.startswith("chance_encoder.")}, name
    sd.update(mine.state_dict())
    theirs.load_state_dict(sd, strict=True)
    theirs.eval()
    obs_shape, A, C = SB.CONFIGS[name][:3]
    g = torch.Generator().manual_seed(6000 + seed)
    obs = torch.rand((B,) + tuple(obs_shape), generator=g)
    action = torch.randint(0, A, (B,), generator=g)
    chance = torch.randint(0, C, (B,), generator=g)
    out = {}
    with torch.no_grad():
        a0, b0 = theirs.initial_inference(obs), mine.initial_inference(obs)
        for f in ("value", "policy_logits", "latent_state"):
            assert torch.equal(getattr(a0, f), getattr(b0, f)), (name, "initial", f)
            out["init_" + f] = getattr(a0, f).numpy()
        latent = a0.latent_state * 1.0
        a1, b1 = theirs.recurrent_inference(latent, action, afterstate=False), mine.recurrent_inference(latent, action, False)
        for f in ("value", "reward", "policy_logits", "latent_state"):
            assert torch.equal(getattr(a1, f), getattr(b1, f)), (name, "afterstate", f)
            out["after_" + f] = getattr(a1, f).numpy()
        after = a1.latent_state * 1.0
        a2, b2 = theirs.recurrent_inference(after, chance, afterstate=True), mine.recurrent_inference(after, chance, True)
        for f in ("value", "reward", "policy_logits", "latent_state"):
            assert torch.equal(getattr(a2, f), getattr(b2, f)), (name, "dynamics", f)
            out["rec_" + f] = getattr(a2, f).numpy()
    out.update(obs=obs.numpy(), action=action.numpy().astype(np.int64), chance=chance.numpy().astype(np.int64), seed=seed,
               weights_sha256=weights_digest(mine))
    return out


def main():
    mod = reference_module()
    for seed, name in enumerate(SB.CONFIGS):
        np.savez_compressed(os.path.join(HERE, f"stoch_board_{name}.npz"), **case_outputs(mod, name, seed))
        print(name, "restatement == reference class bit for bit; fixture written")


if __name__ == "__main__":
    main()
