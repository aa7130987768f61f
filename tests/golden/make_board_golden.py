"""Pin the board-network restatement (tests/board_model_ref.py) to the REFERENCE'S OWN MuZeroModel with downsample=False and
generate tests/golden/board_<name>.npz for every config of tests/board_model_ref.BOARD_CONFIGS: the shipped boards and the
corners (1x8 and 8x1 boards, 1 and 16 planes, 1 and 64 actions, 4 blocks, 1 and 16 head channels, 608 support bins).

Run where the reference sources are (LZ_REFERENCE, default /root/reference):   python tests/golden/make_board_golden.py

Same procedure as make_model_golden.py: the restated model is built under a fixed seed with emulate_trained_ weights, its
state_dict is loaded into the reference class (strict), both run the same seeded inputs and must agree bit for bit; the
reference's outputs are stored with the inputs.  tests/test_board_oracle.py rebuilds the restatement on any machine and checks
it against the stored vectors, and regenerates the vectors from the reference class when the reference is present."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import board_model_ref as BR  # noqa: E402
from make_model_golden import import_reference_models, weights_digest  # noqa: E402

B = 5
CASES = [(name, seed) for seed, name in enumerate(BR.BOARD_CONFIGS)]


def case_outputs(mz_mod, name, seed):
    """the fixture arrays of one case: inputs and the reference class's outputs (asserting the restatement equals them)"""
    mine = BR.build(name, seed)
    theirs = mz_mod.MuZeroModel(**BR.model_kwargs(name), downsample=False)
    theirs.load_state_dict(mine.state_dict(), strict=True)
    theirs.eval()
    obs_shape, A = BR.BOARD_CONFIGS[name][0], BR.BOARD_CONFIGS[name][1]
    g = torch.Generator().manual_seed(2000 + seed)
    obs = torch.rand((B,) + tuple(obs_shape), generator=g)
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
    mz_mod = import_reference_models()[0]
    for name, seed in CASES:
        np.savez_compressed(os.path.join(HERE, f"board_{name}.npz"), **case_outputs(mz_mod, name, seed))
        print(name, "restatement == reference class bit for bit; fixture written")


if __name__ == "__main__":
    main()
