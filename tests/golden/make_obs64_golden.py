"""The 64x64-observation model fixtures tests/golden/obs64_*.npz (8x8 latent, no pooling2: the shipped Atari configs,
zoo/atari/config/atari_{muzero,efficientzero}_config.py).  Same procedure as make_model_golden.py, whose run_case this
uses: the restatement is built under a fixed seed, its state_dict is loaded into the REFERENCE'S OWN model class, both run
the same seeded inputs and must agree bit for bit, and the reference's outputs are stored.  Unlike 84x84, the reference
classes can be built at 64x64, so these fixtures pin the 8x8 path to them directly.

Run with the reference sources at $LZ_REFERENCE:   python tests/golden/make_obs64_golden.py [fixture names]
(savez_compressed does not rewrite a fixture byte for byte: name the ones to write when adding a case)
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_model_golden import import_reference_models, run_case  # noqa: E402

CASES = [
    # name,                  kind,            obs,          A,  res blocks, B, seed
    ("obs64_muzero_a6",      "muzero",        (4, 64, 64),   6, 1, 4, 6),
    ("obs64_ez_a6",          "efficientzero", (4, 64, 64),   6, 1, 3, 7),
    ("obs64_muzero_a18_r2",  "muzero",        (4, 64, 64),  18, 2, 3, 8),
]


def main(names=()):
    mods = import_reference_models()
    for case in CASES:
        if not names or case[0] in names:
            run_case(mods, *case)


if __name__ == "__main__":
    main(sys.argv[1:])
