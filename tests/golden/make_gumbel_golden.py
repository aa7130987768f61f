"""Writes tests/golden/gumbel_*.npz from the compiled reference Gumbel MuZero tree (oracle/build_gmz_ref.py).

Each fixture holds the inputs of one search driven by synthetic network outputs (root logits / values / noise, legal
lists, and per simulation the reward, value and policy logits fed to the back-up; values quantised so that scores tie
exactly) and what the reference returned: per simulation the leaf choice (ix, iy, last action, search length, virtual
to_play), and at the end visit counts, root values, trajectories, get_policies and get_children_values.  A fixture is a
tree_drive case: tree_drive.check_fixture replays it through any module with the gmz_tree API (the compiled reference
or lightzero_b200.gmz_tree).

usage: python tests/golden/make_gumbel_golden.py   (needs oracle/_ref/gmz_tree*.so, built by __graft_entry__.build())
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle.tree_drive import PER_SIM, drive, recorded  # noqa: E402

# name -> (B, A, S, m, legal kind, noise, to_play, seed)
CASES = {
    "gumbel_masked_a6": (7, 6, 16, 4, "mixed", True, -1, 1),
    "gumbel_single_a18": (5, 18, 16, 18, "single", False, -1, 2),
    "gumbel_m1_a6": (7, 6, 16, 1, "mixed", True, -1, 3),
    "gumbel_atari_a18_2p": (4, 18, 50, 18, "mixed", True, 1, 4),
}


def _q(rng, shape, step):
    return (np.round(rng.normal(size=shape) / step) * step).astype(np.float32)


def make_inputs(B, A, S, m, kind, noise, to_play, seed):
    rng = np.random.default_rng(seed)
    legal = np.full((B, A), -1, np.int32)
    nlegal = np.zeros(B, np.int32)
    for b in range(B):
        if kind == "single" or b % 3 == 0:
            l = [int(rng.integers(A))]
        else:
            l = sorted(rng.choice(A, int(rng.integers(1, A + 1)), replace=False).tolist())
        legal[b, :len(l)] = l
        nlegal[b] = len(l)
    noises = np.zeros((B, A), np.float32)
    for b in range(B):
        noises[b, :nlegal[b]] = rng.dirichlet([0.3] * int(nlegal[b]))
    return dict(B=B, A=A, S=S, m=m, noise=int(noise), to_play=to_play, discount=np.float32(0.997),
                legal=legal, nlegal=nlegal, noises=noises, root_logits=_q(rng, (B, A), 0.5), root_values=_q(rng, (B,), 0.25),
                rewards=_q(rng, (S, B), 0.5), values=_q(rng, (S, B), 0.25), logits=_q(rng, (S, B, A), 1.0))


def expected(trace):
    """A tree_drive.drive trace under the fixtures' exp_* names (tree_drive.fixture_trace reads them back)."""
    return dict(exp_rec=np.stack([trace[k] for k in PER_SIM[:5]]), exp_dist=trace["distributions"],
                exp_root_value=trace["root_values_bits"].view(np.float32), exp_traj=trace["trajectories"],
                exp_policy=trace["policies"], exp_children_values=trace["children_values"])


def make_case(ref, *case):
    d = make_inputs(*case)
    trace, _ = drive(ref, d, "gumbel", recorded(d, "gumbel"))
    return dict(d, **expected(trace))


def main():
    from oracle import build_gmz_ref
    ref = build_gmz_ref.load()
    if ref is None:
        raise SystemExit("oracle/_ref/gmz_tree*.so is missing: run __graft_entry__.build() with the reference sources present")
    for name, case in CASES.items():
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **make_case(ref, *case))
        print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
