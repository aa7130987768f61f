"""Generate the committed Stochastic MuZero tree fixtures tests/golden/tree_stoch_*.npz by RUNNING THE COMPILED, UNMODIFIED
REFERENCE tree (oracle/_ref/stochastic_mz_tree, built by oracle/build_stoch_ref.py and linked with the rand() and
std::random_device shims, so that its decision ties take the first maximum and every chance draw is std::mt19937(chance_seed)'s).

Run where the reference sources are:
    python -m oracle.build_stoch_ref && python tests/golden/make_stoch_tree_golden.py

Each fixture is a replay-mode trace of the reference loop (oracle/tree_drive.py, kind "stoch") on seeded random inputs and
network outputs: legal lists, root logits, noise, chance_seed, the per-simulation reward / value / policy-logit batches
(max(A, C) wide; a chance leaf reads the first C logits, a decision leaf the first A) and everything the tree produces:
per simulation (is_chance, ix, iy, last_action, search_len, virtual_to_play), the visit distributions, the root values as
fp32 bits and the trajectories.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.tree_drive import _pad, drive, random_case  # noqa: E402

CASES = [
    # name,                    B,  A,  C,  S,  masks, noise, two_player, scale, seed, chance_seed
    ("tree_stoch_c3_a2",      16,  2,  3, 40, 0, 1, 0, 1.0, 31, 7),      # C > A (cartpole's shape)
    ("tree_stoch_a9_c4_mask", 12,  9,  4, 50, 1, 1, 0, 2.0, 32, 1234),   # A > C, masked roots
    ("tree_stoch_2p_a6_c3",   10,  6,  3, 40, 1, 0, 1, 1.0, 33, 99),     # two players
    ("tree_stoch_c1_a4",       8,  4,  1, 60, 0, 1, 0, 0.5, 34, 5),      # C = 1: every chance node has one outcome
    ("tree_stoch_c40_a3",      6,  3, 40, 50, 1, 1, 0, 3.0, 35, 2024),   # C = 40, A = 3
]
PB_C_BASE, PB_C_INIT, DISCOUNT, DELTA, NOISE_W = 19652, 1.25, 0.997, 0.01, 0.25


def make_case(mod, B, A, C, S, masks, noise, two_player, scale, seed, chance_seed):
    """One fixture: the reference loop on `mod` with random_case's seeded inputs and network outputs, the inputs and the
    trace it returned"""
    c, leaves = random_case(B, A, S, seed, masks, noise, two_player, scale, C=C, chance_seed=chance_seed)
    t, _ = drive(mod, c, "stoch", leaves)
    legal = [np.asarray(l, np.int32) for l in c.pop("legal")]
    del c["lstm_horizon_len"]
    c.update(legal=_pad(legal, A), nlegal=np.asarray([len(l) for l in legal], np.int32),
             rewards=np.stack([d[0] for d in leaves.drawn]), values_in=np.stack([d[1] for d in leaves.drawn]),
             policies=np.stack([d[2] for d in leaves.drawn]), pb_c_base=PB_C_BASE, pb_c_init=np.float32(PB_C_INIT),
             discount=np.float32(DISCOUNT), delta=np.float32(DELTA), noise_w=np.float32(NOISE_W),
             chance_seed=np.int64(chance_seed), **t)
    return c


def make_all(mod):
    return {name: make_case(mod, *args) for name, *args in CASES}


def main():
    from oracle import build_stoch_ref
    mod = build_stoch_ref.load()
    if mod is None:
        raise SystemExit("oracle/_ref/stochastic_mz_tree is not built: python -m oracle.build_stoch_ref")
    cases, again = make_all(mod), make_all(mod)      # the shimmed reference must be reproducible
    for name, case in cases.items():
        assert all(np.array_equal(case[k], again[name][k]) for k in case), name
        np.savez_compressed(os.path.join(HERE, f"{name}.npz"), **case)
        print(name, "chance leaves:", int(case["is_chance"].sum()), "max search_len:", int(case["search_len"].max()),
              "distinct outcomes:", len(set(case["last_action"][case["is_chance"] == 0].tolist())))


if __name__ == "__main__":
    main()
