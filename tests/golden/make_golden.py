"""Generate the committed golden fixtures for the MuZero and EfficientZero ctree paths by RUNNING THE COMPILED,
UNMODIFIED REFERENCE (oracle/_ref/mz_tree and ez_tree, built from /root/reference by oracle/build_ref.py; ez_tree
is linked with oracle/rand_shim.c so that its rand()-based tie-break is reproducible).

Run in the build container (the GPU box has no /root/reference; it uses the committed .npz files):
    python tests/golden/make_golden.py

Each fixture is a replay-mode trace: all inputs the tree consumes (legal lists, root logits,
Dirichlet noise, per-simulation reward / value / policy-logit batches) and everything it produces
(per-simulation (ix, iy, last_action, search_len, virtual_to_play), final visit distributions,
root values as raw fp32 bits, best-action trajectories).  deterministic=True (SURVEY.md s.0 fact 2).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
from oracle.tree_drive import _pad, drive, random_case  # noqa: E402

CASES = [
    # name,            B,  A,  S,  masks, noise, two_player, scale, seed
    ("survey_b4a6",     4,  6, 10, 0, 0, 0, 1.0, 0),   # SURVEY.md 8c session vector (same draws)
    ("atari_a6",       32,  6, 50, 0, 1, 0, 1.0, 1),
    ("atari_a18",      32, 18, 50, 0, 1, 0, 1.0, 2),
    ("atari_a18_mask", 32, 18, 50, 1, 1, 0, 2.0, 3),
    ("deep_s200",       8, 18, 200, 0, 1, 0, 0.5, 4),
    ("board_2p_a9",    16,  9, 40, 1, 1, 1, 1.0, 5),
    ("wide_a40",        6, 40, 60, 1, 0, 0, 3.0, 6),
    ("cartpole_a2",     8,  2, 25, 0, 1, 0, 1.0, 7),
]
PB_C_BASE, PB_C_INIT, DISCOUNT, DELTA, NOISE_W = 19652, 1.25, 0.997, 0.01, 0.25


def make_case(mod, B, A, S, masks, noise, two_player, scale, seed, horizon=0, reuse=False):
    """One fixture: the reference driver loop (oracle/tree_drive.py) on `mod` with random_case's seeded inputs and
    network outputs, the inputs and the trace it returned."""
    c, leaves = random_case(B, A, S, seed, masks, noise, two_player, scale, reuse=reuse, horizon=horizon)
    kind = ("ez_reuse" if horizon else "reuse") if reuse else ("ez" if horizon else "mz")
    t, _ = drive(mod, c, kind, leaves)
    legal = [np.asarray(l, np.int32) for l in c.pop("legal")]
    c.update(legal=_pad(legal, A), nlegal=np.asarray([len(l) for l in legal], np.int32),
             rewards=np.stack([d[0] for d in leaves.drawn]), values_in=np.stack([d[1] for d in leaves.drawn]),
             policies=np.stack([d[2] for d in leaves.drawn]), pb_c_base=PB_C_BASE, pb_c_init=np.float32(PB_C_INIT),
             discount=np.float32(DISCOUNT), delta=np.float32(DELTA), noise_w=np.float32(NOISE_W), **t)
    if reuse:
        del c["trajectories"]
        c.setdefault("is_reset", np.zeros((S, B), np.int32))
    elif not horizon:
        del c["lstm_horizon_len"]
    return c


EZ_CASES = [
    # name,             B,  A,  S,  masks, noise, two_player, scale, seed, lstm_horizon_len
    ("ez_atari_a6",     32,  6, 50, 0, 1, 0, 1.0, 11, 5),
    ("ez_atari_a18",    32, 18, 50, 1, 1, 0, 2.0, 12, 5),
    ("ez_deep_s120",     8, 18, 120, 0, 1, 0, 0.5, 13, 3),
    ("ez_board_2p_a9",  16,  9, 40, 1, 1, 1, 1.0, 14, 4),
]


REUSE_CASES = [
    # name,               tree,      B,  A,  S, masks, noise, two_player, scale, seed, lstm_horizon_len (EZ only)
    ("reuse_mz_a6",       "mz",     32,  6, 40, 0, 1, 0, 1.0, 21, 0),
    ("reuse_mz_a18_mask", "mz",     24, 18, 40, 1, 1, 0, 2.0, 22, 0),
    ("reuse_mz_2p_a9",    "mz",     16,  9, 30, 1, 1, 1, 1.0, 23, 0),
    ("reuse_ez_a6",       "ez",     32,  6, 40, 0, 1, 0, 1.0, 24, 3),
]


def make_all(mz, ez, mz_rand0):
    """file name -> fixture, for every case above (mz_rand0: the MuZero tree linked with the rand() == 0 shim)"""
    out = {f"tree_{name}": make_case(mz, *args) for name, *args in CASES}
    out.update({f"tree_{name}": make_case(ez, *args) for name, *args in EZ_CASES})
    out.update({name: make_case(mz_rand0 if tree == "mz" else ez, *args, reuse=True) for name, tree, *args in REUSE_CASES})
    return out


def main():
    import ez_tree
    import mz_tree
    from oracle import build_ref
    # the reference's own known-answer test (lzero/mcts/tests/test_muzero_ctree_deterministic.py:4-25)
    roots = mz_tree.Roots(1, [[0, 1, 2]])
    roots.prepare_no_noise([0.], [[0., 0., 0.]], [-1])
    mm = mz_tree.MinMaxStatsList(1); mm.set_delta(0.01)
    acts = []
    for _ in range(5):
        res = mz_tree.ResultsWrapper(1)
        _, _, la, _ = mz_tree.batch_traverse(roots, 19652, 1.25, 0.997, mm, res, [-1], True)
        acts.append(la[0])
    assert acts == [0] * 5, acts
    print("reference KAT ok", acts)
    mods = (mz_tree, ez_tree, build_ref.load_rand0())
    cases, again = make_all(*mods), make_all(*mods)      # the shimmed references must be reproducible
    for name, case in cases.items():
        assert all(np.array_equal(case[k], again[name][k]) for k in case), name
        np.savez_compressed(os.path.join(HERE, f"{name}.npz"), **case)
        print(name, "sum visits ok:", bool((np.where(case["distributions"] < 0, 0, case["distributions"]).sum(1) == case["S"]).all()),
              "resets:", int(case["is_reset"].sum()) if "is_reset" in case else 0, "no-inference marks:", int((case["ix"] == -1).sum()))


if __name__ == "__main__":
    main()
