"""Writes tests/golden/gumbel_*.npz from the compiled reference Gumbel MuZero tree (oracle/build_gmz_ref.py).

Each fixture holds the inputs of one search driven by synthetic network outputs (root logits / values / noise, legal
lists, and per simulation the reward, value and policy logits fed to the back-up; values quantised so that scores tie
exactly) and what the reference returned: per simulation the leaf choice (ix, iy, last action, search length, virtual
to_play), and at the end visit counts, root values, trajectories, get_policies and get_children_values.  `replay` drives
any module with the gmz_tree API (the compiled reference or lightzero_b200.gmz_tree) through the same loop.

usage: python tests/golden/make_gumbel_golden.py   (needs oracle/_ref/gmz_tree*.so, built by __graft_entry__.build())
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

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


def replay(mod, d):
    """The reference search loop (mcts_ctree.py:1104-1172) on module `mod` with the fixture's inputs."""
    B, A, S, m, tp = int(d["B"]), int(d["A"]), int(d["S"]), int(d["m"]), int(d["to_play"])
    disc = float(d["discount"])
    legal = [d["legal"][b, :d["nlegal"][b]].tolist() for b in range(B)]
    roots = mod.Roots(B, legal)
    if int(d["noise"]):
        noises = [d["noises"][b, :d["nlegal"][b]].tolist() for b in range(B)]
        roots.prepare(0.25, noises, [0.0] * B, d["root_values"].tolist(), d["root_logits"].tolist(), [tp] * B)
    else:
        roots.prepare_no_noise([0.0] * B, d["root_values"].tolist(), d["root_logits"].tolist(), [tp] * B)
    mm = mod.MinMaxStatsList(B)
    mm.set_delta(0.01)
    rec = np.zeros((5, S, B), np.int32)
    for sim in range(S):
        res = mod.ResultsWrapper(B)
        ix, iy, la, vtp = mod.batch_traverse(roots, S, m, disc, res, [tp] * B)
        rec[:, sim] = [ix, iy, la, res.get_search_len(), vtp]
        mod.batch_back_propagate(sim + 1, disc, d["rewards"][sim].tolist(), d["values"][sim].tolist(),
                                 d["logits"][sim].tolist(), mm, res, list(vtp))
    dist = np.full((B, A), -1, np.int32)
    for b, v in enumerate(roots.get_distributions()):
        dist[b, :len(v)] = v
    traj = np.full((B, S + 1), -1, np.int32)
    for b, v in enumerate(roots.get_trajectories()):
        traj[b, :len(v)] = v
    out = dict(rec=rec, dist=dist, root_value=np.asarray(roots.get_values(), np.float32), traj=traj,
               policy=np.asarray(roots.get_policies(disc, A), np.float32),
               children_values=np.asarray(roots.get_children_values(disc, A), np.float32))
    if hasattr(roots, "clear") and mod.__name__.startswith("lightzero_b200"):
        roots.clear()
    return out


EXPECTED = ("rec", "dist", "root_value", "traj", "policy", "children_values")


def main():
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle import build_gmz_ref
    ref = build_gmz_ref.load()
    if ref is None:
        raise SystemExit("oracle/_ref/gmz_tree*.so is missing: run __graft_entry__.build() with the reference sources present")
    for name, case in CASES.items():
        d = make_inputs(*case)
        out = replay(ref, d)
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **d, **{"exp_" + k: v for k, v in out.items()})
        print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
