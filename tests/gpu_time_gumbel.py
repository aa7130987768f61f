"""Simulations per second of the fused Gumbel MuZero and MuZero searches on the same 64x64 MuZeroModel (the shipped Atari
Gumbel config: A = 18, max_num_considered_actions = 18), 1024 roots x 50 simulations, timed with CUDA events over repeated
launches after warm-up.  Both timed windows hold the same host work: Roots.prepare (reset + prepare of the already
materialised roots) and search (a fresh reset + prepare of the roots, then one graph launch).  Prints the card name and
power limit with the numbers.  Writes nothing.
usage: python tests/gpu_time_gumbel.py [--roots 1024] [--sims 50] [--reps 10]"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--roots", type=int, default=1024)
    ap.add_argument("--sims", type=int, default=50)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    import lightzero_b200 as lzb
    from lightzero_b200.synthetic_weights import synthetic_state_dict
    B, S, A = a.roots, a.sims, 18
    obs = (4, 64, 64)
    model = lzb.MuZeroModel(observation_shape=obs, action_space_size=A, downsample=True).load_state_dict(
        synthetic_state_dict(observation_shape=obs, action_space_size=A))
    out = model.initial_inference(torch.rand((B,) + obs, generator=torch.Generator().manual_seed(0)).cuda(), return_scalar_value=True)
    legal = [list(range(A)) for _ in range(B)]
    noises = np.random.default_rng(0).dirichlet([0.3] * A, B).astype(np.float32)
    res = {}
    for name, mcts in (("gumbel", lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=S, max_num_considered_actions=A))),
                       ("muzero", lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True)))):
        roots = mcts.roots(B, legal)

        def once():
            if name == "gumbel":
                roots.prepare(0.25, noises, [0.0] * B, out.value_scalar, out.policy_logits, [-1] * B)
            else:
                roots.prepare(0.25, noises, [0.0] * B, out.policy_logits, [-1] * B)
            mcts.search(roots, model, out.latent_state, [-1] * B)
        for _ in range(3):
            once()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ms = []
        for _ in range(a.reps):
            e0.record()
            once()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        med = float(np.median(ms))
        res[name] = (med, B * S / (med / 1e3), mcts.last_num_kernels)
        roots.clear()
    print(f"card: {_card()}")
    for name, (med, sps, nk) in res.items():
        print(f"{name}: {B} roots x {S} simulations, median {med:.3f} ms per search (incl. prepare), {sps / 1e6:.3f} M simulations/s, "
              f"{nk} kernels in the graph")


if __name__ == "__main__":
    main()
