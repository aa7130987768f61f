"""Simulations per second of the fused Stochastic MuZero search (StochasticMuZeroMCTSCtree.search with a
StochasticMuZeroModelMLP, one CUDA graph per search) at the shipped configs: cartpole (obs 4, A 2, chance 3, latent 128) at
B = 1024, S = 25 and lunarlander_disc (obs 8, A 4, chance 2, latent 256, residual dynamics) at B = 1024, S = 50.  Prints the
GPU's name and power limit with the numbers, as JSON.  Run on the GPU:  python tests/gpu_time_stochastic.py"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import stoch_mlp_model_ref as SR  # noqa: E402


def time_search(name, B, S, reps=20):
    import lightzero_b200 as lzb
    ref = SR.build(name, 0)
    cu = lzb.StochasticMuZeroModelMLP(**SR.model_kwargs(name)).load_state_dict(ref.state_dict())
    obs_dim, A, C = SR.CONFIGS[name][:3]
    rng = np.random.default_rng(0)
    o = cu.initial_inference(torch.from_numpy(rng.uniform(-1, 1, (B, obs_dim)).astype(np.float32)).cuda())
    legal = [list(range(A))] * B
    noises = torch.from_numpy(rng.dirichlet([0.3] * A, B).astype(np.float32)).cuda()
    mcts = lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=S, chance_seed=None))
    roots = mcts.roots(B, legal, C)

    def one():
        roots.prepare(0.25, noises, None, o.policy_logits, [-1] * B)
        mcts.search(roots, cu, o.latent_state, [-1] * B)
    for _ in range(3):
        one()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        one()
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / reps
    return dict(config=name, B=B, S=S, ms_per_search=round(ms, 3), simulations_per_s=round(B * S / (ms * 1e-3)),
                graph_kernels=mcts.last_num_kernels)


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rows = [time_search("cartpole", 1024, 25), time_search("lunarlander_disc", 1024, 50)]
    print(json.dumps(dict(gpu=gpu, results=rows)))


if __name__ == "__main__":
    main()
