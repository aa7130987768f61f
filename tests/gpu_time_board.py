"""Median search time of the board-game configs (downsample=False) on the GPU, against the reference pipeline on the same GPU.

Per config (S from the reference's board configs: tictactoe 25, gomoku and connect4 50) and batch size (8 and 32: what a
board collector sends; 1024: a reanalyze batch):
  - this library: `MuZeroMCTSCtree.search` on the board model (prepare + one search graph), CUDA events;
  - the reference pipeline: the compiled, unmodified reference ctree (oracle/_ref/mz_tree) driven by the reference's
    per-simulation host loop (oracle/search_ref.py, including its discarded duplicate recurrent_inference) with the PyTorch
    restatement of the network in eager mode on the same GPU; host clock around work that ends in a device synchronise.
Prints one line per (config, B) with the card's name and power limit.  Sets no threshold.
    python tests/gpu_time_board.py [--reps N] [--ref-reps N]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import board_model_ref as BR  # noqa: E402

CONFIGS = (("tictactoe", 25), ("gomoku", 50), ("connect4", 50))
BATCHES = (8, 32, 1024)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name()


class EagerGPU:
    """the restatement on the GPU behind the reference loop's CPU-tensor interface"""

    def __init__(self, ref):
        self.ref = ref

    def eval(self):
        return self

    def recurrent_inference(self, latent, action):
        o = self.ref.recurrent_inference(latent.cuda(), action.cuda())
        o.latent_state, o.reward, o.value, o.policy_logits = (t.cpu() for t in (o.latent_state, o.reward, o.value, o.policy_logits))
        return o


def median(xs):
    return float(np.median(np.asarray(xs)))


def main():
    import lightzero_b200 as lzb
    from oracle.search_ref import SearchRef, load_tree_module
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--ref-reps", type=int, default=3)
    args = ap.parse_args()
    tree_mod, tree_kind = load_tree_module(prefer_ref=True)
    gpu = card()
    print(f"card: {gpu}; reference tree: {tree_kind}")
    for name, S in CONFIGS:
        ref = BR.build(name, 0)
        cu = lzb.MuZeroModel(**BR.model_kwargs(name)).load_state_dict(ref.state_dict())
        ref_gpu = EagerGPU(ref.cuda().eval())
        obs_shape, A = BR.BOARD_CONFIGS[name][0], BR.BOARD_CONFIGS[name][1]
        sup = BR.BOARD_CONFIGS[name][6]
        for B in BATCHES:
            rng = np.random.default_rng(B)
            obs = torch.rand((B,) + tuple(obs_shape), generator=torch.Generator().manual_seed(B)).cuda()
            legal = [list(range(A))] * B
            noises = [rng.dirichlet([0.3] * A).astype(np.float32).tolist() for _ in range(B)]
            tp = [1 + b % 2 for b in range(B)]
            out = cu.initial_inference(obs)
            mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=1.0))
            ms = []
            for it in range(args.reps + 2):
                roots = mcts.roots(B, legal)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                roots.prepare(0.25, noises, [0.] * B, out.policy_logits, tp)
                mcts.search(roots, cu, out.latent_state, tp)
                b.record()
                torch.cuda.synchronize()
                if it >= 2:
                    ms.append(a.elapsed_time(b))
                roots.clear()
            search = SearchRef(tree_mod, num_simulations=S, discount_factor=1.0, env_type="board_games",
                               value_support_range=sup, reward_support_range=sup, duplicate_inference=True)
            with torch.no_grad():
                r0 = ref_gpu.ref.initial_inference(obs)
            lat = r0.latent_state.cpu().numpy()
            logits = r0.policy_logits.cpu().numpy().tolist()
            ref_ms = []
            for _ in range(args.ref_reps):
                roots = search.roots(B, legal, action_space_size=A)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                roots.prepare(0.25, noises, [0.] * B, logits, tp)
                search.search(roots, ref_gpu, lat, tp)
                torch.cuda.synchronize()
                ref_ms.append((time.perf_counter() - t0) * 1e3)
            m, rm = median(ms), median(ref_ms)
            print(f"{name:9s} B={B:5d} S={S}: search {m:9.3f} ms (median of {len(ms)}) | reference pipeline {rm:10.1f} ms "
                  f"(median of {len(ref_ms)}) | ratio {rm / m:8.1f}x | {gpu}")


if __name__ == "__main__":
    main()
