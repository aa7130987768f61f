"""Median search time of the vector-observation EfficientZero configs (EfficientZeroModelMLP) on the GPU, against the reference
pipeline on the same GPU.

Per (config, B, S): cartpole B = 8 S = 25 (a collector batch), lunarlander B = 8 / 256 / 1024 S = 50 (collector, larger
collectors, a reanalyze batch):
  - this library: `EfficientZeroMCTSCtree.search` on the model (prepare + one search graph), CUDA events;
  - the reference pipeline: the compiled, unmodified reference ez_tree (oracle/_ref, or the C port where it is not built) driven
    by the reference's per-simulation host loop (oracle/search_ref.py SearchRefEZ) with the PyTorch restatement of the network
    in eager mode on the same GPU; host clock around work that ends in a device synchronise.
Before a config's first search, the time of single initial_inference / recurrent_inference calls at B = 1 .. 1024 (one CTA
holds 64 roots).  Prints one line per case with the card's name and power limit.  Sets no threshold.
    python tests/gpu_time_mlp_ez.py [--reps N] [--ref-reps N]
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import mlp_ez_model_ref as MR  # noqa: E402
from gpu_time_board import card, median  # noqa: E402

CASES = (("cartpole", 8, 25), ("lunarlander", 8, 50), ("lunarlander", 256, 50), ("lunarlander", 1024, 50))


class EagerGPU:
    """the restatement on the GPU behind the reference loop's CPU-tensor interface"""

    def __init__(self, ref):
        self.ref = ref

    def eval(self):
        return self

    def recurrent_inference(self, latent, hidden, action):
        o = self.ref.recurrent_inference(latent.cuda(), tuple(h.cuda() for h in hidden), action.cuda())
        o.latent_state, o.value_prefix, o.value, o.policy_logits = (
            t.cpu() for t in (o.latent_state, o.value_prefix, o.value, o.policy_logits))
        o.reward_hidden_state = tuple(h.cpu() for h in o.reward_hidden_state)
        return o


def call_times(cu, name, reps):
    """median time of one initial_inference / recurrent_inference call (CUDA events) at B = 1, 8, 64, 65, 1024: with 64 roots
    per CTA, B = 1 .. 64 is one CTA and B = 1024 sixteen"""
    obs_dim = MR.CONFIGS[name][0]
    for B in (1, 8, 64, 65, 1024):
        obs = torch.rand(B, obs_dim, device="cuda")
        o = cu.initial_inference(obs)
        act = torch.zeros(B, dtype=torch.int32, device="cuda")
        res = []
        for fn in (lambda: cu.initial_inference(obs), lambda: cu.recurrent_inference(o.latent_state, o.reward_hidden_state, act)):
            ts = []
            for it in range(reps + 3):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                torch.cuda.synchronize()
                if it >= 3:
                    ts.append(a.elapsed_time(b) * 1e3)
            res.append(median(ts))
        print(f"{name:11s} B={B:5d}: initial_inference {res[0]:7.1f} us, recurrent_inference {res[1]:7.1f} us (median of {reps})")


def main():
    import lightzero_b200 as lzb
    from oracle.search_ref import SearchRefEZ, load_tree_module
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--ref-reps", type=int, default=3)
    args = ap.parse_args()
    tree_mod, tree_kind = load_tree_module(prefer_ref=True, name="ez_tree")
    gpu = card()
    print(f"card: {gpu}; reference tree: {tree_kind}")
    for name, B, S in CASES:
        ref = MR.build(name, 0)
        cu = lzb.EfficientZeroModelMLP(**MR.model_kwargs(name)).load_state_dict(ref.state_dict())
        ref_gpu = EagerGPU(ref.cuda().eval())
        obs_dim, A = MR.CONFIGS[name][0], MR.CONFIGS[name][1]
        rng = np.random.default_rng(B)
        obs = (torch.rand((B, obs_dim), generator=torch.Generator().manual_seed(B)) * 2 - 1).cuda()
        legal = [list(range(A))] * B
        noises = [rng.dirichlet([0.3] * A).astype(np.float32).tolist() for _ in range(B)]
        tp = [-1] * B
        out = cu.initial_inference(obs)
        if B == 8:
            call_times(cu, name, args.reps)
        mcts = lzb.EfficientZeroMCTSCtree(dict(num_simulations=S, discount_factor=0.997, lstm_horizon_len=5))
        ms = []
        for it in range(args.reps + 2):
            roots = mcts.roots(B, legal)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            roots.prepare(0.25, noises, [0.] * B, out.policy_logits, tp)
            mcts.search(roots, cu, out.latent_state, out.reward_hidden_state, tp)
            b.record()
            torch.cuda.synchronize()
            if it >= 2:
                ms.append(a.elapsed_time(b))
            roots.clear()
        search = SearchRefEZ(tree_mod, num_simulations=S, discount_factor=0.997, lstm_horizon_len=5)
        with torch.no_grad():
            r0 = ref_gpu.ref.initial_inference(obs)
        lat = r0.latent_state.cpu().numpy()
        hid = tuple(h.numpy() for h in r0.reward_hidden_state)
        logits = r0.policy_logits.cpu().numpy().tolist()
        ref_ms = []
        for _ in range(args.ref_reps):
            roots = search.roots(B, legal, action_space_size=A)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            roots.prepare(0.25, noises, [0.] * B, logits, tp)
            search.search(roots, ref_gpu, lat, hid, tp)
            torch.cuda.synchronize()
            ref_ms.append((time.perf_counter() - t0) * 1e3)
        m, rm = median(ms), median(ref_ms)
        print(f"{name:11s} B={B:5d} S={S}: search {m:9.3f} ms (median of {len(ms)}) | reference pipeline {rm:10.1f} ms "
              f"(median of {len(ref_ms)}) | ratio {rm / m:8.1f}x | {gpu}")


if __name__ == "__main__":
    main()
