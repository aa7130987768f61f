"""Median search time of the MuZeroModelMLP configs on the tensor-core MLP kernel (lunarlander MuZero, latent 256) on the GPU,
against the reference pipeline on the same GPU.

Per B in {8, 256, 1024} (a collector batch, larger collectors, a reanalyze batch), S = 50:
  - this library: `MuZeroMCTSCtree.search` on the model, prepare included (prepare + one search graph), CUDA events;
  - the reference pipeline: the compiled, unmodified reference mz_tree (oracle/_ref, or the C port where it is not built) driven
    by the reference's per-simulation host loop (oracle/search_ref.py SearchRef) with the PyTorch restatement of the network in
    eager mode on the same GPU; host clock around work that ends in a device synchronise.
Before the first search, the time of single initial_inference / recurrent_inference calls at B = 1 .. 1024 (one CTA holds 64
roots).  Prints one line per case with the card's name and power limit.  Sets no threshold.
    python tests/gpu_time_mlp_mz.py [--reps N] [--ref-reps N]
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

import mlp_mz_model_ref as MR  # noqa: E402
from gpu_time_board import card, median  # noqa: E402

NAME, S = "lunarlander", 50
BATCHES = (8, 256, 1024)


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


def call_times(cu, reps):
    """median time of one initial_inference / recurrent_inference call (CUDA events) at B = 1, 8, 64, 65, 1024"""
    obs_dim = MR.CONFIGS[NAME][0]
    for B in (1, 8, 64, 65, 1024):
        obs = torch.rand(B, obs_dim, device="cuda")
        o = cu.initial_inference(obs)
        act = torch.zeros(B, dtype=torch.int32, device="cuda")
        res = []
        for fn in (lambda: cu.initial_inference(obs), lambda: cu.recurrent_inference(o.latent_state, act)):
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
        print(f"{NAME:11s} B={B:5d}: initial_inference {res[0]:7.1f} us, recurrent_inference {res[1]:7.1f} us (median of {reps})")


def main():
    import lightzero_b200 as lzb
    from oracle.search_ref import SearchRef, load_tree_module
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--ref-reps", type=int, default=3)
    args = ap.parse_args()
    tree_mod, tree_kind = load_tree_module(prefer_ref=True, name="mz_tree")
    gpu = card()
    print(f"card: {gpu}; reference tree: {tree_kind}")
    ref = MR.build(NAME, 0)
    cu = lzb.MuZeroModelMLP(**MR.model_kwargs(NAME)).load_state_dict(ref.state_dict())
    ref_gpu = EagerGPU(ref.cuda().eval())
    call_times(cu, args.reps)
    obs_dim, A = MR.CONFIGS[NAME][:2]
    for B in BATCHES:
        rng = np.random.default_rng(B)
        obs = (torch.rand((B, obs_dim), generator=torch.Generator().manual_seed(B)) * 2 - 1).cuda()
        legal = [list(range(A))] * B
        noises = [rng.dirichlet([0.3] * A).astype(np.float32).tolist() for _ in range(B)]
        tp = [-1] * B
        out = cu.initial_inference(obs)
        mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, discount_factor=0.997))
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
        search = SearchRef(tree_mod, num_simulations=S, discount_factor=0.997)
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
        print(f"{NAME:11s} B={B:5d} S={S}: search {m:9.3f} ms (median of {len(ms)}) | reference pipeline {rm:10.1f} ms "
              f"(median of {len(ref_ms)}) | ratio {rm / m:8.1f}x | {gpu}")


if __name__ == "__main__":
    main()
