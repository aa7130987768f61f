"""Times of the board Stochastic MuZero network (StochasticMuZeroModel, downsample=False) at the shipped 2048 config
(observation (16, 4, 4), 4 actions, 32 chance outcomes, C = 64, num_simulations = 100, collector_env_num = 8), on the GPU:
  - `StochasticMuZeroMCTSCtree.search` (prepare + one search graph) at B = 8, 256 and 1024, CUDA events, median;
  - the reference pipeline at the same B: the compiled, unmodified reference stochastic ctree (oracle/_ref/stochastic_mz_tree)
    driven by the reference's per-simulation host loop (oracle/tree_drive.py, kind "stoch"; chance leaves and decision leaves
    evaluated as two batches) with the PyTorch restatement in eager mode on the same GPU; host clock around work that ends in
    a device synchronise;
  - one collect step (`StochasticMuZeroCollectPolicy.search_batch`: initial_inference, reset, prepare, search) at B = 8;
  - one launch of each recurrent program at B = 1024, unmasked and with a row mask selecting about half the roots at random
    (as the search splits its leaves): a CTA whose roots mix both kinds runs its MMAs in both launches.
Prints one JSON line with the card's name and power limit.  Sets no threshold.
    python tests/gpu_time_stochastic_board.py [--reps N] [--ref-reps N]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import stoch_board_model_ref as SB  # noqa: E402

NAME, S = "game_2048", 100
CHANCE_SEED = 7


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0]


class EagerGPU:
    """the restatement on the GPU with the reference's host-side read-out (softmax . support -> h^-1) of the scalars"""

    def __init__(self, ref, support):
        self.ref = ref
        self.support = torch.arange(*support, dtype=torch.float32, device="cuda")
        self.action_space_size, self.chance_space_size = ref.action_space_size, ref.chance_space_size

    def eval(self):
        return self

    def _scalar(self, logits):
        v = (torch.softmax(logits, -1) * self.support).sum(-1)
        eps = 0.001
        return torch.sign(v) * (((torch.sqrt(1 + 4 * eps * (torch.abs(v) + 1 + eps)) - 1) / (2 * eps)) ** 2 - 1)

    @torch.no_grad()
    def recurrent_inference(self, state, option, afterstate=False, return_scalars=True):
        o = self.ref.recurrent_inference(state, option.cuda(), afterstate)
        o.reward_scalar, o.value_scalar = self._scalar(o.reward), self._scalar(o.value)
        return o


def events_ms(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def main():
    import lightzero_b200 as lzb
    from lightzero_b200 import cabi
    from oracle import build_stoch_ref
    from oracle.tree_drive import drive, network
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--ref-reps", type=int, default=2)
    args = ap.parse_args()
    obs_shape, A, NC = SB.CONFIGS[NAME][:3]
    sup = SB.CONFIGS[NAME][7]
    ref = SB.build(NAME, 0)
    cu = lzb.StochasticMuZeroModel(**SB.model_kwargs(NAME)).load_state_dict(ref.state_dict())
    eager = EagerGPU(ref.cuda().eval(), sup)
    oracle = build_stoch_ref.load()
    rows = []
    for B in (8, 256, 1024):
        rng = np.random.default_rng(B)
        obs = torch.from_numpy(rng.random((B,) + obs_shape, dtype=np.float32)).cuda()
        legal = [list(range(A))] * B
        noises = [rng.dirichlet([0.3] * A).astype(np.float32).tolist() for _ in range(B)]
        tp = [-1] * B
        o = cu.initial_inference(obs)
        # the compiled reference tree draws its chance outcomes from a pinned random_device: both searches pin the draw
        mcts = lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, chance_seed=CHANCE_SEED))
        roots = mcts.roots(B, legal, NC)

        def one():
            roots.prepare(0.25, noises, [0.] * B, o.policy_logits, tp)
            mcts.search(roots, cu, o.latent_state, tp)
        row = dict(B=B, S=S, search_ms=round(events_ms(one, args.reps), 3), graph_kernels=mcts.last_num_kernels)
        roots.clear()
        if oracle is not None:
            with torch.no_grad():
                r0 = ref.initial_inference(obs)
            c = dict(B=B, A=A, C=NC, S=S, legal=legal, root_logits=r0.policy_logits.cpu().numpy(), noises=noises, to_play=tp,
                     chance_seed=CHANCE_SEED)
            ref_ms = []
            for _ in range(args.ref_reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                drive(oracle, c, "stoch", network(eager, r0.latent_state, stochastic=True), det=True)
                torch.cuda.synchronize()
                ref_ms.append((time.perf_counter() - t0) * 1e3)
            row["reference_pipeline_ms"] = round(float(np.median(ref_ms)), 1)
            row["ratio"] = round(row["reference_pipeline_ms"] / row["search_ms"], 1)
        rows.append(row)

    # one collect step at collector_env_num = 8
    B = 8
    rng = np.random.default_rng(1)
    obs = torch.from_numpy(rng.random((B,) + obs_shape, dtype=np.float32)).cuda()
    mask = torch.ones(B, A, dtype=torch.uint8, device="cuda")
    noises = torch.from_numpy(rng.dirichlet([0.3] * A, B).astype(np.float32)).cuda()
    pol = lzb.StochasticMuZeroCollectPolicy(cu, dict(num_simulations=S, chance_seed=None))
    collect_ms = events_ms(lambda: pol.search_batch(obs, mask, noises, [-1] * B, read_back=False), args.reps)

    # one launch of each recurrent program at B = 1024, unmasked and masked
    B = 1024
    g = torch.Generator().manual_seed(5)
    state = torch.rand((B,) + cu.latent_shape, generator=g).cuda()
    K = cu.value_support_size
    launches = {}
    for afterstate in (False, True):
        opt = torch.randint(0, NC if afterstate else A, (B,), generator=g).int().cuda()
        outs = [torch.empty(s, device="cuda") for s in ((B,) + cu.latent_shape, (B, K), (B, K), (B, max(A, NC)), (B,), (B,))]
        mask = torch.randint(0, 2, (B,), generator=g).int().cuda()
        for masked in (False, True):
            def launch():
                cabi.check(cu._lib.lz_model_recurrent_inference_stochastic(
                    cu._h, int(afterstate), B, state.data_ptr(), opt.data_ptr(), mask.data_ptr() if masked else None, 1,
                    outs[0].data_ptr(), None, None, outs[3].data_ptr(), outs[4].data_ptr(), outs[5].data_ptr(),
                    cabi.stream_ptr()), "launch")
            launches[f"{'rec' if afterstate else 'after'}_{'masked' if masked else 'full'}_ms"] = round(
                events_ms(launch, 5 * args.reps), 4)
    print(json.dumps(dict(card=card(), config=NAME, search=rows, collect_B8_ms=round(collect_ms, 3), launch_B1024=launches)))


if __name__ == "__main__":
    main()
