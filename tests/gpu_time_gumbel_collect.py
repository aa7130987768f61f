"""Collect-step time of Gumbel MuZero for the shipped Atari (64x64, A = 18), tictactoe and lunarlander configs: the fused
device collect (GumbelMuZeroCollectPolicy.forward_collect: one initial inference, one search graph, one read-out kernel, one
read-back) against the reference's _forward_collect pipeline (lzero/policy/gumbel_muzero.py:549-605) on the same GPU and the
same network: initial_inference, the latents / logits / values to the host, Roots.prepare, GumbelMuZeroMCTSCtree.search,
get_distributions / get_values / get_children_values / get_policies read back as lists, and per root the masked arg-max and
select_action on the host.  Pinned host observations in, the output dict out, median over --reps steps after warm-up, timed
with a host clock around work that ends in a device synchronise.  Prints the card name and power limit with the numbers.
Writes nothing.
usage: python tests/gpu_time_gumbel_collect.py [--envs 8,256] [--sims 50] [--reps 10]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CONFIGS = {   # name: (model kind, observation shape, A, max_num_considered_actions, to_play)
    "atari": ("conv", (4, 64, 64), 18, 18, -1),
    "tictactoe": ("board", (3, 3, 3), 9, 9, 1),
    "lunarlander": ("mlp", (8,), 4, 4, -1),
}


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def _model(name):
    import lightzero_b200 as lzb
    from lightzero_b200.synthetic_weights import synthetic_state_dict
    kind, obs, A, _, _ = CONFIGS[name]
    if kind == "conv":
        return lzb.MuZeroModel(observation_shape=obs, action_space_size=A, downsample=True).load_state_dict(
            synthetic_state_dict(observation_shape=obs, action_space_size=A))
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    if kind == "board":
        import board_model_ref as BR
        return lzb.MuZeroModel(**BR.model_kwargs(name)).load_state_dict(BR.build(name, 0).state_dict())
    import mlp_mz_model_ref as MR
    return lzb.MuZeroModelMLP(**MR.model_kwargs(name)).load_state_dict(MR.build(name, 0).state_dict())


def reference_step(model, mcts, obs, mask, tp, temperature, discount):
    """GumbelMuZeroPolicy._forward_collect (gumbel_muzero.py:549-605) on this project's network and Gumbel search"""
    from lightzero_b200.collect import select_action
    B, A = mask.shape
    out = model.initial_inference(obs.cuda(non_blocking=True), return_scalar_value=True)
    pred_values = out.value_scalar.cpu().numpy()
    latent = out.latent_state.cpu().numpy()
    logits = out.policy_logits.cpu().numpy().tolist()
    legal = [np.nonzero(mask[j])[0].tolist() for j in range(B)]
    noises = [np.random.dirichlet([0.3] * int(sum(mask[j]))).astype(np.float32).tolist() for j in range(B)]
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.0] * B, list(pred_values), logits, tp)
    mcts.search(roots, model, latent, tp)
    dist, values = roots.get_distributions(), roots.get_values()
    completed = roots.get_children_values(discount, A)
    improved = np.array(roots.get_policies(discount, A))
    output = {}
    for i in range(B):
        _, ent = select_action(dist[i], temperature=temperature, deterministic=False)
        output[i] = dict(action=np.argmax(np.where(mask[i] == 1, improved[i], 0.0)), visit_count_distributions=dist[i],
                         visit_count_distribution_entropy=ent, searched_value=values[i],
                         roots_completed_value=np.where(mask[i] == 1, completed[i], 0.0), improved_policy_probs=improved[i],
                         predicted_value=pred_values[i], predicted_policy_logits=logits[i])
    roots.clear()
    return output


def _median_ms(step, reps):
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        step()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ms)), float(np.min(ms)), float(np.max(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", default="8,256")
    ap.add_argument("--sims", type=int, default=50)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures GPU time and has nothing to measure without one")
    import lightzero_b200 as lzb
    S = a.sims
    print(f"card: {_card()}")
    for name in a.configs.split(","):
        _, shape, A, m, tp0 = CONFIGS[name]
        model = _model(name)
        cfg = dict(num_simulations=S, max_num_considered_actions=m, discount_factor=0.997)
        for B in (int(x) for x in a.envs.split(",")):
            rng = np.random.default_rng(0)
            obs = torch.rand((B,) + shape, generator=torch.Generator().manual_seed(0)).pin_memory()
            mask = (rng.random((B, A)) < 0.7).astype(np.uint8)
            mask[np.arange(B), rng.integers(0, A, B)] = 1
            tp = [tp0] * B
            pol = lzb.GumbelMuZeroCollectPolicy(model, cfg)
            mcts = lzb.GumbelMuZeroMCTSCtree(cfg)
            fused = _median_ms(lambda: pol.forward_collect(obs, mask, temperature=1.0, to_play=tp), a.reps)
            ref = _median_ms(lambda: reference_step(model, mcts, obs, mask, tp, 1.0, 0.997), a.reps)
            print(f"{name}: {B} envs x {S} simulations, collect step median {fused[0]:.3f} ms (min {fused[1]:.3f}, max "
                  f"{fused[2]:.3f}) fused vs {ref[0]:.3f} ms (min {ref[1]:.3f}, max {ref[2]:.3f}) reference pipeline: "
                  f"{ref[0] / fused[0]:.2f}x; {pol.last_num_kernels} kernels in the search graph")


if __name__ == "__main__":
    main()
