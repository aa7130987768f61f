"""Collect-step time of Stochastic MuZero for the shipped vector-observation configs (cartpole at 25 simulations, lunarlander_disc
and pendulum_cont_disc at 50): the fused device collect (StochasticMuZeroCollectPolicy.forward_collect: one initial inference
and root preparation, one search graph, one read-back) against the reference's _forward_collect pipeline
(lzero/policy/stochastic_muzero.py:578-653) on the same GPU and the same network: initial_inference, the latents / logits /
values to the host, Roots.prepare, StochasticMuZeroMCTSCtree.search, get_distributions / get_values read back as lists, and per
root select_action on the host.  Pinned host observations in, the output dict out, median over --reps steps after warm-up,
timed with a host clock around work that ends in a device synchronise.  A third number is the step of the collector loop of
INTEGRATION.md section 5: search_batch(read_back=False) with select_action on the device, and only the actions copied back.
Prints the card name and power limit with the numbers.  Writes nothing.
usage: python tests/gpu_time_stochastic_collect.py [--envs 8,1024] [--reps 10]"""
import argparse
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from gpu_time_gumbel_collect import _card, _median_ms  # noqa: E402

CONFIGS = {"cartpole": 25, "lunarlander_disc": 50, "pendulum_cont_disc": 50}     # name: num_simulations


def reference_step(model, mcts, obs, mask, tp, temperature):
    """StochasticMuZeroPolicy._forward_collect (stochastic_muzero.py:614-653) on this project's network and stochastic search"""
    from lightzero_b200.collect import select_action
    B = mask.shape[0]
    out = model.initial_inference(obs.cuda(non_blocking=True), return_scalar_value=True)
    pred_values = out.value_scalar.cpu().numpy()
    latent = out.latent_state.cpu().numpy()
    logits = out.policy_logits.cpu().numpy().tolist()
    legal = [np.nonzero(mask[j])[0].tolist() for j in range(B)]
    noises = [np.random.dirichlet([0.3] * int(sum(mask[j]))).astype(np.float32).tolist() for j in range(B)]
    roots = mcts.roots(B, legal, model.chance_space_size)
    roots.prepare(0.25, noises, [0.0] * B, logits, tp)
    mcts.search(roots, model, latent, tp)
    dist, values = roots.get_distributions(), roots.get_values()
    output = {}
    for i in range(B):
        d = dist[i][:len(legal[i])]
        pos, ent = select_action(d, temperature=temperature, deterministic=False)
        output[i] = dict(action=legal[i][pos], visit_count_distributions=d, visit_count_distribution_entropy=ent,
                         searched_value=values[i], predicted_value=pred_values[i], predicted_policy_logits=logits[i])
    roots.clear()
    return output


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", default="8,1024")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures GPU time and has nothing to measure without one")
    import lightzero_b200 as lzb
    import stoch_mlp_model_ref as SR
    from lightzero_b200.collect import _legal_dirichlet
    print(f"card: {_card()}")
    for name in a.configs.split(","):
        S = CONFIGS[name]
        A = SR.CONFIGS[name][1]
        model = lzb.StochasticMuZeroModelMLP(**SR.model_kwargs(name)).load_state_dict(SR.build(name, 0).state_dict())
        cfg = dict(num_simulations=S, discount_factor=0.997)
        for B in (int(x) for x in a.envs.split(",")):
            rng = np.random.default_rng(0)
            obs = torch.rand((B, SR.CONFIGS[name][0]), generator=torch.Generator().manual_seed(0)).pin_memory()
            mask = (rng.random((B, A)) < 0.7).astype(np.uint8)
            mask[np.arange(B), rng.integers(0, A, B)] = 1
            tp = [-1] * B
            pol = lzb.StochasticMuZeroCollectPolicy(model, cfg)
            mcts = lzb.StochasticMuZeroMCTSCtree(cfg)
            fused = _median_ms(lambda: pol.forward_collect(obs, mask, temperature=1.0, to_play=tp), a.reps)
            ref = _median_ms(lambda: reference_step(model, mcts, obs, mask, tp, 1.0), a.reps)
            loop = _median_ms(lambda: pol.search_batch(obs, mask, _legal_dirichlet(mask, 0.3), tp, read_back=False,
                                                       select=(1.0, False, 0))["action"].cpu(), a.reps)
            print(f"{name}: {B} envs x {S} simulations, collect step median {fused[0]:.3f} ms (min {fused[1]:.3f}, max "
                  f"{fused[2]:.3f}) fused vs {ref[0]:.3f} ms (min {ref[1]:.3f}, max {ref[2]:.3f}) reference pipeline: "
                  f"{ref[0] / fused[0]:.2f}x; device-loop step (actions only back) {loop[0]:.3f} ms (min {loop[1]:.3f}, max "
                  f"{loop[2]:.3f}); {pol.last_num_kernels} kernels in the search graph")


if __name__ == "__main__":
    main()
