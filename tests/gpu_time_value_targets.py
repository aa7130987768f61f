"""Times the replay buffer's reward / value targets for one sampled batch, N = 256 segments x 6 rows, two ways:
  device  compute_target_reward_value: one call, initial_inference (value scalars only) [+ root search] + k_value_targets;
  ref     the reference's structure on the same CUDA model (game_buffer_muzero.py:467-575, game_buffer_efficientzero.py:167-323):
          initial_inference in mini_infer_size slices, host copies of the latents, value scalars and policy logits (and the
          LSTM state), [Roots.prepare + EfficientZeroMCTSCtree.search + get_values], then the host loops (oracle/targets_ref.py).
Configs: Atari MuZero 64x64 (A = 6), Atari EfficientZero 64x64 with use_root_value at S = 50, connect4 MuZero.
Host clock around work that ends in a device synchronise; medians over repetitions after one warm-up.  Prints the results with
the card's name and power limit as JSON, and also writes them to PATH with --out PATH.
Run: python tests/gpu_time_value_targets.py [--out PATH]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import test_gpu_value_targets as G  # noqa: E402
from oracle.targets_ref import reward_value_targets  # noqa: E402
from value_targets_cases import CASES  # noqa: E402


def timed(fn, reps):
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return float(np.median(out)), out


def reference_structure(model, obs, ctx, case, mini, root=None):
    ez = case["kind"] == "ez"
    vals, lats, logits, hid = [], [], [], []
    with torch.no_grad():
        for beg in range(0, obs.shape[0], mini):
            o = model.initial_inference(obs[beg:beg + mini].to(model.device, non_blocking=True))
            lats.append(o.latent_state.cpu().numpy())
            vals.append(model.inverse_scalar_transform(o.value).cpu().numpy())
            logits.append(o.policy_logits.cpu().numpy())
            if ez:
                hid.append((o.reward_hidden_state[0].cpu().numpy(), o.reward_hidden_state[1].cpu().numpy()))
    values = np.concatenate(vals).reshape(-1)
    if root is not None:
        S, noises = root
        T = obs.shape[0]
        import lightzero_b200 as lzb
        mcts = lzb.EfficientZeroMCTSCtree(dict(num_simulations=S, lstm_horizon_len=case["H"]))
        legal = [np.nonzero(ctx["action_mask"][j])[0].tolist() for j in range(T)]
        roots = mcts.roots(T, legal)
        tp = ctx["to_play"].tolist()
        roots.prepare(0.25, [n[:len(l)].tolist() for n, l in zip(noises, legal)], [0.0] * T, np.concatenate(logits).tolist(), tp)
        h = (np.concatenate([x[0] for x in hid], axis=1), np.concatenate([x[1] for x in hid], axis=1))
        mcts.search(roots, model, np.concatenate(lats), h, tp)
        values = np.asarray(roots.get_values(), np.float32)
        roots.clear()
    return reward_value_targets(values, *G.args_of(ctx), num_unroll_steps=case["K1"] - 1, discount_factor=case["discount"],
                                env_type=ctx["env_type"], efficientzero=ez, lstm_horizon_len=case.get("H", 5))


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    N, mini, S = 256, 10240, 50
    configs = [("atari_mz6", dict(CASES["mz_f32_n7_k6"], N=N), False),
               ("atari_ez", dict(CASES["ez_root_f32_n7_k6_h5"], N=N), True),
               ("connect4", dict(CASES["mz_2p_f32_n64_k6"], N=N), False)]
    res = dict(gpu=smi, N=N, rows=N * 6, S=S, cases=[])
    for family, case, root in configs:
        model, obs_shape, A, _ = G.model_of(family)
        ctx, obs = G.case_inputs(case, N, obs_shape, A)
        obs = obs.pin_memory()
        if root:
            dev = lambda: G.device_root(model, obs, ctx, case, S, True, ctx["noises"], mini)            # noqa: E731
            ref = lambda: reference_structure(model, obs, ctx, case, mini, (S, ctx["noises"]))         # noqa: E731
        else:
            dev = lambda: G.device_targets(model, obs, ctx, case, mini)                                 # noqa: E731
            ref = lambda: reference_structure(model, obs, ctx, case, mini)                             # noqa: E731
        d0, r0 = dev(), ref()
        if root:     # the same values feed both: the targets agree bit for bit
            G.assert_bits(d0, r0)
        else:        # the reference structure bootstraps from h^-1 of the logits: the targets agree up to the scalar contract
            assert np.abs(d0[1] - r0[1]).max() <= 5e-4 and np.array_equal(d0[0], r0[0])
        t_dev, all_dev = timed(dev, 9)
        t_ref, all_ref = timed(ref, 5)
        c = dict(config=family + ("_root" if root else ""), device_s=t_dev, ref_s=t_ref, device_all=all_dev, ref_all=all_ref)
        res["cases"].append(c)
        print(json.dumps(c))
    if "--out" in sys.argv:
        path = sys.argv[sys.argv.index("--out") + 1]
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(dict(gpu=smi, summary=[{k: v for k, v in c.items() if not k.endswith("_all")} for c in res["cases"]])))


if __name__ == "__main__":
    main()
