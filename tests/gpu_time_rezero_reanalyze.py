"""Times one Atari MuZero ReZero reanalyze sweep (64x64 observations, A = 6, L = 5, S = 50, N = 256 and 1024) three ways:
  device  compute_target_policy_reanalyzed_rezero: one call, initial_inference + L searches + targets on the device;
  mirrors the reference's per-position loop over the existing mirrors (MuZeroMCTSCtree.search / search_with_reuse, a fresh Roots
          with prepare, get_values / get_distributions round trips between searches, targets in Python);
  ref     the reference pipeline: the compiled reference trees driven from the host (oracle/tree_drive.py), the same CUDA network
          evaluating the leaves (one repetition: it takes seconds).
Host clock around work that ends in a device synchronise; medians over repetitions after one warm-up of every shape.  Prints
the results with the card's name and power limit as JSON, and also writes them to PATH with --out PATH.
Run: python tests/gpu_time_rezero_reanalyze.py [--out PATH]"""
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

import test_gpu_rezero_reanalyze as T  # noqa: E402


def timed(fn, reps):
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return float(np.median(out)), out


def mirror_loop(model, obs, mask, tp, ta, pm, noises, pos, L, S, mini):
    import lightzero_b200 as lzb
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True))
    rows = obs.shape[0]
    N = rows // L
    lat, logit = [], []
    for beg in range(0, rows, mini):
        o = model.initial_inference(obs[beg:beg + mini].to(model.device, non_blocking=True))
        lat.append(o.latent_state)
        logit.append(o.policy_logits)
    lat, logit = torch.cat(lat), torch.cat(logit)
    values, dists = None, [None] * L
    for it in range(L):
        idx = [n * L + L - 1 - it for n in range(N)]
        roots = mcts.roots(N, mask[idx])
        roots.prepare(0.25, noises[idx], [0.] * N, logit[idx], tp[idx].tolist())
        if it == 0:
            mcts.search(roots, model, lat[idx], tp[idx].tolist())
        else:
            mcts.search_with_reuse(roots, model, lat[idx], tp[idx].tolist(), ta[idx].tolist(), values)
        values = roots.get_values()
        dists[it] = roots.get_distributions()
        roots.clear()
    A = mask.shape[1]
    out = np.zeros((N, L, A))
    for n in range(N):
        for p in range(L):
            if pm[n * L + p]:
                d = dists[L - 1 - p][n]
                s = sum(d)
                out[n, p, :len(d)] = [v / s for v in d]
    return out


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ref_trees = T._ref_trees()
    model, obs_shape, A, _, _, _ = T.make_model("atari_mz6")
    L, S, mini = 5, 50, 10240
    res = dict(gpu=smi, L=L, S=S, A=A, obs=list(obs_shape), cases=[])
    for N in (256, 1024):
        args = T.make_inputs(N, L, obs_shape, A, N, False, False, True)
        obs = args[0].pin_memory()
        args = (obs,) + args[1:]
        dev = lambda: T.device_sweep(model, False, *args, L, S, False, True, True, mini)      # noqa: E731
        mir = lambda: mirror_loop(model, *args, L, S, mini)                                   # noqa: E731
        d0, m0 = dev(), mir()
        assert np.array_equal(d0[0], m0), "device sweep and mirror loop disagree"
        t_dev, all_dev = timed(dev, 7)
        t_mir, all_mir = timed(mir, 5)
        case = dict(N=N, device_s=t_dev, mirrors_s=t_mir, device_all=all_dev, mirrors_all=all_mir)
        if ref_trees[0] is not None:
            t0 = time.perf_counter()
            e = T.oracle_sweep(ref_trees, model, False, *args, L, S, A, False, True, True, mini)
            torch.cuda.synchronize()
            case["ref_s"] = time.perf_counter() - t0
            assert np.array_equal(d0[0], e[0]), "device sweep and reference loop disagree"
        res["cases"].append(case)
        print(json.dumps(case))
    if "--out" in sys.argv:
        path = sys.argv[sys.argv.index("--out") + 1]
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(dict(gpu=smi, summary=[{k: v for k, v in c.items() if not k.endswith("_all")} for c in res["cases"]])))


if __name__ == "__main__":
    main()
