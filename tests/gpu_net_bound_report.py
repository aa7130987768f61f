"""Worst |err| / bound per layer of the latent-grid tensor-core network (tests/test_gpu_net_layers.py), for the
3xFP16 (tc3) and single-pass (tc1) builds, plus the heads' float64 margin with the FC weights' lo parts dropped.
Backs the table of DESIGN.md 4.3.  Run on a GPU:  python tests/gpu_net_bound_report.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_net_layers as T  # noqa: E402


def main():
    print(torch.cuda.get_device_name(0))
    print("TAU", {k: f"{v:.4g}" for k, v in T.TAU.items()})
    cases = [("A18 hc16", dict(A=18, seed=11)), ("A6 hc8", dict(A=6, hc=(8, 8, 8), seed=5)),
             ("A608 nres2 hc1/16/8 K608", dict(A=608, nres=2, hc=(1, 16, 8), hid=8, support=(-304., 304., 1.), seed=610))]
    for name, kw in cases:
        support = kw.get("support", T.SUPPORT)
        for math in ("tc3", "tc1"):
            ref64, cu = T.make_models(math=math, **kw)
            for B in (131, 1024):
                latent = T.make_latents(B, seed=B)
                action = (torch.arange(B) % kw["A"]).cuda()
                for which in (0, 1):
                    r, _, _, _ = T.run_program(cu, ref64, which, latent, action, support)
                    print(f"{name:22s} {math} B={B:5d} {'rec ' if which == 0 else 'tail'}",
                          " ".join(f"{k}={v:.3g}" for k, v in r.items()), flush=True)
                    if math == "tc3":
                        r, _, _, _ = T.run_program(cu, ref64, which, latent, action, support, hi_only=True)
                        print(f"{name:22s} f64 hi-only B={B:5d} {'rec ' if which == 0 else 'tail'}",
                              " ".join(f"{k}={v:.3g}" for k, v in r.items() if k.endswith("head")), flush=True)


if __name__ == "__main__":
    main()
