"""Reports, per DownSample tower stage, the worst element of |y_cuda - y_f64| / (TAU M + ALPHA S) (the bound of
tests/test_gpu_tower_layers.py) for the 3xFP16 (tc3) and single-pass (tc1) tensor-core builds, at 84 and 96 px, float and
uint8 frames.  tc3 should stay <= 0.25 and tc1 should reach >= 8 on every wgmma stage.  The card's name and power limit are
printed with the numbers.

  python tests/gpu_tower_bound_report.py [--B 1024] [--json FILE]
"""
import argparse
import json
import math
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=1024)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    import test_gpu_tower_layers as T
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(f"# {card}; B = {args.B}; TAU = {['2^%d' % round(math.log2(t)) for t in T.TAU]}")
    rows = {}
    for px in T.PX:
        for mode in ("tc3", "tc1"):
            _, ref64, cu = T._models((4, px, px), math=mode)
            for kind in T.KINDS:
                obs, x64 = T._inputs(kind, args.B, 4, px, seed=px + args.B)
                ratios, _, _, _ = T.stage_ratios(cu, ref64, obs, x64)
                rows[f"{px} {mode} {kind}"] = ratios
                print(f"{px:3d} {mode} {kind:5s} " + " ".join(f"{n}={r:.3g}" for n, r in zip(T.STAGE_NAMES, ratios)), flush=True)
                torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card, B=args.B, ratios=rows), f, indent=1)


if __name__ == "__main__":
    main()
