"""clock64 phase stamps of CTA 0 for the LAST simulation of a persistent search launch (bench size by default).
Run on the GPU box:  LZ_TC_DEBUG=1 python tests/gpu_debug_search.py   (not a pytest; needs a build with the dbg stamps)."""
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("LZ_TC_DEBUG", "1")
import lightzero_b200 as lzb
from lightzero_b200 import cabi
from oracle.model_ref import MuZeroModelRef, emulate_trained_


def main():
    B, S, A = int(os.environ.get("DBG_B", 1024)), int(os.environ.get("DBG_S", 50)), int(os.environ.get("DBG_A", 18))
    torch.manual_seed(0)
    ref = emulate_trained_(MuZeroModelRef((4, 84, 84), A), 0)
    model = lzb.MuZeroModel(observation_shape=(4, 84, 84), action_space_size=A).load_state_dict(ref.state_dict())
    lib = cabi.load()
    obs = torch.rand(B, 4, 84, 84).cuda()
    out0 = model.initial_inference(obs)
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    rng = np.random.default_rng(0)
    noise = torch.from_numpy(rng.dirichlet([0.3] * A, size=B).astype(np.float32)).cuda()
    mask = torch.ones(B, A, dtype=torch.uint8)
    ms = []
    for it in range(4):
        roots = mcts.roots(B, mask)
        roots.prepare(0.25, noise, None, out0.policy_logits, None)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        mcts.search(roots, model, out0.latent_state, None)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    print(f"search (B={B}, S={S}, A={A}) ms per call: {['%.3f' % m for m in ms]}  (instrumented build: slower than the bench)")
    buf = (ctypes.c_ulonglong * 64)()
    cabi.check(lib.lz_debug_tc_stamps(buf), "stamps")
    s = list(buf)
    t0 = s[50]
    rel = lambda i: s[i] - t0
    print("== last simulation of CTA 0, cycles since the start of the simulation (tree phase first)")
    print(f"   tree: backprop done {rel(56):8d}  traverse done (warp 0) + CTA barrier {rel(51):8d}")
    print(f"   load done                        {rel(1):8d}")
    prev = 1
    for L in range(5):
        print(f"   L{L}: MMAs done {rel(2 + 2 * L):8d}  epilogue (+ hooks) done {rel(3 + 2 * L):8d}"
              f"   [mma {s[2 + 2 * L] - s[prev]:6d}  epi {s[3 + 2 * L] - s[2 + 2 * L]:6d}]")
        prev = 3 + 2 * L
    print(f"   layers done                      {rel(24):8d}")
    print(f"   heads: B operand ready {rel(44):8d}  FC1 {rel(45):8d}  hidden {rel(46):8d}  FC2 {rel(47):8d}  all done {rel(27):8d}")
    print(f"   total kernel cycles (start stamp -> end of last sim) {s[27] - s[0]}  = {(s[27] - s[0]) / S:.0f} per simulation")


if __name__ == "__main__":
    main()
