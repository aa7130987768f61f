"""Times the fused MuZero search (bench size by default) with CUDA events, uninstrumented: the A/B tool for kernel variants
(LZ_LIB_TAG=<tag> picks lightzero_b200/_lib/<tag>/liblzb200.so)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lightzero_b200 as lzb
from lightzero_b200.synthetic_weights import synthetic_state_dict

B, S, A = int(os.environ.get("DBG_B", 1024)), int(os.environ.get("DBG_S", 50)), int(os.environ.get("DBG_A", 18))
model = lzb.MuZeroModel(observation_shape=(4, 84, 84), action_space_size=A).load_state_dict(synthetic_state_dict((4, 84, 84), A))
obs = torch.rand(B, 4, 84, 84).cuda()
out0 = model.initial_inference(obs)
mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=0.997))
noise = torch.from_numpy(np.random.default_rng(0).dirichlet([0.3] * A, size=B).astype(np.float32)).cuda()
mask = torch.ones(B, A, dtype=torch.uint8)
ms = []
for it in range(int(os.environ.get("DBG_N", 8))):
    roots = mcts.roots(B, mask)
    roots.prepare(0.25, noise, None, out0.policy_logits, None)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    mcts.search(roots, model, out0.latent_state, None)
    b.record()
    torch.cuda.synchronize()
    ms.append(a.elapsed_time(b))
vis = np.asarray(roots.get_distributions()).sum()
print(f"tag={os.environ.get('LZ_LIB_TAG', '-')} B={B} S={S} A={A}: search ms min {min(ms[2:]):.3f} median {sorted(ms[2:])[len(ms[2:]) // 2]:.3f}  (visits {int(vis)})")
