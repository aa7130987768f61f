"""Times the fused MuZero search and initial_inference at one observation size with CUDA events, uninstrumented
(DBG_OBS: 64 by default, the 8x8 latent grid; 84 / 96 for the 6x6 grid).  Same method as gpu_time_search.py /
gpu_time_tower.py; LZ_LIB_TAG=<tag> picks lightzero_b200/_lib/<tag>/liblzb200.so."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lightzero_b200 as lzb
from lightzero_b200.synthetic_weights import synthetic_state_dict

PX = int(os.environ.get("DBG_OBS", 64))
B, S, A = int(os.environ.get("DBG_B", 1024)), int(os.environ.get("DBG_S", 50)), int(os.environ.get("DBG_A", 18))
model = lzb.MuZeroModel(observation_shape=(4, PX, PX), action_space_size=A, downsample=True)
model.load_state_dict(synthetic_state_dict((4, PX, PX), A))


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


obs = [torch.rand(B, 4, PX, PX).cuda() for _ in range(3)]
ms_init = [timed(lambda: model.initial_inference(obs[i % 3])) for i in range(12)][3:]
out0 = model.initial_inference(obs[0])
mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=0.997))
noise = torch.from_numpy(np.random.default_rng(0).dirichlet([0.3] * A, size=B).astype(np.float32)).cuda()
mask = torch.ones(B, A, dtype=torch.uint8)
ms_search = []
for it in range(int(os.environ.get("DBG_N", 8))):
    roots = mcts.roots(B, mask)
    roots.prepare(0.25, noise, None, out0.policy_logits, None)
    ms_search.append(timed(lambda: mcts.search(roots, model, out0.latent_state, None)))
ms_search = ms_search[2:]
vis = np.asarray(roots.get_distributions()).sum()
print(f"tag={os.environ.get('LZ_LIB_TAG', '-')} obs={PX} latent={model.latent_hw}x{model.latent_hw} B={B} S={S} A={A}: "
      f"search ms min {min(ms_search):.3f} median {sorted(ms_search)[len(ms_search) // 2]:.3f} (visits {int(vis)}); "
      f"initial_inference ms min {min(ms_init):.3f} median {sorted(ms_init)[len(ms_init) // 2]:.3f}")
