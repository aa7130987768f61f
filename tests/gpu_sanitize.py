"""Small end-to-end exercise of every kernel family for compute-sanitizer (memcheck / racecheck / synccheck):
   compute-sanitizer --tool memcheck python tests/gpu_sanitize.py
Sizes are tiny: the sanitizer slows kernels 10-100x."""
import os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lightzero_b200 as lzb
from lightzero_b200.collect import MuZeroCollectPolicy
from oracle.model_ref import MuZeroModelRef, emulate_trained_, MuZeroModelMLPRef, emulate_trained_mlp_

torch.manual_seed(0)
A, B, S = 6, 9, 6
ref = emulate_trained_(MuZeroModelRef((4, 84, 84), A), 0)
for math in ("tc3", "tc1"):
    cu = lzb.MuZeroModel(observation_shape=(4, 84, 84), action_space_size=A).load_state_dict(ref.state_dict()).set_math(math)
    pol = MuZeroCollectPolicy(cu, dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    obs = torch.rand(B, 4, 84, 84)
    mask = (np.random.default_rng(0).random((B, A)) < 0.7).astype(np.uint8); mask[:, 0] = 1
    noise = np.random.default_rng(1).dirichlet([0.3] * A, size=B).astype(np.float32)
    r = pol.search_batch(obs.pin_memory(), mask, noise, None)
    assert int(r["visits"].clamp(min=0).sum()) == B * S
    r2 = pol.search_batch(obs.cuda(), mask, noise, None, deterministic=False)
    assert int(r2["visits"].clamp(min=0).sum()) == B * S
    print(math, "ok", r["values"][:3].tolist())
mref = emulate_trained_mlp_(MuZeroModelMLPRef(4, 2), 0)
mcu = lzb.MuZeroModelMLP(4, 2, res_connection_in_dynamics=True).load_state_dict(mref.state_dict())
mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=5, deterministic=True))
o = mcu.initial_inference((torch.rand(5, 4) * 2 - 1).cuda())
roots = mcts.roots(5, [[0, 1]] * 5)
roots.prepare_no_noise([0.] * 5, o.policy_logits, [1, 2, 1, 2, 1])     # two-player sign flips
mcts.search(roots, mcu, o.latent_state, [1, 2, 1, 2, 1])
print("mlp ok", roots.get_distributions(), roots.get_trajectories()[:2])
# EfficientZero: value-prefix trees, LSTM value-prefix head, multi-kernel search graph, collect from host buffers
from lightzero_b200.collect import EfficientZeroCollectPolicy
from oracle.model_ref import EfficientZeroModelRef
eref = emulate_trained_(EfficientZeroModelRef((4, 96, 96), A), 1)
ecu = lzb.EfficientZeroModel(observation_shape=(4, 96, 96), action_space_size=A).load_state_dict(eref.state_dict())
epol = EfficientZeroCollectPolicy(ecu, dict(num_simulations=8, discount_factor=0.997, lstm_horizon_len=2))
eobs = torch.rand(B, 4, 96, 96)
r = epol.search_batch(eobs.pin_memory(), mask, noise, None)
assert int(r["visits"].clamp(min=0).sum()) == B * 8
emcts = lzb.EfficientZeroMCTSCtree(dict(num_simulations=8, lstm_horizon_len=2))
eo = ecu.initial_inference(eobs.cuda())
eroots = emcts.roots(B, [list(range(A))] * B)
eroots.prepare(0.25, noise, [0.] * B, eo.policy_logits, [1, 2] * (B // 2) + [1])     # two-player branch
emcts.search(eroots, ecu, eo.latent_state, eo.reward_hidden_state, [1, 2] * (B // 2) + [1])
print("efficientzero ok", r["values"][:3].tolist(), eroots.get_distributions()[:2])
# a batch that leaves the last CTA of the persistent kernel partly filled (8 roots per CTA), the fused reuse searches, the
# uint8 entry point fed by the device-resident frame stack, GameSegment statistics
from lightzero_b200.collector import FrameStack, SegmentStats
B2 = 132 * 7 + 5
cu = lzb.MuZeroModel(observation_shape=(4, 84, 84), action_space_size=A).load_state_dict(ref.state_dict())
pol = MuZeroCollectPolicy(cu, dict(num_simulations=4, deterministic=True, discount_factor=0.997))
fs = FrameStack(B2, 4, 84, 84)
rng = np.random.default_rng(5)
fs.push(rng.integers(0, 256, (B2, 84, 84), dtype=np.uint8), reset=np.ones(B2, np.uint8))
fs.push(rng.integers(0, 256, (B2, 84, 84), dtype=np.uint8))
mask2 = torch.ones(B2, A, dtype=torch.uint8).cuda()
noise2 = torch.from_numpy(rng.dirichlet([0.3] * A, size=B2).astype(np.float32)).cuda()
r = pol.search_batch(fs.view(), mask2, noise2, None, read_back=False)
assert int(r["visits"].clamp(min=0).sum()) == B2 * 4
seg = SegmentStats(B2, 3, A)
seg.store_search_stats(r["visits"], r["values"])
seg.reset(np.ones(B2, np.uint8))
mcts2 = lzb.MuZeroMCTSCtree(dict(num_simulations=4, deterministic=True))
o2 = cu.initial_inference(torch.rand(20, 4, 84, 84).cuda())
roots2 = mcts2.roots(20, [list(range(A))] * 20)
roots2.prepare(0.25, noise[:1].repeat(20, 0), [0.] * 20, o2.policy_logits, [-1] * 20)
mcts2.search_with_reuse(roots2, cu, o2.latent_state, [-1] * 20, [1] * 20, [0.3] * 20)
eroots2 = emcts.roots(B, [list(range(A))] * B)
eroots2.prepare(0.25, noise, [0.] * B, eo.policy_logits, [-1] * B)
emcts.search_with_reuse(eroots2, ecu, eo.latent_state, eo.reward_hidden_state, [-1] * B, [2] * B, [0.1] * B)
print("round-2 paths ok", fs.get_obs().shape, eroots2.get_distributions()[:1])
torch.cuda.synchronize()
print("sanitize script finished")
