"""The tensor-core DownSample tower with its fused ResBlock kernel (k_resblock_tc): initial_inference against the PyTorch fp32
restatement (oracle/model_ref.py) at the 1e-5 parity tolerance, at both frame sizes and at batch sizes that leave a partial image
group and a last band shorter than the others; and uint8 frames, scaled inside the stem, equal to the scaled float frames bit for
bit."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = dict(rtol=1e-5, atol=1e-5)


def _models(A, obs, seed):
    import lightzero_b200 as lzb
    from oracle.model_ref import MuZeroModelRef, emulate_trained_
    torch.manual_seed(seed)
    ref = emulate_trained_(MuZeroModelRef(obs, A), seed)
    cu = lzb.MuZeroModel(observation_shape=obs, action_space_size=A).load_state_dict(ref.state_dict())
    cu.set_math("tc3")
    return ref, cu


@pytest.mark.parametrize("px", [84, 96])
@pytest.mark.parametrize("B", [1, 3, 131, 1024])
def test_tower_initial_inference_matches_oracle(px, B):
    A = 18
    ref, cu = _models(A, (4, px, px), seed=11)
    obs = torch.rand(B, 4, px, px, generator=torch.Generator().manual_seed(B))
    with torch.no_grad():
        exp = ref.initial_inference(obs)
    out = cu.initial_inference(obs.cuda())
    assert torch.allclose(out.latent_state.cpu(), exp.latent_state, **TOL)
    assert torch.allclose(out.policy_logits.cpu(), exp.policy_logits, **TOL)
    assert torch.allclose(out.value.cpu(), exp.value, **TOL)


def test_tower_uint8_frames_equal_scaled_float_frames():
    from lightzero_b200.collect import MuZeroCollectPolicy
    B, A, S = 131, 18, 4
    _, cu = _models(A, (4, 84, 84), seed=12)
    u8 = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(5))
    f32 = torch.from_numpy((u8.numpy() / 255.).astype(np.float32))
    pol = MuZeroCollectPolicy(cu, dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    mask = torch.ones(B, A, dtype=torch.uint8)
    noise = torch.from_numpy(np.random.default_rng(0).dirichlet([0.3] * A, size=B).astype(np.float32))
    res = []
    for o in (f32.cuda(), u8.cuda()):
        r = pol.search_batch(o, mask, noise, None, deterministic=True, read_back=True)
        res.append({k: v.clone() for k, v in r.items()})
    for k in ("visits", "values", "pred_value", "policy_logits"):
        assert torch.equal(res[0][k], res[1][k]), k
