"""GPU parity tests of the CUDA MuZero model (lz_model_*) against the plain-PyTorch fp32 restatement
of the reference model (oracle/model_ref.py), tolerance 1e-5 (north_star) on every logit / latent.

Scalar outputs (after InverseScalarTransform) are compared at 2e-4: the reference's fp32 formula
sqrt(1 + 4*eps*(|v|+1+eps)) - 1 cancels ~9 bits, so ITS OWN output is quantised in steps of ~1.2e-4
around |v| < 1 (one ulp of the sqrt argument); two correct fp32 softmax implementations that differ
by 1e-7 in v land on adjacent quanta ~0.3% of the time (DESIGN.md, "scalar transform quantisation").
The pre-transform expectation is therefore checked separately at 1e-5."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = dict(rtol=1e-5, atol=1e-5)


def _models(A, seed=0, obs=(4, 84, 84), nres=1):
    import lightzero_b200 as lzb
    from oracle.model_ref import MuZeroModelRef, emulate_trained_
    torch.manual_seed(seed)
    ref = emulate_trained_(MuZeroModelRef(obs, A, num_res_blocks=nres), seed)
    cu = lzb.MuZeroModel(observation_shape=obs, action_space_size=A, num_res_blocks=nres).load_state_dict(ref.state_dict())
    return ref, cu


@pytest.mark.parametrize("B,A", [(5, 6), (130, 18), (300, 6), (1024, 18)])
def test_initial_inference_matches_oracle(B, A):
    ref, cu = _models(A)
    obs = torch.rand(B, 4, 84, 84)
    with torch.no_grad():
        exp = ref.initial_inference(obs)
    out = cu.initial_inference(obs.cuda(), return_scalar_value=True)
    assert out.latent_state.shape == exp.latent_state.shape
    assert torch.allclose(out.latent_state.cpu(), exp.latent_state, **TOL)
    assert torch.allclose(out.policy_logits.cpu(), exp.policy_logits, **TOL)
    assert torch.allclose(out.value.cpu(), exp.value, **TOL)
    assert out.reward == [0.] * B
    from oracle.model_ref import DiscreteSupport, InverseScalarTransform
    inv = InverseScalarTransform(DiscreteSupport(-300., 301., 1.))
    assert torch.allclose(out.value_scalar.cpu(), inv(exp.value).reshape(-1), rtol=2e-4, atol=2e-4)


@pytest.mark.parametrize("B,A", [(7, 6), (130, 18), (520, 6), (1024, 18)])
def test_recurrent_inference_matches_oracle(B, A):
    ref, cu = _models(A, seed=1)
    g = torch.Generator().manual_seed(B)
    latent = torch.rand(B, 64, 6, 6, generator=g) * 2.0
    action = torch.randint(0, A, (B,), generator=g)
    with torch.no_grad():
        exp = ref.recurrent_inference(latent, action)
    out = cu.recurrent_inference(latent.cuda(), action.cuda(), return_scalars=True)
    assert torch.allclose(out.latent_state.cpu(), exp.latent_state, **TOL)
    assert torch.allclose(out.reward.cpu(), exp.reward, **TOL)
    assert torch.allclose(out.value.cpu(), exp.value, **TOL)
    assert torch.allclose(out.policy_logits.cpu(), exp.policy_logits, **TOL)
    from oracle.model_ref import DiscreteSupport, InverseScalarTransform
    inv = InverseScalarTransform(DiscreteSupport(-300., 301., 1.))
    assert torch.allclose(out.value_scalar.cpu(), inv(exp.value).reshape(-1), rtol=2e-4, atol=2e-4)
    assert torch.allclose(out.reward_scalar.cpu(), inv(exp.reward).reshape(-1), rtol=2e-4, atol=2e-4)
    # (B,1) actions, as the reference accepts (muzero_model.py:334-337)
    out2 = cu.recurrent_inference(latent.cuda(), action.cuda().unsqueeze(-1))
    assert torch.equal(out2.policy_logits, out.policy_logits)


def test_two_res_blocks_and_96px():
    ref, cu = _models(6, seed=2, obs=(4, 96, 96), nres=2)
    obs = torch.rand(9, 4, 96, 96)
    with torch.no_grad():
        exp = ref.initial_inference(obs)
        exp2 = ref.recurrent_inference(exp.latent_state, torch.arange(9) % 6)
    out = cu.initial_inference(obs.cuda())
    assert torch.allclose(out.latent_state.cpu(), exp.latent_state, **TOL)
    assert torch.allclose(out.value.cpu(), exp.value, **TOL)
    out2 = cu.recurrent_inference(exp.latent_state.cuda(), (torch.arange(9) % 6).cuda())
    assert torch.allclose(out2.latent_state.cpu(), exp2.latent_state, **TOL)
    assert torch.allclose(out2.reward.cpu(), exp2.reward, **TOL)


def test_inverse_scalar_transform_matches_reference_forms():
    """lzero/policy/tests/test_scaling_transform.py:7-19: the class and the function agree exactly
    (checked on the oracle restatement), and the CUDA transform agrees with both within the
    quantisation bound; the softmax expectation itself within 1e-5."""
    import lightzero_b200 as lzb
    from oracle.model_ref import DiscreteSupport, InverseScalarTransform, inverse_scalar_transform
    torch.manual_seed(0)
    logits = torch.randn(16, 601)
    sup = DiscreteSupport(-300., 301., 1.)
    a = InverseScalarTransform(sup)(logits.clone())
    b = inverse_scalar_transform(logits.clone(), sup)
    assert torch.equal(a, b)
    cu = lzb.InverseScalarTransform(lzb.DiscreteSupport(-300., 301., 1.))
    c = cu(logits.cuda()).cpu()
    assert c.shape == a.shape
    assert torch.allclose(c, a, rtol=2e-4, atol=2e-4)
    # peaked distributions: large magnitudes
    big = torch.zeros(8, 601)
    big[torch.arange(8), torch.tensor([0, 100, 300, 301, 400, 600, 299, 50])] = 30.0
    assert torch.allclose(cu(big.cuda()).cpu(), InverseScalarTransform(sup)(big.clone()), rtol=1e-4, atol=2e-4)


def test_model_rejects_unsupported_configs():
    import lightzero_b200 as lzb
    with pytest.raises(NotImplementedError):
        lzb.MuZeroModel(categorical_distribution=False)
    with pytest.raises(Exception):
        lzb.MuZeroModel(observation_shape=(4, 64, 64))
    m = lzb.MuZeroModel()
    with pytest.raises(RuntimeError):
        m.initial_inference(torch.zeros(1, 4, 84, 84).cuda())
    # the conv models run on the tensor cores only: tc3 (mode 1) or tc1 (mode 2)
    with pytest.raises(ValueError, match="tc3"):
        m.set_math("fp32")
    from lightzero_b200 import cabi
    with pytest.raises(cabi.LzError, match="tc3"):
        m.set_math(0)                                               # mode 0 passed straight to lz_model_set_math


# ------------------------------------------------------------------ tensor-core path (lz_model_set_math)
@pytest.mark.parametrize("B,A", [(7, 6), (50, 18), (1000, 6), (1024, 18)])
def test_tensor_core_3xfp16_recurrent_matches_oracle(B, A):
    """math='tc3': wgmma MMAs on fp16 hi/lo splits (3 passes), fp32 accumulation in registers -- must meet the
    1e-5 bar against the fp32 restatement."""
    ref, cu = _models(A, seed=4)
    cu.set_math("tc3")
    g = torch.Generator().manual_seed(B)
    latent = torch.rand(B, 64, 6, 6, generator=g) * 2.0
    action = torch.randint(0, A, (B,), generator=g)
    with torch.no_grad():
        exp = ref.recurrent_inference(latent, action)
    out = cu.recurrent_inference(latent.cuda(), action.cuda(), return_scalars=True)
    assert torch.allclose(out.latent_state.cpu(), exp.latent_state, **TOL)
    assert torch.allclose(out.reward.cpu(), exp.reward, **TOL)
    assert torch.allclose(out.value.cpu(), exp.value, **TOL)
    assert torch.allclose(out.policy_logits.cpu(), exp.policy_logits, **TOL)
    from oracle.model_ref import DiscreteSupport, InverseScalarTransform
    inv = InverseScalarTransform(DiscreteSupport(-300., 301., 1.))
    assert torch.allclose(out.value_scalar.cpu(), inv(exp.value).reshape(-1), rtol=2e-4, atol=2e-4)
    assert torch.allclose(out.reward_scalar.cpu(), inv(exp.reward).reshape(-1), rtol=2e-4, atol=2e-4)


@pytest.mark.parametrize("B,A,nres", [(5, 6, 1), (300, 18, 1), (9, 6, 2), (1024, 18, 1)])
def test_tensor_core_3xfp16_initial_matches_oracle(B, A, nres):
    ref, cu = _models(A, seed=5, nres=nres)
    cu.set_math("tc3")
    obs = torch.rand(B, 4, 84, 84)
    with torch.no_grad():
        exp = ref.initial_inference(obs)
        exp2 = ref.recurrent_inference(exp.latent_state, torch.arange(B) % A)
    out = cu.initial_inference(obs.cuda())
    assert torch.allclose(out.latent_state.cpu(), exp.latent_state, **TOL)
    assert torch.allclose(out.policy_logits.cpu(), exp.policy_logits, **TOL)
    assert torch.allclose(out.value.cpu(), exp.value, **TOL)
    out2 = cu.recurrent_inference(exp.latent_state.cuda(), (torch.arange(B) % A).cuda())
    assert torch.allclose(out2.latent_state.cpu(), exp2.latent_state, **TOL)
    assert torch.allclose(out2.reward.cpu(), exp2.reward, **TOL)


def test_tensor_core_single_pass_is_close():
    """math='tc1' (one fp16 pass): not the parity mode; logits within 1e-3 of fp32."""
    ref, cu = _models(6, seed=6)
    cu.set_math("tc1")
    latent = torch.rand(64, 64, 6, 6) * 2.0
    action = torch.randint(0, 6, (64,))
    with torch.no_grad():
        exp = ref.recurrent_inference(latent, action)
    out = cu.recurrent_inference(latent.cuda(), action.cuda())
    assert torch.allclose(out.latent_state.cpu(), exp.latent_state, rtol=5e-3, atol=5e-3)
    assert torch.allclose(out.value.cpu(), exp.value, rtol=1e-3, atol=1e-3)
    assert torch.allclose(out.policy_logits.cpu(), exp.policy_logits, rtol=1e-3, atol=1e-3)
